"""rtti_b200 — region-diffusion sampler for the H100 (drop-in for the hot path of
songweige/rich-text-to-image: RegionDiffusion / RegionDiffusionXL, get_token_maps).

Python host code calling hand-written sm_90a CUDA through the C ABI in include/rtti_b200.h.
The directory name carries a dash, so the importable alias is the top-level package `rtti_b200`.
"""
__version__ = "0.1.0"
