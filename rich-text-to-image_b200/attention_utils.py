"""Token maps: layer allow-lists and get_token_maps (drop-in for utils/attention_utils.py:12-67, 233-341).

The captured maps arrive as fp32 DEVICE tensors (unet.TokenMapAccumulator) instead of fp16 CPU tensors:
averaging and the bicubic resizes run on the GPU, and so does the spectral clustering of the affinity
(utils/attention_utils.py:262-265): `spectral_clustering` takes the spectral embedding from a float64 `eigh` of the
normalised Laplacian and runs the 100 k-means restarts in one kernel (rtti_kmeans_fit), with the random draws taken
from NumPy's global RandomState exactly as scikit-learn takes them, so the segment labels are the ones scikit-learn's
SpectralClustering gives for the same affinity. Affinities whose k-th eigenvalue is not separated from the next one
are handed to scikit-learn (see EIGENGAP_MIN). Maps on the CPU (the reference's fp16 host maps) keep the
scikit-learn call. The debug JPEG / matplotlib dumps of the reference are not reproduced.
"""
import random

import numpy as np
import torch

SelfAttentionLayers = [f"{b}.transformer_blocks.0.attn1" for b in (
    "down_blocks.0.attentions.0", "down_blocks.0.attentions.1", "down_blocks.1.attentions.0",
    "down_blocks.1.attentions.1", "down_blocks.2.attentions.0", "down_blocks.2.attentions.1",
    "mid_block.attentions.0", "up_blocks.1.attentions.0", "up_blocks.1.attentions.1", "up_blocks.1.attentions.2",
    "up_blocks.2.attentions.0", "up_blocks.2.attentions.1", "up_blocks.2.attentions.2", "up_blocks.3.attentions.0",
    "up_blocks.3.attentions.1", "up_blocks.3.attentions.2")]

CrossAttentionLayers = [f"{b}.transformer_blocks.0.attn2" for b in (
    "down_blocks.1.attentions.0", "down_blocks.2.attentions.0", "down_blocks.2.attentions.1",
    "mid_block.attentions.0", "up_blocks.1.attentions.0", "up_blocks.1.attentions.1", "up_blocks.1.attentions.2",
    "up_blocks.2.attentions.1")]

CrossAttentionLayers_XL = (
    [f"down_blocks.2.attentions.1.transformer_blocks.{i}.attn2" for i in (3, 4)]
    + [f"mid_block.attentions.0.transformer_blocks.{i}.attn2" for i in (0, 1, 2, 3)]
    + [f"up_blocks.0.attentions.0.transformer_blocks.{i}.attn2" for i in (1, 2, 3, 4, 5, 6, 7)]
    + ["up_blocks.1.attentions.0.transformer_blocks.0.attn2"])


def seed_everything(seed):
    """utils/richtext_utils.py:22-27."""
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed)


def _resize(x, size):
    return torch.nn.functional.interpolate(x, size, mode="bicubic", antialias=True)


def self_affinity(selfattn_maps, resolution=32):
    """utils/attention_utils.py:241-256: layers whose side is `resolution`, averaged -> [res^2, res^2] (device)."""
    keep = []
    for m in selfattn_maps.values():
        r = int(round(float(np.sqrt(m.shape[1]))))
        if r != resolution:
            continue
        a = m.reshape(1, r, r, r * r).permute(3, 0, 1, 2).float()
        a = _resize(a, (resolution, resolution))  # identity-sized resize, kept because antialiased bicubic is not a no-op
        keep.append(a.permute(1, 2, 3, 0).reshape(1, resolution ** 2, r * r))
    return torch.cat(keep).mean(0)


def cross_maps_mean(crossattn_maps, resolution=32):
    """utils/attention_utils.py:281-291 -> [res, res, 77] (device)."""
    outs = []
    for m in crossattn_maps.values():
        r = int(round(float(np.sqrt(m.shape[1]))))
        a = m.reshape(1, r, r, -1).permute(0, 3, 1, 2).float()
        outs.append(_resize(a, (resolution, resolution)).permute(0, 2, 3, 1))
    return torch.cat(outs).mean(0)


_PALETTE = np.array([[68, 1, 84], [59, 82, 139], [33, 145, 140], [94, 201, 98], [253, 231, 37], [230, 85, 13], [158, 1, 66],
                     [116, 196, 118], [107, 174, 214], [240, 240, 240], [82, 82, 82], [188, 128, 189]], dtype=np.uint8)


def render_segments(clusters, scale=8):
    """uint8 RGB image of the segment label map (the reference returns a matplotlib canvas of `plt.imshow(clusters)`,
    utils/attention_utils.py:266-276; same content, not the same pixels: matplotlib is not a dependency here)."""
    img = _PALETTE[np.asarray(clusters) % len(_PALETTE)]
    return np.repeat(np.repeat(img, scale, axis=0), scale, axis=1)


def render_token_maps(resized):
    """uint8 grey image with the region masks side by side (stands in for plot_attention_maps, :96-149, 334-335)."""
    tiles = [(m.clamp(0, 1) * 255).round().to(torch.uint8).cpu().numpy() for m in resized]
    return np.concatenate(tiles, axis=1)


# Smallest eigengap lambda_{k+1} - lambda_k of the normalised Laplacian for which spectral_clustering runs on the
# device. Below it the k-th eigenvector is only defined up to rounding: scikit-learn's own float32 ARPACK embedding,
# and with it its labels, are then decided by rounding noise that a different eigensolver cannot reproduce. With the
# guard disabled, eigh + the restated kernel gave scikit-learn's labels and RNG state at gaps of 3.8e-7, 1.0e-6, 2.0e-6
# and 3.9e-6 (near-uniform affinities, k = 4; GAP_SWEEP in tests/test_token_map_clustering.py), 3.9e-6 to 1.3e-5
# (synth_maps, k = 9) and 2.5e-4 and up (soft blobs). Near-uniform affinities at k = 9 with gaps of 1.2e-11 and 4.9e-12 gave different labels. The threshold
# keeps the device path to gaps that were shown to match, with the smallest matching gap (3.8e-7) below it.
EIGENGAP_MIN = 1e-6


def kmeans_draws(rs, n, k, n_init):
    """The random numbers KMeans(k, n_init=n_init).fit takes from RandomState `rs` for n samples of unit weight, in the
    order it takes them, as [n_init, 1 + (k-1)*trials] float64: per restart the index of the first centre
    (`rs.choice(n, p=w)`) and then the k-1 `rs.uniform(size=trials)` draws of k-means++
    (sklearn/cluster/_kmeans.py:_kmeans_plusplus). Leaves `rs` in the state KMeans leaves it in."""
    trials = 2 + int(np.log(k))
    u = rs.random_sample(n_init * (1 + (k - 1) * trials)).reshape(n_init, -1)
    p = np.ones(n, np.float32)
    cdf = (p / p.sum()).astype(np.float64).cumsum()     # RandomState.choice(n, p=...)
    cdf /= cdf[-1]
    u[:, 0] = cdf.searchsorted(u[:, 0], side="right")
    return u


def spectral_embedding(affinity, k):
    """[n, k] float32 embedding that scikit-learn's SpectralClustering feeds to k-means, up to a rotation inside each
    eigenspace (which k-means++ and Lloyd do not see), and the eigenvalues of the normalised Laplacian (float64).
    Same construction as sklearn.manifold.spectral_embedding with drop_first=False: S = (A + A^T)/2, degrees without
    the self-loops (zero degrees count as 1), L = I - D^-1/2 S D^-1/2 with unit diagonal, the k eigenvectors of the
    smallest eigenvalues divided by sqrt(degree)."""
    a = affinity.to(torch.float64)
    s = 0.5 * (a + a.T)
    deg = s.sum(1) - s.diagonal()
    deg = torch.where(deg == 0, torch.ones_like(deg), deg)
    dh = deg.sqrt()
    lap = -s / dh[:, None] / dh[None, :]
    lap.diagonal().fill_(1.0)
    evals, evecs = torch.linalg.eigh(lap)
    return (evecs[:, :k] / dh[:, None]).to(torch.float32), evals


def select_restart(labels, inertia, k):
    """KMeans.fit's choice among restarts: a restart replaces the best so far only when its inertia is strictly lower
    and its labels are not the same clustering up to a renaming."""
    def same(a, b):   # sklearn's _is_same_clustering: every label of a maps to one label of b
        return len(np.unique(a.astype(np.int64) * k + b)) == len(np.unique(a))
    best = 0
    for r in range(1, len(inertia)):
        if inertia[r] < inertia[best] and not same(labels[r], labels[best]):
            best = r
    return best


def _sklearn_spectral(affinity, n_clusters, n_init):
    from sklearn.cluster import SpectralClustering
    sc = SpectralClustering(n_clusters, affinity="precomputed", n_init=n_init, assign_labels="kmeans")
    return sc.fit_predict(affinity.cpu().numpy()).astype(np.int32)


def spectral_clustering(affinity, n_clusters, n_init=100, kmeans_fit=None):
    """Drop-in for SpectralClustering(n_clusters, affinity="precomputed", n_init=n_init, assign_labels="kmeans")
    .fit_predict(affinity) on NumPy's global RandomState: the same int32 labels [n], and np.random left in the same
    state. affinity: [n, n] float32 tensor (CUDA for the kernel path). kmeans_fit defaults to rtti_b200.ops.kmeans_fit
    (the tests substitute a NumPy restatement).
    The affinity is handed to scikit-learn instead when the kernel does not take the shape (k > 32, n > 4096, ...),
    when the eigengap lambda_{k+1} - lambda_k is below EIGENGAP_MIN, or when a restart relocated empty clusters in an
    order scikit-learn leaves unspecified (the RNG is rewound first)."""
    from . import ops
    n = affinity.shape[0]
    if not ops.kmeans_supported(n, n_clusters):
        return _sklearn_spectral(affinity, n_clusters, n_init)
    emb, evals = spectral_embedding(affinity, n_clusters)
    if n_clusters < n and float(evals[n_clusters] - evals[n_clusters - 1]) < EIGENGAP_MIN:
        return _sklearn_spectral(affinity, n_clusters, n_init)
    rs = np.random.mtrand._rand
    state = rs.get_state()
    rs.uniform(-1, 1, n)   # the ARPACK start vector (sklearn.utils._arpack._init_arpack_v0)
    draws = kmeans_draws(rs, n, n_clusters, n_init)
    if kmeans_fit is None:
        kmeans_fit = ops.kmeans_fit
        draws = torch.from_numpy(draws).to(emb.device)
    labels, inertia, _, flags = (np.asarray(v.cpu()) if torch.is_tensor(v) else np.asarray(v)
                                 for v in kmeans_fit(emb, draws))
    if flags.any():
        rs.set_state(state)
        return _sklearn_spectral(affinity, n_clusters, n_init)
    return labels[select_restart(labels, inertia, n_clusters)].astype(np.int32)


def get_token_maps(selfattn_maps, crossattn_maps, n_maps, save_dir, width, height, obj_tokens, seed=0,
                   tokens_vis=None, preprocess=False, segment_threshold=0.3, num_segments=5, return_vis=False,
                   save_attn=False, device=None, return_clusters=False):
    """Same signature and return value as utils/attention_utils.py:233-341: a list of N masks
    [1, 4, height, width] fp32 (spans..., background) that sum to one per pixel."""
    resolution = 32
    some = next(iter(selfattn_maps.values()))
    device = device or some.device
    aff = self_affinity(selfattn_maps, resolution)
    seed_everything(seed)
    if aff.is_cuda:
        clusters = spectral_clustering(aff, num_segments).reshape(resolution, resolution)
    else:   # the reference's fp16 host maps: scikit-learn, the only path on the CPU
        from sklearn.cluster import SpectralClustering
        sc = SpectralClustering(num_segments, affinity="precomputed", n_init=100, assign_labels="kmeans")
        clusters = sc.fit_predict(aff.numpy()).reshape(resolution, resolution)
    cross = cross_maps_mean(crossattn_maps, resolution).cpu().numpy()

    normalized_span_maps = []
    for token_ids in obj_tokens:
        span = cross[:, :, np.asarray(token_ids.cpu())]
        norm = np.zeros_like(span)
        for i in range(span.shape[-1]):
            cur = span[:, :, i]
            norm[:, :, i] = (cur - np.abs(cur.min())) / (cur.max() - cur.min())   # sic, :302-303
        normalized_span_maps.append(norm)
    fg = [np.zeros([resolution, resolution]) for _ in normalized_span_maps]
    bg = np.zeros([resolution, resolution])
    for c in range(num_segments):
        cluster_mask = np.zeros_like(clusters)
        cluster_mask[clusters == c] = 1.0
        is_fg = False
        for norm, fg_map, token_ids in zip(normalized_span_maps, fg, obj_tokens):
            scores = [(cluster_mask * norm[:, :, i]).sum() / cluster_mask.sum() for i in range(len(token_ids))]
            if max(scores) > segment_threshold:
                fg_map += cluster_mask
                is_fg = True
        if not is_fg:
            bg += cluster_mask
    fg.append(bg)
    maps = torch.from_numpy(np.stack(fg)).to(device)                       # float64, as the reference
    resized = _resize(maps[:, None], (height, width))[:, 0].clamp(0, 1)     # (height, width) order, :325
    resized = resized / (resized.sum(0, True) + 1e-8)
    out = [m[None, None].repeat(1, 4, 1, 1).to(torch.float32) for m in resized]
    if return_clusters:   # (masks, int label image): extension used by the tests
        return out, clusters
    if return_vis:
        return out, render_segments(clusters), render_token_maps(resized)
    return out
