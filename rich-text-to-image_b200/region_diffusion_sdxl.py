"""RegionDiffusionXL — H100 drop-in for models/region_diffusion_sdxl.py of the reference.

Same public surface (`sample(...)`, `register_tokenmap_hooks / remove_tokenmap_hooks`, `.masks`,
`.selfattn_maps / .crossattn_maps / .n_maps`, `.unet .vae .scheduler .tokenizer`) and the same per-step
semantics (models/region_diffusion_sdxl.py:772-914), re-organised for the hardware:

  * the 2 + 2*inject + (N-1) UNet passes of a step (uncond, base+font-size, reference uncond, reference
    base, N-1 regions; :787-821) run as ONE batched UNet call — they share the timestep and, up to the
    reference latent, the input; the hook choreography becomes a RegionControl;
  * region blend + CFG (+ guidance rescale) + scheduler update is one kernel (rtti_region_blend_cfg, or
    rtti_region_blend_cfg_rescale with guidance_rescale > 0, in the form of the scheduler's update: stepping.py);
    colour-guidance loss fwd/bwd,
    guidance update, x0 prediction and background injection are kernels too;
  * with torch.distributed initialised the passes are sharded over the ranks (region_parallel.py) and the
    per-pass noise predictions are all-gathered before the (replicated, deterministic) blend.
"""
import math
from typing import List, Optional

import numpy as np
import torch

from . import ops, region_parallel, stepping, vae_guidance
from .attention_utils import CrossAttentionLayers_XL
from .lora import LoraLoaderMixin
from .schedulers import DDIMScheduler, EulerDiscreteScheduler
from .stepping import _step_kind  # noqa: F401  (re-exported)
from .textual_inversion import TextualInversionLoaderMixin
from .unet import CrossKVCache, RegionControl, TokenMapAccumulator, UNet2DConditionModel, UNetConfig
from .vae import AutoencoderKLDecoder, VAEConfig


def _rescale_phi(guidance_scale, guidance_rescale):
    """The guidance rescale in effect: the reference applies it only with classifier-free guidance on (:903)."""
    return float(guidance_rescale) if guidance_scale > 1.0 and guidance_rescale > 0.0 else 0.0


class StableDiffusionXLPipelineOutput(dict):
    def __init__(self, images):
        super().__init__(images=images)
        self.images = images


class RegionDiffusionXL(LoraLoaderMixin, TextualInversionLoaderMixin):
    def __init__(self, load_path: str = "stabilityai/stable-diffusion-xl-base-1.0", device: str = "cuda",
                 force_zeros_for_empty_prompt: bool = True, unet=None, vae=None, scheduler=None,
                 text_encoders=None):
        """Either pass pre-built components (tests / synthetic benchmarks) or a local diffusers-format
        directory as `load_path` (models/region_diffusion_sdxl.py:87-137 downloads from the hub; there is
        no network here, so only local paths are supported)."""
        self.device = torch.device(device)
        torch.backends.cudnn.benchmark = True   # static shapes: let cuDNN pick its fastest conv algorithm once
        self.device_type = device
        if unet is None:
            from .loading import load_sdxl_components
            unet, vae, scheduler, text_encoders = load_sdxl_components(load_path, self.device)
        self.unet = unet
        self.vae = vae
        self.scheduler = scheduler or EulerDiscreteScheduler()
        self.text_encoders = text_encoders
        self.tokenizer = getattr(text_encoders, "tokenizer", None)
        self.tokenizer_2 = getattr(text_encoders, "tokenizer_2", None)
        self.force_zeros_for_empty_prompt = force_zeros_for_empty_prompt
        self.vae_scale_factor = 8
        self.default_sample_size = unet.config.sample_size
        self.masks = []
        self.attention_maps = None
        self.selfattn_maps = None
        self.crossattn_maps = None
        self.n_maps = None
        self._capture = None
        self.capture_all_resolutions = False
        self._exchanges = {}
        self.use_cuda_graphs = True  # replay the batched UNet pass of a step as one CUDA graph (launch-bound otherwise)
        self.profile_events = None   # dict -> CUDA-event pairs per phase of a step (bench.py breakdown)
        self.fused_exchange = True   # multi-GPU: fused peer-memory gather+blend kernel instead of NCCL all-gather
        self.stripe_guidance = True  # multi-GPU: colour guidance (VAE fwd+bwd) split by image rows over the ranks
        self._stripe_engines = {}
        self.graph_guidance = True   # replay decode -> colour loss -> decoder backward as one CUDA graph (launch-bound on >1 GPU)
        self._guidance_graphs = {}
        self.region_group = None     # torch.distributed group the passes of one image are sharded over (None = all ranks)
        self.remote_qk = True        # multi-GPU: pass D on one rank, its Q|K / feature pushed to the region-pass ranks
        self._remote = {}            # (instead of replicating D on every rank that owns a region pass)
        self.last_step_stats = {}

    @classmethod
    def from_synthetic(cls, unet_cfg: Optional[UNetConfig] = None, vae_cfg: Optional[VAEConfig] = None, seed=0,
                       device="cuda", with_vae=True):
        """Random-weight model of the right architecture (benchmarks / tests; no checkpoints available)."""
        with torch.device(device):  # build directly on the GPU: CPU default-init of 2.6 B parameters is slow
            unet = UNet2DConditionModel(unet_cfg or UNetConfig.sdxl())
        unet.finalize(device).init_synthetic(seed)
        vae = None
        if with_vae:
            vae = AutoencoderKLDecoder(vae_cfg or VAEConfig.sdxl()).init_synthetic(seed + 1).finalize(device)
        return cls(device=device, unet=unet, vae=vae, scheduler=EulerDiscreteScheduler())

    # ------------------------------------------------------------------ token-map capture API
    def register_tokenmap_hooks(self):
        """models/region_diffusion_sdxl.py:959-1009 — here: arm the on-device accumulators."""
        res = None if self.capture_all_resolutions else (32,)
        self._capture = TokenMapAccumulator(CrossAttentionLayers_XL, self_layers=None, start_after=10,
                                            sd_overwrite_bug=False, self_resolutions=res)
        self.selfattn_maps = self._capture.selfattn_maps
        self.crossattn_maps = self._capture.crossattn_maps
        self.n_maps = self._capture.n_maps

    def remove_tokenmap_hooks(self):
        self._capture = None
        self.selfattn_maps = None
        self.crossattn_maps = None
        self.n_maps = None

    def _lora_components(self):
        te = self.text_encoders
        return self.unet, (() if te is None else (te.text_encoder, te.text_encoder_2))

    def _textual_inversion_components(self):
        te = self.text_encoders
        return [] if te is None else [(te.tokenizer, te.text_encoder), (te.tokenizer_2, te.text_encoder_2)]

    # ------------------------------------------------------------------ helpers
    def encode_prompt(self, prompt, negative_prompt):
        if self.text_encoders is None:
            raise RuntimeError("no text encoders loaded: pass prompt_embeds / pooled_prompt_embeds explicitly")
        return self.text_encoders.encode(prompt, negative_prompt, self.device, self.force_zeros_for_empty_prompt)

    def prepare_latents(self, height, width, generator=None, latents=None):
        shape = (1, self.unet.config.in_channels, height // self.vae_scale_factor, width // self.vae_scale_factor)
        if latents is None:
            latents = torch.randn(shape, generator=generator, device=self.device, dtype=torch.float16)
        else:
            latents = latents.to(self.device, torch.float16)
        return latents * self.scheduler.init_noise_sigma

    def predict_x0(self, x_t, eps_t, t):
        """models/region_diffusion_sdxl.py:955-957 (alphas_cumprod[int(t)] with the post-step latents)."""
        alpha = float(self.scheduler.alphas_cumprod[int(float(t))])
        return ops.predict_x0(x_t.contiguous(), eps_t.contiguous(), alpha), alpha

    def _color_guidance(self, latents, noise_pred, t, tfd):
        """models/region_diffusion_sdxl.py:849-867 with the clamp / masked mean / MSE forward+backward in
        rtti_color_loss_fwd_bwd and the VAE (third-party) in PyTorch autograd with frozen weights."""
        x0, alpha = self.predict_x0(latents, noise_pred, t)
        sf = self.vae.config.scaling_factor
        # the reference pairs maps and targets with zip() (sdxl.py:857 / region_diffusion.py:159): sample.py hands over
        # R colour maps + the background map but only R target colours, and the background map is dropped
        n_col = min(len(tfd["color_obj_atten"]), len(tfd["target_RGB"]))
        masks = torch.stack([m[0, 0].to(self.device, torch.float32) for m in tfd["color_obj_atten"][:n_col]]).contiguous()
        tgt = torch.stack([r.reshape(3).to(self.device, torch.float32) for r in tfd["target_RGB"][:n_col]]).contiguous()

        def grad_image(img):
            loss, g = ops.color_loss_fwd_bwd(img[0].contiguous(), masks, tgt)
            self.last_step_stats["color_loss"] = loss
            return g[None]

        z = x0.float() / sf
        engine = self._stripe_engine(x0)
        if self.graph_guidance and isinstance(self.vae, AutoencoderKLDecoder):
            eng = engine if engine is not None else vae_guidance.default_engine(self.vae)
            gkey = (id(eng), tuple(z.shape), tuple(masks.shape))
            gg = self._guidance_graphs.get(gkey)
            if gg is None:
                gg = self._guidance_graphs[gkey] = vae_guidance.GuidanceGraph(eng)
            self.last_step_stats["color_loss"], grad_lat = gg(z.contiguous(), masks, tgt)
            grad_lat = grad_lat / (sf * math.sqrt(alpha))
        else:
            grad_lat = vae_guidance.image_and_latent_grad(self.vae, z, grad_image, engine=engine) / (sf * math.sqrt(alpha))
        atten_all = tfd["color_obj_atten_all"].to(self.device, torch.float32).expand_as(grad_lat).contiguous()
        return ops.latent_guidance_update(latents.contiguous(), grad_lat.contiguous(), atten_all,
                                          float(tfd["color_guidance_weight"]))

    def _stripe_engine(self, x0):
        """Stripe-parallel VAE engine (stripe_parallel.py) when running on >1 GPU, else None (single-GPU engine)."""
        import torch.distributed as dist
        if not (self.stripe_guidance and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
            return None
        from .vae import AutoencoderKLDecoder
        h, w = int(x0.shape[2]), int(x0.shape[3])
        if not isinstance(self.vae, AutoencoderKLDecoder) or x0.shape[0] != 1 or h % dist.get_world_size() != 0:
            return None
        if (h, w) not in self._stripe_engines:   # symmetric arena allocated once per latent shape
            try:
                from .stripe_parallel import StripedDecoderFwdBwd
                self._stripe_engines[(h, w)] = StripedDecoderFwdBwd(self.vae, h, w, self.device)
            except Exception as e:               # no peer-mappable memory: replicated guidance
                import warnings
                warnings.warn(f"rtti_b200: stripe-parallel colour guidance unavailable ({e!r}); running it replicated")
                self.stripe_guidance = False
                return None
        return self._stripe_engines[(h, w)]

    # ------------------------------------------------------------------ sampling
    @torch.no_grad()
    def sample(self, prompt=None, height: Optional[int] = None, width: Optional[int] = None,
               num_inference_steps: int = 50, guidance_scale: float = 5.0, negative_prompt=None,
               num_images_per_prompt: int = 1, eta: float = 0.0, generator=None, latents=None, prompt_embeds=None,
               negative_prompt_embeds=None, pooled_prompt_embeds=None, negative_pooled_prompt_embeds=None,
               output_type: Optional[str] = "pil", return_dict: bool = True, callback=None, callback_steps: int = 1,
               cross_attention_kwargs=None, guidance_rescale: float = 0.0, original_size=None,
               crops_coords_top_left=(0, 0), target_size=None, use_guidance: bool = False,
               inject_selfattn: float = 0.0, inject_background: float = 0.0, text_format_dict: Optional[dict] = None,
               run_rich_text: bool = False):
        """Signature of models/region_diffusion_sdxl.py:556-587. `prompt` is the list of region prompts with the
        base prompt last (sample.py:107); embeddings may be passed instead of text. `guidance_rescale` (applied when
        guidance_scale > 1) rescales the CFG prediction as diffusers' rescale_noise_cfg in both passes; the reference
        implements it for the plain pass only (:903-905) and raises NotImplementedError in the rich-text pass (:827-830).
        `self.scheduler` may be EulerDiscreteScheduler, EulerAncestralDiscreteScheduler, DDIMScheduler,
        DPMSolverMultistepScheduler, UniPCMultistepScheduler, HeunDiscreteScheduler, LMSDiscreteScheduler or
        DPMSolverSinglestepScheduler (schedulers.py); `eta` > 0 (stochastic DDIM, which the reference's plain pass
        forwards to DDIM) is not implemented.
        With a multistep or UniPC scheduler the rich-text pass keeps one history per trajectory: where the reference
        steps the reference latents jointly with the main latents only on a prefix of the steps (inject_selfattn = 0,
        0 < inject_background < 1, :831-846) and then steps the main latents alone, the main latents keep their own
        history here instead of continuing a batch-2 one. UniPC's corrector restarts from its own last corrected
        sample, so colour guidance and background injection reach its next update only through the x0 prediction of
        the next step, as in the reference with UniPC assigned to its scheduler.
        With HeunDiscreteScheduler each iteration is one stage of Heun's method (2N - 1 UNet evaluations for N steps);
        each trajectory keeps the latents and prediction of its last first stage, so colour guidance and background
        injection after a first stage reach the second stage only through its prediction, as in the reference. Where
        the reference stops stepping the reference latents right after a first stage (inject_selfattn = 0), it would
        add a batch-1 prediction to a batch-2 saved state; here the reference latents keep their first-stage value.
        `callback` is called by the reference's rule (:874-877): after the second stages and the last iteration.
        With LMSDiscreteScheduler each trajectory keeps the fp16 predictions of its last three steps. Every step starts
        from the current latents, so colour guidance and background injection carry into the next update in full. As
        with the multistep schedulers, where the reference steps the reference latents jointly only on a prefix of the
        steps (inject_selfattn = 0, 0 < inject_background < 1), it would go on to add a batch-1 prediction to batch-2
        ones; here each trajectory keeps its own history.
        With DPMSolverSinglestepScheduler (DPM-Solver++(2S)) the steps form blocks of two; each trajectory keeps one fp32
        x0 prediction and the fp16 latents that entered its block's first step. The second step restarts from those
        latents, so colour guidance and background injection applied after a first step reach the second step only
        through its prediction, as in the reference with DPMSolverSinglestepScheduler assigned to its scheduler. Where
        the reference steps the reference latents jointly only on a prefix of the steps (inject_selfattn = 0,
        0 < inject_background < 1), here each trajectory keeps its own state; if the prefix ends after a first step, the
        reference latents keep their first-step value, as with Heun and LMS.
        With EulerAncestralDiscreteScheduler the noise z of each step is drawn as diffusers' randn_tensor draws it, fp16,
        from `generator` when one is given (on its device: a CPU generator draws on the CPU), otherwise from the global
        RNG of the sampling device. The plain pass draws [1, ...] per step, as the reference does. The rich-text pass
        draws one [2, ...] tensor on the steps where the reference steps the main and reference latents jointly (first
        half to the main latents, second half to the reference latents) and [1, ...] on the others. Unlike the reference,
        which passes no generator to the rich-text pass's step, that pass also draws from `generator`: a seeded run is
        reproducible from start to end. With generator=None both passes draw exactly what the reference draws. On more
        than one GPU every rank must add the same noise: sample() compares a digest of the noise source's state over
        the ranks once and raises on every rank if they disagree.
        `cross_attention_kwargs={"scale": s}` with a LoRA loaded (load_lora_weights) re-merges it at scale s before the
        prompt is encoded, so the UNet and both text encoders use s. Unlike diffusers, where a call without the keyword
        runs at scale 1.0, the scale stays in effect for later calls. With no LoRA loaded the argument is ignored."""
        if cross_attention_kwargs and "scale" in cross_attention_kwargs and self._lora is not None:
            self.set_lora_scale(cross_attention_kwargs["scale"])
        kind = _step_kind(self.scheduler)
        multistep = kind == "multistep"
        if multistep and eta > 0 and not run_rich_text and isinstance(self.scheduler, DDIMScheduler):
            raise NotImplementedError("RegionDiffusionXL: DDIM with eta > 0 is not implemented")
        height = height or self.default_sample_size * self.vae_scale_factor
        width = width or self.default_sample_size * self.vae_scale_factor
        original_size = original_size or (height, width)
        target_size = target_size or (height, width)
        if prompt_embeds is None:
            prompt_embeds, negative_prompt_embeds, pooled_prompt_embeds, negative_pooled_prompt_embeds = \
                self.encode_prompt(prompt, negative_prompt)
        dev = self.device
        # [uncond, prompts...] like :760-763
        ctx = torch.cat([negative_prompt_embeds, prompt_embeds], 0).to(dev, torch.float16)
        pooled = torch.cat([negative_pooled_prompt_embeds, pooled_prompt_embeds], 0).to(dev, torch.float16)
        time_ids = torch.tensor([list(original_size) + list(crops_coords_top_left) + list(target_size)],
                                dtype=torch.float32, device=dev)
        if kind == "ancestral":
            region_parallel.check_noise_source(generator, dev, group=self.region_group)
        self.scheduler.set_timesteps(num_inference_steps, device=dev)
        timesteps = self.scheduler.timesteps
        latents = self.prepare_latents(height, width, generator, latents)

        if run_rich_text:
            latents = self._rich_text_loop(ctx, pooled, time_ids, latents, timesteps, guidance_scale, use_guidance,
                                           inject_selfattn, inject_background, text_format_dict or {}, callback,
                                           callback_steps, guidance_rescale, generator)
        else:
            latents = self._plain_loop(ctx, pooled, time_ids, latents, timesteps, guidance_scale, callback, callback_steps,
                                       guidance_rescale, generator)

        if output_type == "latent":
            return StableDiffusionXLPipelineOutput(images=latents)
        image = self.vae.decode_tensor(latents.float() / self.vae.config.scaling_factor)
        image = (image / 2 + 0.5).clamp(0, 1)
        if output_type == "pt":
            return StableDiffusionXLPipelineOutput(images=image)
        arr = (image.permute(0, 2, 3, 1).float().cpu().numpy() * 255).round().astype("uint8")
        if output_type == "np":
            return StableDiffusionXLPipelineOutput(images=arr)
        from PIL import Image
        return StableDiffusionXLPipelineOutput(images=[Image.fromarray(a) for a in arr])

    def _plain_loop(self, ctx, pooled, time_ids, latents, timesteps, guidance_scale, callback, callback_steps,
                    guidance_rescale=0.0, generator=None):
        """:879-914 — CFG batch [uncond, cond]; with capture armed the attention kernels accumulate the maps.
        guidance_rescale rescales the CFG prediction inside the blend kernel (:903-905); the scheduler update runs in it
        too (stepping.py), with Euler Ancestral's z [1, ...] drawn after the UNet pass, as the reference's step draws
        it (:908). The callback follows the reference's rule (:874-877): iteration i calls it when (i is the last
        iteration or (i + 1) % scheduler.order == 0) and i % callback_steps == 0 — every iteration
        i % callback_steps == 0 for the order-1 schedulers, only second stages and the last iteration for Heun."""
        phi = _rescale_phi(guidance_scale, guidance_rescale)
        ctx2 = torch.cat([ctx[:1], ctx[-1:]])
        pooled2 = torch.cat([pooled[:1], pooled[-1:]])
        kv = CrossKVCache()
        ones = None
        stepper = stepping.stepper(self.scheduler, latents.shape, latents.device, generator)
        state = stepper.state()
        for i, t in enumerate(timesteps):
            norm = stepper.input_norm(i, t)
            x = (latents if norm is None else latents / norm).expand(2, -1, -1, -1)
            ctrl = RegionControl(capture=self._capture, capture_row=1, kv_cache=kv)
            eps = self.unet(x, t, ctx2, {"text_embeds": pooled2, "time_ids": time_ids}, ctrl)["sample"]
            n = eps[0].numel()
            if ones is None:
                ones = torch.ones(1, n, dtype=torch.float32, device=eps.device)
            stepper.begin(i, t, 1)
            lat = latents.contiguous()
            e16, latents = ops.region_blend_cfg(eps[0:1].contiguous(), [eps[1:2].contiguous()], ones, guidance_scale,
                                                latents=lat, guidance_rescale=phi, step=stepper.step(state))
            state = stepper.advance(state, lat, e16)
            if callback is not None and self._calls_back(i, len(timesteps), callback_steps):
                callback(i, t, latents)
        return latents

    def _calls_back(self, i, n_iterations, callback_steps):
        """The reference's callback rule (:874-877 and :910-914; num_warmup_steps = len(timesteps) - N * order is
        never positive here)."""
        return (i == n_iterations - 1 or (i + 1) % self.scheduler.order == 0) and i % callback_steps == 0

    def build_pass_batch(self, n_regions, inject):
        """Order of the batched passes of one step and the context row each one uses.
        rows index [uncond, region_1..region_{N-1}, base] (ctx); `x_ref` marks the reference-latent passes."""
        last = n_regions  # ctx row of the base prompt
        passes = [dict(kind="A", ctx=0, ref=False), dict(kind="B", ctx=last, ref=False)]
        if inject:
            passes += [dict(kind="C", ctx=0, ref=True), dict(kind="D", ctx=last, ref=True)]
        for j in range(n_regions - 1):
            passes.append(dict(kind="E", ctx=j + 1, ref=False, region=j))
        return passes

    def prepare_rich_text(self, ctx, pooled, time_ids, latents, timesteps, guidance_scale, use_guidance,
                          inject_selfattn, inject_background, tfd, guidance_rescale=0.0, generator=None):
        """Everything of :772-778 that is constant over the steps, as a state object for rich_text_step().
        guidance_rescale: the CFG rescale the reference leaves as a TODO (:827-830), applied to the blended prediction
        (eps_text = the masked sum of the text passes) and, when it is stepped, to the reference-latent pair C/D.
        generator: the source of Euler Ancestral's noise (None: the global RNG of the sampling device)."""
        dev = self.device
        N = len(self.masks)
        assert ctx.shape[0] == N + 1, "prompts must be [region_1..region_{N-1}, base] matching self.masks"
        inject = inject_selfattn > 0 or inject_background > 0
        st = type("RichTextState", (), {})()
        st.ctx, st.pooled, st.time_ids = ctx, pooled, time_ids
        st.latents = latents
        st.latents_ref = latents.clone() if inject else None
        st.timesteps, st.n_t = timesteps, len(timesteps)
        st.guidance_scale, st.use_guidance = guidance_scale, use_guidance
        st.guidance_rescale = _rescale_phi(guidance_scale, guidance_rescale)
        st.inject, st.inject_selfattn, st.inject_background = inject, inject_selfattn, inject_background
        st.tfd = tfd
        st.N = N
        st.masks = torch.stack([m.to(dev, torch.float32).reshape(-1) for m in self.masks]).contiguous()  # [N, n] (:776)
        st.ones = torch.ones(1, latents[0].numel(), dtype=torch.float32, device=dev)
        st.passes = self.build_pass_batch(N, inject)
        st.kind = {p["kind"] + str(p.get("region", "")): k for k, p in enumerate(st.passes)}
        st.plan = region_parallel.RegionParallelPlan(st.passes, inject, group=self.region_group,
                                                     remote_qk=self.remote_qk and self.fused_exchange)
        word_pos, font_size = tfd.get("word_pos"), tfd.get("font_size")
        if word_pos is not None and font_size is not None:
            if int(word_pos.max()) >= ctx.shape[1] or int(word_pos.min()) < 0:   # the reference's advanced indexing raises here
                raise IndexError(f"word_pos {word_pos.tolist()} outside the {ctx.shape[1]} text tokens")
            st.word_pos = word_pos.to(dev, torch.int32).contiguous()
            st.font_size = font_size.to(dev, torch.float32).contiguous()
        else:
            st.word_pos = st.font_size = None
        st.kv_caches = {}
        st.graphs = {}
        st.noise_pred = None
        # the fused scheduler update and its state per trajectory (main, reference)
        st.stepper = stepping.stepper(self.scheduler, latents.shape, dev, generator)
        st.main = st.stepper.state()
        st.ref = st.stepper.state() if inject else None
        return st

    def _unet_pass(self, st, x, t, local, feat_inject_step):
        """The batched UNet call of one step: eager, or (use_cuda_graphs) captured once per batch composition
        and replayed — the pass is ~1400 kernel launches whose CPU launch cost exceeds their GPU time."""
        passes, plan = st.passes, st.plan
        rows = [passes[p]["ctx"] for p in local]
        inj = bool(feat_inject_step and st.inject)
        key = (tuple(local), inj)
        kvc = st.kv_caches.setdefault(tuple(local), CrossKVCache())

        rq = self._remote_qk(st, x) if inj else None
        role = plan.remote_role(local) if rq is not None else None

        def make_ctrl(remote=True):
            ctrl = RegionControl(kv_cache=kvc)
            if inj:
                src = plan.injection_sources(local)                                     # :1018-1061
                if src is not None:         # None: this rank's region passes take pass D's tensors from another rank
                    ctrl.qk_src = src
                    ctrl.feature_src = src
                    ikey = ("idx",) + key
                    if ikey not in st.graphs:   # built once, outside any capture
                        st.graphs[ikey] = torch.as_tensor(src, device=self.device)
                    ctrl.feature_idx = st.graphs[ikey]
                if rq is not None and remote:
                    ctrl.remote = rq.begin_pass(role)
            if st.word_pos is not None:
                ctrl.word_pos, ctrl.font_size = st.word_pos, st.font_size               # :792-797
                ctrl.fs_batch_mask = sum(1 << k for k, p in enumerate(local) if passes[p]["kind"] == "B")
            return ctrl

        def unet(x_, t_, ctx_, added_, remote=True):
            """`remote=False`: the eager warm-up before a capture — pass D's tensors are neither pushed nor awaited
            (region passes use their own Q, K; the result is discarded). Producer and consumers then execute the
            hand-off exactly once per step — in the replayed graph — which is what keeps the single-buffered receive
            regions safe and every rank's sequence base in step."""
            out = self.unet(x_, t_, ctx_, added_, make_ctrl(remote))["sample"]
            if rq is not None and remote:
                rq.end_pass()
            return out

        if not self.use_cuda_graphs:
            return unet(x, t, st.ctx[rows], {"text_embeds": st.pooled[rows], "time_ids": st.time_ids})
        g = st.graphs.get(key)
        if g is None:
            g = {"x": torch.empty_like(x), "t": torch.zeros(1, dtype=torch.float32, device=self.device),
                 "ctx": st.ctx[rows].contiguous(), "added": {"text_embeds": st.pooled[rows].contiguous(), "time_ids": st.time_ids}}
            g["x"].copy_(x)
            g["t"].fill_(float(t))
            side = torch.cuda.Stream(device=self.device)
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):      # warm-up outside capture: fills the prompt K/V cache, sets func attributes
                unet(g["x"], g["t"], g["ctx"], g["added"], remote=False)
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            n0 = ops.LAUNCHES
            with torch.cuda.graph(graph, pool=st.graphs.get("pool")):
                g["out"] = unet(g["x"], g["t"], g["ctx"], g["added"])
            g["launches"] = ops.LAUNCHES - n0   # rtti kernels inside the graph (for the launch accounting)
            if "pool" not in st.graphs:   # the graphs of one sampling call share a memory pool
                st.graphs["pool"] = graph.pool()
            g["graph"] = graph
            st.graphs[key] = g
        g["x"].copy_(x)
        g["t"].fill_(float(t))
        g["graph"].replay()
        ops._count(g["launches"])
        return g["out"]

    def _remote_qk(self, st, x):
        """RemoteQK buffers for this latent shape (created collectively by every rank of the region group on the first
        feature-injection step), or None: single GPU, remote_qk off, no peer-mappable memory, or the plan replicates D."""
        if not (st.plan.remote_qk and st.plan.world > 1):
            return None
        key = (int(x.shape[2]), int(x.shape[3]))
        if key not in self._remote:
            try:
                self._remote[key] = region_parallel.RemoteQK(self.unet.injection_layout(*key), self.device, group=self.region_group)
            except Exception as e:   # no peer-mappable memory (the same on every rank): replicate pass D instead
                import warnings
                warnings.warn(f"rtti_b200: RemoteQK unavailable ({e!r}); pass D is replicated on the region-pass ranks")
                self._remote[key] = None
        if self._remote[key] is None:
            st.plan.remote_qk = False
            st.plan._cache.clear()
        return self._remote[key]

    def rich_text_step(self, st, i):
        """One iteration of the region loop, models/region_diffusion_sdxl.py:779-878."""
        t = st.timesteps[i]
        passes, kind, plan, N = st.passes, st.kind, st.plan, st.N
        feat_inject_step = bool(float(t) > (1 - st.inject_selfattn) * 1000)            # :782
        background_inject_step = i < st.inject_background * st.n_t                      # :783
        norm = st.stepper.input_norm(i, t)                                               # :784
        if feat_inject_step and st.inject:
            self._remote_qk(st, st.latents)   # collective on first use: every rank of the group, also those without passes
        local = plan.local_passes(feat_inject_step)
        pe = self.profile_events
        if pe is not None:
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            ev[0].record()
        if local:
            x = torch.cat([(st.latents_ref if passes[p]["ref"] else st.latents) for p in local])
            if norm is not None:
                x = x * (1.0 / norm)
            eps_local = self._unet_pass(st, x, t, local, feat_inject_step)
        else:   # more ranks than passes on this step: this rank only takes part in the exchange
            eps_local = st.latents.new_empty((0,) + tuple(st.latents.shape[1:]))
            rq = self._remote_qk(st, st.latents) if (feat_inject_step and st.inject) else None
            if rq is not None:   # keep this rank's sequence base in step with the ranks that ran a pass
                rq.begin_pass(None)
                rq.end_pass()
        if pe is not None:
            ev[1].record()
        step_ref = st.inject and (st.inject_selfattn > 0 or background_inject_step)                       # :830-841
        stepper = st.stepper
        stepper.begin(i, t, 2 if step_ref else 1)
        st.latents = lat = st.latents.contiguous()
        if step_ref:
            st.latents_ref = lat_ref = st.latents_ref.contiguous()
        ex = None
        if plan.world > 1 and self.fused_exchange:
            xkey = (tuple(p["kind"] for p in passes), st.latents[0].numel())
            if xkey not in self._exchanges:   # symmetric buffers are allocated once per problem shape
                try:
                    self._exchanges[xkey] = region_parallel.PeerExchange(passes, st.latents[0].numel(), self.device, group=self.region_group)
                except Exception as e:        # no peer-mappable memory (e.g. GPUs without P2P): NCCL all-gather path
                    import warnings
                    warnings.warn(f"rtti_b200: symmetric peer memory unavailable ({e!r}); using the NCCL all-gather exchange")
                    self.fused_exchange = False
            ex = self._exchanges.get(xkey)
        if ex is not None:
            # fused all-gather + blend + CFG + scheduler update over NVLink peer memory (csrc/gather_blend.cu); the
            # reference trajectory's stepped prediction is written into eps_ref where its state keeps it
            _, owner = plan._plan(feat_inject_step)
            sid = ex.publish(eps_local, local, owner)
            eps_ref = torch.empty_like(lat_ref) if step_ref and stepper.writes_eps_ref() else None
            st.noise_pred, st.latents, ref_out = ops.gather_blend_step(
                ex.slot_ptrs, ex.flag_ptrs, ex.rank, ex.slot_owner(owner), N, st.masks, st.guidance_scale, lat,
                lat_ref if step_ref else None, 0.0, sid, guidance_rescale=st.guidance_rescale,
                step=stepper.step_pair(st.main, st.ref, step_ref, eps_ref))
            if step_ref:
                st.latents_ref = ref_out
        else:
            eps = plan.gather(eps_local, local, feat_inject_step)   # NCCL all-gather; identity on one GPU
            one = lambda name: eps[kind[name]:kind[name] + 1].contiguous()
            regions = [one(f"E{j}") for j in range(N - 1)] + [one("B")]
            st.noise_pred, st.latents = ops.region_blend_cfg(one("A"), regions, st.masks, st.guidance_scale, latents=lat,
                                                              guidance_rescale=st.guidance_rescale,
                                                              step=stepper.step(st.main))  # :810-830
            if step_ref:
                eps_ref, st.latents_ref = ops.region_blend_cfg(one("C"), [one("D")], st.ones, st.guidance_scale,
                                                               latents=lat_ref, guidance_rescale=st.guidance_rescale,
                                                               step=stepper.step(st.ref, 1))
        st.main = stepper.advance(st.main, lat, st.noise_pred)
        if step_ref:
            st.ref = stepper.advance(st.ref, lat_ref, eps_ref)
        if pe is not None:
            ev[2].record()
        if st.use_guidance and float(t) < st.tfd["guidance_start_step"]:                                  # :849
            torch.cuda.nvtx.range_push("guidance")
            st.latents = self._color_guidance(st.latents, st.noise_pred, t, st.tfd)
            torch.cuda.nvtx.range_pop()
        if i == int(st.inject_background * st.n_t) and st.inject_background > 0:                          # :870-872
            st.latents = ops.bg_inject_blend(st.latents.contiguous(), st.latents_ref.contiguous(), st.masks[-1].contiguous())
        if pe is not None:
            ev[3].record()
            pe.update(unet=(ev[0], ev[1]), exchange_blend=(ev[1], ev[2]), color_guidance=(ev[2], ev[3]))
        return st.latents

    def _rich_text_loop(self, ctx, pooled, time_ids, latents, timesteps, guidance_scale, use_guidance,
                        inject_selfattn, inject_background, tfd, callback, callback_steps, guidance_rescale=0.0,
                        generator=None):
        """:772-878."""
        st = self.prepare_rich_text(ctx, pooled, time_ids, latents, timesteps, guidance_scale, use_guidance,
                                    inject_selfattn, inject_background, tfd, guidance_rescale, generator)
        for i, t in enumerate(timesteps):
            self.rich_text_step(st, i)
            if callback is not None and self._calls_back(i, len(timesteps), callback_steps):
                callback(i, t, st.latents)
        for ex in self._exchanges.values():
            ex.check()
        for eng in self._stripe_engines.values():
            eng.arena.check()
        return st.latents
