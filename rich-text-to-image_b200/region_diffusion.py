"""RegionDiffusion (SD1.5) — H100 drop-in for models/region_diffusion.py of the reference.

Public surface kept: `RegionDiffusion(device)`, `produce_attn_maps`, `produce_latents`, `prompt_to_img`,
`predict_x0`, `register_tokenmap_hooks / remove_tokenmap_hooks`, attributes `.unet .vae .tokenizer
.scheduler .masks .selfattn_maps .crossattn_maps .n_maps`. Step semantics follow
models/region_diffusion.py:86-174 (including its differences from the SDXL loop: no scale_model_input,
joint stepping on every step when injecting, `i == int(...)` background flag, and the self-attention
capture that overwrites instead of accumulating, :423), executed as one batched UNet call per step.

`.scheduler` is PLMS (PNDMScheduler) by default and steps on the host; DDIMScheduler, DPMSolverMultistepScheduler,
UniPCMultistepScheduler and DPMSolverSinglestepScheduler (schedulers.py) step inside the fused blend kernels, with
their state kept per trajectory (stepping.py).
"""
import math
from typing import Optional

import numpy as np
import torch

from . import ops, region_parallel, stepping, vae_guidance
from .attention_utils import CrossAttentionLayers, SelfAttentionLayers
from .lora import LoraLoaderMixin
from .schedulers import PNDMScheduler
from .textual_inversion import TextualInversionLoaderMixin
from .unet import CrossKVCache, RegionControl, TokenMapAccumulator, UNet2DConditionModel, UNetConfig
from .vae import AutoencoderKLDecoder, VAEConfig


# the updates that run fused here; any other scheduler steps on the host, on the concatenated batch
_FUSED = ("multistep", "unipc", "singlestep")


class RegionDiffusion(LoraLoaderMixin, TextualInversionLoaderMixin):
    def __init__(self, device="cuda", unet=None, vae=None, text_encoder=None, load_path="runwayml/stable-diffusion-v1-5"):
        self.device = torch.device(device)
        torch.backends.cudnn.benchmark = True   # static shapes: let cuDNN pick its fastest conv algorithm once
        self.num_train_timesteps = 1000
        if unet is None:
            from .loading import load_sd15_components
            unet, vae, text_encoder = load_sd15_components(load_path, self.device)
        self.unet, self.vae, self.text_encoder = unet, vae, text_encoder
        self.tokenizer = getattr(text_encoder, "tokenizer", None)
        self.scheduler = PNDMScheduler()
        self.alphas_cumprod = self.scheduler.alphas_cumprod
        self.masks = []
        self.attention_maps = None
        self.selfattn_maps = None
        self.crossattn_maps = None
        self.n_maps = None
        self._capture = None
        self.last_step_stats = {}

    @classmethod
    def from_synthetic(cls, unet_cfg: Optional[UNetConfig] = None, vae_cfg: Optional[VAEConfig] = None, seed=0,
                       device="cuda", with_vae=True):
        with torch.device(device):
            unet = UNet2DConditionModel(unet_cfg or UNetConfig.sd15())
        unet.finalize(device).init_synthetic(seed)
        vae = AutoencoderKLDecoder(vae_cfg or VAEConfig.sd15()).init_synthetic(seed + 1).finalize(device) if with_vae else None
        return cls(device=device, unet=unet, vae=vae)

    def _lora_components(self):
        return self.unet, (() if self.text_encoder is None else (self.text_encoder.text_encoder,))

    def _textual_inversion_components(self):
        te = self.text_encoder
        return [] if te is None else [(te.tokenizer, te.text_encoder)]

    # ------------------------------------------------------------------ capture API (:397-450)
    def register_tokenmap_hooks(self):
        self._capture = TokenMapAccumulator(CrossAttentionLayers, self_layers=SelfAttentionLayers, start_after=10,
                                            sd_overwrite_bug=True, self_resolutions=None)
        self.selfattn_maps = self._capture.selfattn_maps
        self.crossattn_maps = self._capture.crossattn_maps
        self.n_maps = self._capture.n_maps

    def remove_tokenmap_hooks(self):
        self._capture = None
        self.selfattn_maps = self.crossattn_maps = self.n_maps = None

    def reset_attention_maps(self):
        if self._capture is not None:
            self._capture.selfattn_maps.clear()
            self._capture.crossattn_maps.clear()

    # ------------------------------------------------------------------ text
    def get_text_embeds(self, prompt, negative_prompt):
        if self.text_encoder is None:
            raise RuntimeError("no text encoder loaded: call produce_latents / produce_attn_maps with embeddings")
        return self.text_encoder.encode_pair(prompt, negative_prompt, self.device)

    # ------------------------------------------------------------------ loops
    def predict_x0(self, x_t, eps_t, t):
        """:176-178."""
        alpha = float(self.scheduler.alphas_cumprod[int(t)])
        return ops.predict_x0(x_t.contiguous(), eps_t.contiguous(), alpha), alpha

    def decode_latents(self, latents):
        """:227-236."""
        imgs = self.vae.decode_tensor((1 / 0.18215) * latents.float())
        return (imgs / 2 + 0.5).clamp(0, 1)

    def _color_guidance(self, latents, noise_pred, t, tfd):
        """:151-168."""
        x0, alpha = self.predict_x0(latents, noise_pred, t)
        # the reference pairs maps and targets with zip() (sdxl.py:857 / region_diffusion.py:159): sample.py hands over
        # R colour maps + the background map but only R target colours, and the background map is dropped
        n_col = min(len(tfd["color_obj_atten"]), len(tfd["target_RGB"]))
        masks = torch.stack([m[0, 0].to(self.device, torch.float32) for m in tfd["color_obj_atten"][:n_col]]).contiguous()
        tgt = torch.stack([r.reshape(3).to(self.device, torch.float32) for r in tfd["target_RGB"][:n_col]]).contiguous()

        def grad_image(img):
            loss, g = ops.color_loss_fwd_bwd(img[0].contiguous(), masks, tgt)
            self.last_step_stats["color_loss"] = loss
            return g[None]

        grad_lat = vae_guidance.image_and_latent_grad(self.vae, (1 / 0.18215) * x0.float(), grad_image) \
            * ((1 / 0.18215) / math.sqrt(alpha))
        atten_all = tfd["color_obj_atten_all"].to(self.device, torch.float32).expand_as(grad_lat).contiguous()
        return ops.latent_guidance_update(latents.contiguous(), grad_lat.contiguous(), atten_all,
                                          float(tfd["color_guidance_weight"]))

    @torch.no_grad()
    def produce_latents(self, text_embeddings, height=512, width=512, num_inference_steps=50, guidance_scale=7.5,
                        latents=None, use_guidance=False, text_format_dict={}, inject_selfattn=0, inject_background=0):
        """:86-174. text_embeddings = [uncond, region_1..region_{N-1}, base].
        With DPMSolverSinglestepScheduler each trajectory keeps its x0 prediction and the latents that entered its
        current two-step block; the second step of a block restarts from those latents, so colour guidance and
        background injection applied after a first step reach the second step only through its prediction, as in the
        reference with DPMSolverSinglestepScheduler assigned to its scheduler."""
        dev = self.device
        tfd = text_format_dict or {}
        if latents is None:
            latents = torch.randn((1, self.unet.in_channels, height // 8, width // 8), device=dev)
        latents = latents.to(dev, torch.float16)
        ctx = text_embeddings.to(dev, torch.float16)
        N = len(self.masks)
        assert ctx.shape[0] - 1 == N
        inject = inject_selfattn > 0 or inject_background > 0
        latents_ref = latents.clone() if inject else None
        self.scheduler.set_timesteps(num_inference_steps)
        timesteps = self.scheduler.timesteps
        masks = torch.stack([m.to(dev, torch.float32).reshape(-1) for m in self.masks]).contiguous()
        ones = torch.ones(1, latents[0].numel(), dtype=torch.float32, device=dev)
        passes = [dict(kind="A", ctx=0, ref=False), dict(kind="B", ctx=N, ref=False)]
        if inject:
            passes += [dict(kind="C", ctx=0, ref=True), dict(kind="D", ctx=N, ref=True)]
        passes += [dict(kind="E", ctx=j + 1, ref=False, region=j) for j in range(N - 1)]
        kind = {p["kind"] + str(p.get("region", "")): k for k, p in enumerate(passes)}
        plan = region_parallel.RegionParallelPlan(passes, inject)
        word_pos, font_size = tfd.get("word_pos"), tfd.get("font_size")
        if word_pos is not None and font_size is not None:
            word_pos = word_pos.to(dev, torch.int32).contiguous()
            font_size = font_size.to(dev, torch.float32).contiguous()
        else:
            word_pos = font_size = None
        kv_caches = {}
        n_t = len(timesteps)
        stepper = stepping.stepper(self.scheduler, latents.shape, dev, kinds=_FUSED)
        if stepper is not None:   # both trajectories are stepped on every step
            main, ref = stepper.state(), (stepper.state() if inject else None)
        for i, t in enumerate(timesteps):
            feat_inject_step = bool(int(t) > (1 - inject_selfattn) * 1000)                                   # :104
            background_inject_step = (i == int(inject_background * n_t)) and inject_background > 0           # :105
            local = plan.local_passes(feat_inject_step)
            kvc = kv_caches.setdefault(tuple(local), CrossKVCache())
            rows = [passes[p]["ctx"] for p in local]
            x = torch.cat([(latents_ref if passes[p]["ref"] else latents) for p in local])
            ctrl = RegionControl(kv_cache=kvc)
            if feat_inject_step and inject:
                src = plan.injection_sources(local)
                ctrl.qk_src = src
                ctrl.feature_src = src
            if word_pos is not None:
                ctrl.word_pos, ctrl.font_size = word_pos, font_size
                ctrl.fs_batch_mask = sum(1 << k for k, p in enumerate(local) if passes[p]["kind"] == "B")
            eps_local = self.unet(x, t, ctx[rows], None, ctrl)["sample"]
            eps = plan.gather(eps_local, local, feat_inject_step)
            regions = [eps[kind[f"E{j}"]:kind[f"E{j}"] + 1].contiguous() for j in range(N - 1)]
            regions.append(eps[kind["B"]:kind["B"] + 1].contiguous())
            if stepper is not None:
                stepper.begin(i, t, 2 if inject else 1)
                lat = latents.contiguous()
                noise_pred, latents = ops.region_blend_cfg(eps[kind["A"]:kind["A"] + 1].contiguous(), regions, masks,
                                                           guidance_scale, latents=lat, step=stepper.step(main))
                main = stepper.advance(main, lat, noise_pred)
                if inject:
                    lat_ref = latents_ref.contiguous()
                    eps_ref, latents_ref = ops.region_blend_cfg(eps[kind["C"]:kind["C"] + 1].contiguous(),
                                                                [eps[kind["D"]:kind["D"] + 1].contiguous()], ones,
                                                                guidance_scale, latents=lat_ref,
                                                                step=stepper.step(ref, 1))
                    ref = stepper.advance(ref, lat_ref, eps_ref)
            else:
                noise_pred = ops.region_blend_cfg(eps[kind["A"]:kind["A"] + 1].contiguous(), regions, masks, guidance_scale)  # :119-132
                if inject:                                                                                  # :134-143
                    ref = ops.region_blend_cfg(eps[kind["C"]:kind["C"] + 1].contiguous(),
                                               [eps[kind["D"]:kind["D"] + 1].contiguous()], ones, guidance_scale)
                    both = self.scheduler.step(torch.cat([noise_pred, ref]), t, torch.cat([latents, latents_ref]))["prev_sample"]
                    latents, latents_ref = [c.to(torch.float16) for c in torch.chunk(both, 2, dim=0)]
                else:
                    latents = self.scheduler.step(noise_pred, t, latents)["prev_sample"].to(torch.float16)
            if use_guidance and int(t) < tfd["guidance_start_step"]:                                        # :151
                latents = self._color_guidance(latents, noise_pred, t, tfd)
            if background_inject_step:                                                                       # :171-173
                latents = ops.bg_inject_blend(latents.contiguous(), latents_ref.contiguous(), masks[-1].contiguous())
        return latents

    @torch.no_grad()
    def produce_attn_maps(self, prompts, negative_prompts="", height=512, width=512, num_inference_steps=50,
                          guidance_scale=7.5, latents=None, text_embeddings=None, decode=True):
        """:180-225 — plain CFG loop (batch [uncond, cond]); with capture armed, fills the token maps."""
        dev = self.device
        if text_embeddings is None:
            prompts = [prompts] if isinstance(prompts, str) else prompts
            negative_prompts = [negative_prompts] if isinstance(negative_prompts, str) else negative_prompts
            text_embeddings = self.get_text_embeds(prompts, negative_prompts)
        ctx = text_embeddings.to(dev, torch.float16)
        if latents is None:
            latents = torch.randn((ctx.shape[0] // 2, self.unet.in_channels, height // 8, width // 8), device=dev)
        latents = latents.to(dev, torch.float16)
        self.scheduler.set_timesteps(num_inference_steps)
        kv = CrossKVCache()
        ones = torch.ones(1, latents[0].numel(), dtype=torch.float32, device=dev)
        stepper = stepping.stepper(self.scheduler, latents.shape, dev, kinds=_FUSED)
        state = stepper.state() if stepper is not None else None
        for i, t in enumerate(self.scheduler.timesteps):
            x = latents.expand(2, -1, -1, -1)
            ctrl = RegionControl(capture=self._capture, capture_row=1, kv_cache=kv)
            eps = self.unet(x, t, ctx, None, ctrl)["sample"]
            if stepper is not None:
                stepper.begin(i, t, 1)
                lat = latents.contiguous()
                e16, latents = ops.region_blend_cfg(eps[0:1].contiguous(), [eps[1:2].contiguous()], ones, guidance_scale,
                                                    latents=lat, step=stepper.step(state))
                state = stepper.advance(state, lat, e16)
                continue
            noise_pred = ops.region_blend_cfg(eps[0:1].contiguous(), [eps[1:2].contiguous()], ones, guidance_scale)
            latents = self.scheduler.step(noise_pred, t, latents)["prev_sample"].to(torch.float16)
        self._last_latents = latents
        if not decode or self.vae is None:
            return latents
        imgs = self.decode_latents(latents).detach().cpu().permute(0, 2, 3, 1).numpy()
        return (imgs * 255).round().astype("uint8")

    @torch.no_grad()
    def prompt_to_img(self, prompts, negative_prompts="", height=512, width=512, num_inference_steps=50,
                      guidance_scale=7.5, latents=None, text_format_dict={}, use_guidance=False, inject_selfattn=0,
                      inject_background=0, text_embeddings=None):
        """:248-274."""
        if text_embeddings is None:
            prompts = [prompts] if isinstance(prompts, str) else prompts
            negative_prompts = [negative_prompts] if isinstance(negative_prompts, str) else negative_prompts
            text_embeddings = self.get_text_embeds(prompts, negative_prompts)
        latents = self.produce_latents(text_embeddings, height=height, width=width, latents=latents,
                                       num_inference_steps=num_inference_steps, guidance_scale=guidance_scale,
                                       use_guidance=use_guidance, text_format_dict=text_format_dict,
                                       inject_selfattn=inject_selfattn, inject_background=inject_background)
        imgs = self.decode_latents(latents).detach().cpu().permute(0, 2, 3, 1).numpy()
        return (imgs * 255).round().astype("uint8")
