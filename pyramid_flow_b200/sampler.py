"""Host-side mirror of the reference sampler loop, so the hot path can be driven end-to-end without the reference tree.

Mirrors `PyramidDiTForVideoGeneration.generate` / `generate_i2v` (P:791-1003) / `generate_one_unit` / `get_pyramid_latent` / `sample_block_noise` /
`decode_latent` (pyramid_dit/pyramid_dit_for_video_gen_pipeline.py:1006-1219, 706-788, 555-570, 697-703, 1221-1243) from
the point where text embeddings exist (the prompt encoders run on the library too, as
`pyramid_flow_b200.text_encoder.B200FluxTextEncoder` / `B200SD3TextEncoder`).  In a reference checkout the
pipeline itself stays the call surface (INTEGRATION.md); this mirror is what tests and bench.py drive on the GPU, and
it is pinned against the unmodified reference loop by tests/golden/sampler_small.pt (oracle/pin/make_golden.py).

Only latent-space glue runs in torch here (bilinear/nearest resampling of `[1,16,T,h,w]` latents, CFG combine, Euler
update — the reference's own host-side code); the DiT forward and the VAE decode are libpf_b200 kernels.
"""
from __future__ import annotations

import math
from typing import Callable, List, Optional, Sequence

import torch
import torch.nn.functional as F


def _resize_frames(x: torch.Tensor, size, mode: str) -> torch.Tensor:
    """'b c t h w -> (b t) c h w' -> interpolate -> back (P:561-565, P:731-733, P:1112-1116)."""
    b, c, t, h, w = x.shape
    y = x.permute(0, 2, 1, 3, 4).reshape(b * t, c, h, w)
    y = F.interpolate(y, size=size, mode=mode)
    return y.reshape(b, t, c, size[0], size[1]).permute(0, 2, 1, 3, 4)


def block_noise(bs: int, ch: int, temp: int, height: int, width: int, gamma: float,
                generator: Optional[torch.Generator] = None) -> torch.Tensor:
    """sample_block_noise (P:697-703): every 2x2 block ~ N(0, (1+g) I - g 11^T); vectorised (one Cholesky factor) instead
    of the reference's python loop of `block_number` MultivariateNormal.sample() calls.  Same distribution, different RNG
    consumption — parity tests inject the noise instead."""
    cov = torch.eye(4) * (1 + gamma) - torch.ones(4, 4) * gamma
    l = torch.linalg.cholesky(cov)
    n = bs * ch * temp * (height // 2) * (width // 2)
    z = torch.randn(n, 4, generator=generator) @ l.T
    z = z.reshape(bs, ch, temp, height // 2, width // 2, 2, 2).permute(0, 1, 2, 3, 5, 4, 6)
    return z.reshape(bs, ch, temp, height, width)


class B200PyramidSampler:
    def __init__(self, dit, scheduler, vae=None, stages: Sequence[int] = (1, 2, 4), frame_per_unit: int = 1,
                 model_name: str = "pyramid_flux", downsample: int = 8,
                 block_noise_fn: Optional[Callable[..., torch.Tensor]] = None, fused_step: bool = False,
                 gpu_stage_hop: bool = False):
        self.dit, self.scheduler, self.vae = dit, scheduler, vae
        self.stages = list(stages)
        self.frame_per_unit = frame_per_unit
        self.downsample = downsample
        self.model_name = model_name
        self.block_noise_fn = block_noise_fn
        # fused_step: CFG combine + Euler update in ONE kernel on fp32 velocities (pf_cfg_euler_step, reference P:771-776 +
        # S:278-286); the result is rounded to the latent dtype once.  Opt-in: it rounds less than the reference's bf16 chain
        # (bf16 CFG combine, bf16 dsigma*v), so outputs differ from the reference at bf16 resolution.
        self.fused_step = fused_step
        # gpu_stage_hop: the stage transition (nearest x2 up-sample, block noise, renoise; P:729-743) as ONE kernel with the
        # normals drawn on the device (pf_stage_hop) instead of CPU randn + Cholesky matmul + H2D copy + 3 torch ops.  Opt-in:
        # same distribution, different RNG stream than the reference (parity tests inject the noise instead).
        self.gpu_stage_hop = gpu_stage_hop
        # latent normalisation constants (P:160-176)
        if model_name == "pyramid_flux":
            self.vae_shift_factor, self.vae_scale_factor = -0.04, 1 / 1.8726
        else:
            self.vae_shift_factor, self.vae_scale_factor = 0.1490, 1 / 1.8415
        self.vae_video_shift_factor, self.vae_video_scale_factor = -0.2343, 1 / 3.0986
        self.dit_calls = 0

    # ------------------------------------------------------------------------------------------------------------------
    def get_pyramid_latent(self, x: torch.Tensor, stage_num: int) -> List[torch.Tensor]:
        out = [x]
        h, w = x.shape[-2], x.shape[-1]
        for _ in range(stage_num):
            h //= 2
            w //= 2
            x = _resize_frames(x, (h, w), "bilinear")
            out.append(x)
        return list(reversed(out))

    @torch.no_grad()
    def generate_one_unit(self, latents, past_conditions, prompt_embeds, prompt_attention_mask, pooled_prompt_embeds,
                          num_inference_steps, height, width, temp, device, dtype, is_first_frame: bool,
                          guidance_scale: float, video_guidance_scale: float, do_cfg: bool = True):
        """P:706-788."""
        inter = []
        for i_s in range(len(self.stages)):
            self.scheduler.set_timesteps(num_inference_steps[i_s], i_s, device=device)
            timesteps = self.scheduler.timesteps
            if i_s > 0:
                height *= 2
                width *= 2
                ori_sigma = 1 - self.scheduler.ori_start_sigmas[i_s]
                gamma = self.scheduler.config.gamma
                alpha = 1 / (math.sqrt(1 + (1 / gamma)) * (1 - ori_sigma) + ori_sigma)
                beta = alpha * (1 - ori_sigma) / math.sqrt(gamma)
                if self.gpu_stage_hop and self.block_noise_fn is None and latents.is_cuda:
                    from . import ops
                    bs, ch, temp = latents.shape[:3]
                    z = torch.randn(bs, ch, temp, height, width, device=latents.device, dtype=torch.float32,
                                    generator=getattr(self, "device_generator", None))
                    latents = ops.stage_hop(latents.contiguous(), z, alpha, beta, gamma)
                else:
                    latents = _resize_frames(latents, (height, width), "nearest")
                    bs, ch, temp, height, width = latents.shape
                    fn = self.block_noise_fn or (lambda *a: block_noise(*a, gamma))
                    noise = fn(bs, ch, temp, height, width).to(device=device, dtype=dtype)
                    latents = alpha * latents + beta * noise
            for t in timesteps:
                x_in = torch.cat([latents] * 2) if do_cfg else latents
                timestep = t.expand(x_in.shape[0]).to(x_in.dtype)          # rounded to the latent dtype (bf16), P:750
                clips = past_conditions[i_s] + [x_in]
                v = self.dit(sample=[clips], timestep_ratio=timestep, encoder_hidden_states=prompt_embeds,
                             encoder_attention_mask=prompt_attention_mask, pooled_projections=pooled_prompt_embeds)[0]
                self.dit_calls += 1
                if self.fused_step and do_cfg and v.dtype == torch.float32:
                    from . import ops
                    g = guidance_scale if is_first_frame else video_guidance_scale
                    x32 = latents.float().contiguous()
                    ops.cfg_euler_step(v.contiguous(), float(g), self.scheduler.delta_sigma(), x32, x32)
                    self.scheduler.advance()
                    latents = x32.to(latents.dtype) if latents.dtype != torch.float32 else x32
                    continue
                if do_cfg:
                    vu, vc = v.chunk(2)
                    g = guidance_scale if is_first_frame else video_guidance_scale
                    v = vu + g * (vc - vu)
                latents = self.scheduler.step(model_output=v, timestep=timestep, sample=latents).prev_sample
            inter.append(latents)
        return inter

    def _past_conditions(self, generated: List[torch.Tensor], unit: int, do_cfg: bool = True) -> List[List[torch.Tensor]]:
        """Compressed history per stage (P:1159-1182 == P:923-952): the last clean unit at the stage's own resolution, older
        units at successively coarser stages, everything older than that at the coarsest; oldest first."""
        n_stage = len(self.stages)
        clean = self.get_pyramid_latent(torch.cat(generated, dim=2), n_stage - 1)
        fpu = self.frame_per_unit
        dup = (lambda x: torch.cat([x] * 2)) if do_cfg else (lambda x: x)
        past = []
        for i_s in range(n_stage):
            stage_input = [dup(clean[i_s][:, :, -fpu:])]
            cur_stage, ptx = i_s, 1
            while ptx < unit:
                cur_stage = max(cur_stage - 1, 0)
                if cur_stage == 0:
                    break
                ptx += 1
                stage_input.append(dup(clean[cur_stage][:, :, -(ptx * fpu): -((ptx - 1) * fpu)]))
            if cur_stage == 0 and ptx < unit:
                stage_input.append(dup(clean[0][:, :, :-(ptx * fpu)]))
            past.append(list(reversed(stage_input)))
        return past

    @torch.no_grad()
    def generate_i2v(self, input_image_tensor: Optional[torch.Tensor], prompt_embeds, prompt_attention_mask,
                     pooled_prompt_embeds, height: int, width: int, temp: int = 1, num_inference_steps=(10, 10, 10),
                     guidance_scale: float = 7.0, video_guidance_scale: float = 4.0,
                     generator: Optional[torch.Generator] = None, output_type: str = "latent", save_memory: bool = True,
                     image_latent: Optional[torch.Tensor] = None):
        """P:791-1003 after text encoding and the PIL -> tensor transform: `input_image_tensor` is `[1, 3, 1, H, W]` in
        [-1, 1] (ToTensor + Normalize(0.5, 0.5), P:907-910).  The image latent is `vae.encode(...).latent_dist.sample()`
        shifted/scaled with the IMAGE factors (P:911); `image_latent` injects it instead (tests without a VAE).  The first
        unit is the image itself; every later unit runs with `is_first_frame=False` and ONE step list (P:954-968)."""
        device, dtype = prompt_embeds.device, prompt_embeds.dtype
        n_stage = len(self.stages)
        num_inference_steps = [num_inference_steps] * n_stage if isinstance(num_inference_steps, int) else list(num_inference_steps)
        c_lat = (self.dit.config.in_channels // 4) if self.model_name == "pyramid_flux" else self.dit.config.in_channels
        shape = (1, c_lat, int(temp), int(height) // self.downsample, int(width) // self.downsample)
        latents = torch.randn(shape, generator=generator, dtype=dtype).to(device)      # prepare_latents, P:881-890
        temp, h, w = latents.shape[-3:]
        for _ in range(n_stage - 1):                                                 # P:894-899
            h //= 2
            w //= 2
            latents = _resize_frames(latents, (h, w), "bilinear") * 2
        num_units = temp // self.frame_per_unit                                      # P:903 (the image is unit 0)
        if image_latent is None:
            x = input_image_tensor.to(device=self.vae.device, dtype=self.vae.dtype)
            image_latent = self.vae.encode(x).latent_dist.sample()
        image_latent = ((image_latent - self.vae_shift_factor) * self.vae_scale_factor).to(device=device, dtype=dtype)
        generated = [image_latent]
        fpu = self.frame_per_unit
        for unit in range(1, num_units):
            past = self._past_conditions(generated, unit)
            inter = self.generate_one_unit(latents[:, :, (unit - 1) * fpu: unit * fpu], past, prompt_embeds,
                                           prompt_attention_mask, pooled_prompt_embeds, num_inference_steps, h, w, fpu,
                                           device, dtype, False, guidance_scale, video_guidance_scale)
            generated.append(inter[-1])
        out = torch.cat(generated, dim=2)
        if output_type == "latent":
            return out
        return self.decode_latent(out, save_memory=save_memory)

    @torch.no_grad()
    def generate(self, prompt_embeds, prompt_attention_mask, pooled_prompt_embeds, height: int, width: int, temp: int = 1,
                 num_inference_steps=(20, 20, 20), video_num_inference_steps=(10, 10, 10), guidance_scale: float = 7.0,
                 video_guidance_scale: float = 5.0, generator: Optional[torch.Generator] = None,
                 output_type: str = "latent", save_memory: bool = True, latents: Optional[torch.Tensor] = None):
        """P:1006-1219 after text encoding: `prompt_embeds` etc. are already the CFG batch [negative ; positive]."""
        device, dtype = prompt_embeds.device, prompt_embeds.dtype
        n_stage = len(self.stages)
        num_inference_steps = [num_inference_steps] * n_stage if isinstance(num_inference_steps, int) else list(num_inference_steps)
        video_num_inference_steps = [video_num_inference_steps] * n_stage if isinstance(video_num_inference_steps, int) else list(video_num_inference_steps)
        assert (temp - 1) % self.frame_per_unit == 0
        c_lat = (self.dit.config.in_channels // 4) if self.model_name == "pyramid_flux" else self.dit.config.in_channels
        if latents is None:   # prepare_latents: CPU generator then move (randn_tensor semantics, P:676-695)
            shape = (1, c_lat, int(temp), int(height) // self.downsample, int(width) // self.downsample)
            latents = torch.randn(shape, generator=generator, dtype=dtype).to(device)
        temp, h, w = latents.shape[-3:]
        for _ in range(n_stage - 1):                              # P:1112-1116: start noise at the coarsest stage
            h //= 2
            w //= 2
            latents = _resize_frames(latents, (h, w), "bilinear") * 2
        num_units = 1 + (temp - 1) // self.frame_per_unit
        generated = []
        for unit in range(num_units):
            if unit == 0:
                past = [[] for _ in range(n_stage)]
                inter = self.generate_one_unit(latents[:, :, :1], past, prompt_embeds, prompt_attention_mask,
                                               pooled_prompt_embeds, num_inference_steps, h, w, 1, device, dtype, True,
                                               guidance_scale, video_guidance_scale)
            else:
                fpu = self.frame_per_unit
                past = self._past_conditions(generated, unit)
                sl = slice(1 + (unit - 1) * fpu, 1 + unit * fpu)
                inter = self.generate_one_unit(latents[:, :, sl], past, prompt_embeds, prompt_attention_mask,
                                               pooled_prompt_embeds, video_num_inference_steps, h, w, fpu, device, dtype,
                                               False, guidance_scale, video_guidance_scale)
            generated.append(inter[-1])
        out = torch.cat(generated, dim=2)
        if output_type == "latent":
            return out
        return self.decode_latent(out, save_memory=save_memory)

    @torch.no_grad()
    def decode_latent(self, latents: torch.Tensor, save_memory: bool = True) -> torch.Tensor:
        """P:1221-1243 up to the uint8 frames: returns uint8 `[(B T), H, W, C]` on the device."""
        if hasattr(self.vae, "decode_latent_u8"):
            # one pass: un-normalisation fused into the latent pack, uint8 conversion into conv_out's epilogue
            return self.vae.decode_latent_u8(latents, self.vae_scale_factor, self.vae_shift_factor,
                                             self.vae_video_scale_factor, self.vae_video_shift_factor,
                                             window_size=1 if save_memory else 2,
                                             tile_sample_min_size=256 if save_memory else 512)
        latents = latents.clone()
        if latents.shape[2] == 1:
            latents = (latents / self.vae_scale_factor) + self.vae_shift_factor
        else:
            latents[:, :, :1] = (latents[:, :, :1] / self.vae_scale_factor) + self.vae_shift_factor
            latents[:, :, 1:] = (latents[:, :, 1:] / self.vae_video_scale_factor) + self.vae_video_shift_factor
        if save_memory:
            image = self.vae.decode(latents, temporal_chunk=True, window_size=1, tile_sample_min_size=256).sample
        else:
            image = self.vae.decode(latents, temporal_chunk=True, window_size=2, tile_sample_min_size=512).sample
        image = image.float().mul(127.5).add(127.5).clamp(0, 255).byte()
        b, c, t, h, w = image.shape
        return image.permute(0, 2, 3, 4, 1).reshape(b * t, h, w, c)
