"""ORACLE (test infrastructure only) for image-to-image: CPU restatements of the pieces of [3P] diffusers==0.30.0
(requirements.txt:25; not vendored) that `StableDiffusionXLImg2ImgPipeline` adds on top of the text-to-image path.
**Parity unpinned**, like the other [3P] restatements under oracle/: diffusers is not installable here and the
reference holds no golden vector for these; the structure follows the public SDXL `vae/config.json` and the diffusers
0.30.0 sources as published.

* `VAEEncoderRef`: `AutoencoderKL.encoder` + `quant_conv` (keys `encoder.*`, `quant_conv.*`), fp32;
* `posterior_sample_ref`: `DiagonalGaussianDistribution.sample`;
* `tiled_encode_ref`: `AutoencoderKL.tiled_encode` (moments are blended, before sampling);
* `img2img_timesteps`: `StableDiffusionXLImg2ImgPipeline.get_timesteps` (denoising_start = None);
* `add_noise_ref`: `EulerDiscreteScheduler.add_noise` at the pipeline's begin index;
* `prepare_img2img_latents`: `prepare_latents` with fp16 latents -- its rounding points and RNG order:
    per generator, the posterior eps is drawn before the noise; with one generator eps is drawn for the IMAGE batch and
    the sampled latents are then tiled to the prompt batch with torch.cat (image order [0, 1, 0, 1, ...]);
* `img2img_denoise_loop`: the loop of oracle.scheduler_ref.denoise_loop over timesteps[t_start:] (step counter and
  sigma index start at t_start; gating fractions and callback indices count from the start of the truncated list).
"""
from __future__ import annotations

from typing import Callable, List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.scheduler_ref import euler_tables, rescale_noise_cfg
from oracle.vae_ref import MidRef, ResnetRef


class DownsampleRef(nn.Module):
    """Downsample2D(use_conv=True, padding=0): pad one zero row / column at the bottom / right, conv stride 2."""

    def __init__(self, ch):
        super().__init__()
        self.conv = nn.Conv2d(ch, ch, 3, stride=2, padding=0)

    def forward(self, x):
        return self.conv(F.pad(x, (0, 1, 0, 1), mode="constant", value=0))


class DownBlockRef(nn.Module):
    def __init__(self, cin, cout, n_res, groups, add_down):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetRef(cin if j == 0 else cout, cout, groups) for j in range(n_res)])
        if add_down:
            self.downsamplers = nn.ModuleList([DownsampleRef(cout)])
        self.has_down = add_down

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        return self.downsamplers[0](x) if self.has_down else x


class EncoderRef(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        ch = cfg.block_out_channels
        g = cfg.norm_num_groups
        self.conv_in = nn.Conv2d(cfg.out_channels, ch[0], 3, padding=1)
        downs, prev = [], ch[0]
        for i, c in enumerate(ch):
            downs.append(DownBlockRef(prev, c, cfg.layers_per_block, g, add_down=i < len(ch) - 1))
            prev = c
        self.down_blocks = nn.ModuleList(downs)
        self.mid_block = MidRef(ch[-1], g)
        self.conv_norm_out = nn.GroupNorm(g, ch[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(ch[-1], 2 * cfg.latent_channels, 3, padding=1)      # double_z

    def forward(self, x):
        x = self.conv_in(x)
        for b in self.down_blocks:
            x = b(x)
        x = self.mid_block(x)
        return self.conv_out(F.silu(self.conv_norm_out(x)))


class VAEEncoderRef(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.config = cfg
        self.encoder = EncoderRef(cfg)
        self.quant_conv = nn.Conv2d(2 * cfg.latent_channels, 2 * cfg.latent_channels, 1)

    def encode(self, image):
        """AutoencoderKL.encode(image).latent_dist.parameters: the moments [B, 2L, H/8, W/8]."""
        return self.quant_conv(self.encoder(image))


def posterior_sample_ref(moments: torch.Tensor, eps: torch.Tensor) -> torch.Tensor:
    """DiagonalGaussianDistribution(moments).sample() with the drawn eps; arithmetic in the moments' dtype."""
    mean, logvar = torch.chunk(moments, 2, dim=1)
    logvar = torch.clamp(logvar, -30.0, 20.0)
    std = torch.exp(0.5 * logvar)
    return mean + std * eps


def tiled_encode_ref(vae: VAEEncoderRef, x: torch.Tensor) -> torch.Tensor:
    """AutoencoderKL.tiled_encode: tiles of sample_size pixels every 3/4 tile, each through encoder + quant_conv,
    moments blended with the upper and the left neighbour over blend_extent latents and cropped to row_limit."""
    cfg = vae.config
    tile_sample = cfg.sample_size
    tl = cfg.tile_latent_min_size
    overlap_size = int(tile_sample * (1 - cfg.tile_overlap_factor))
    blend_extent = int(tl * cfg.tile_overlap_factor)
    row_limit = tl - blend_extent
    rows = []
    for i in range(0, x.shape[2], overlap_size):
        row = []
        for j in range(0, x.shape[3], overlap_size):
            row.append(vae.encode(x[:, :, i:i + tile_sample, j:j + tile_sample]))
        rows.append(row)
    result_rows = []
    for i, row in enumerate(rows):
        result_row = []
        for j, tile in enumerate(row):
            if i > 0:
                a, b = rows[i - 1][j], tile
                ext = min(a.shape[2], b.shape[2], blend_extent)
                for y in range(ext):
                    b[:, :, y, :] = a[:, :, -ext + y, :] * (1 - y / ext) + b[:, :, y, :] * (y / ext)
            if j > 0:
                a, b = row[j - 1], tile
                ext = min(a.shape[3], b.shape[3], blend_extent)
                for xx in range(ext):
                    b[:, :, :, xx] = a[:, :, :, -ext + xx] * (1 - xx / ext) + b[:, :, :, xx] * (xx / ext)
            result_row.append(tile[:, :, :row_limit, :row_limit])
        result_rows.append(torch.cat(result_row, dim=3))
    return torch.cat(result_rows, dim=2)


def img2img_timesteps(num_inference_steps: int, strength: float):
    """get_timesteps: -> (t_start, timesteps[t_start:]) of the leading-spacing Euler schedule."""
    timesteps, _, _ = euler_tables(num_inference_steps)
    init_timestep = min(int(num_inference_steps * strength), num_inference_steps)
    t_start = max(num_inference_steps - init_timestep, 0)
    return t_start, timesteps[t_start:]


def add_noise_ref(latents: torch.Tensor, noise: torch.Tensor, sigma: float) -> torch.Tensor:
    """EulerDiscreteScheduler.add_noise before the first step: the sigma table is cast to the latents' dtype."""
    s = torch.tensor(sigma, dtype=torch.float32, device=latents.device).to(latents.dtype)
    return latents + noise * s


def _randn(shape, generator, dtype):
    """diffusers randn_tensor on the generator's device, returned on the CPU."""
    if isinstance(generator, list):
        parts = [torch.randn((1,) + tuple(shape[1:]), generator=g, device=g.device, dtype=dtype) for g in generator]
        return torch.cat([p.cpu() for p in parts], dim=0)
    dev = generator.device if generator is not None else "cpu"
    return torch.randn(tuple(shape), generator=generator, device=dev, dtype=dtype).cpu()


def prepare_img2img_latents(encode: Callable, image: torch.Tensor, batch_size: int, generator, sigma: float,
                            scaling_factor: float, latent_channels: int = 4, force_upcast: bool = True,
                            dtype=torch.float16) -> torch.Tensor:
    """StableDiffusionXLImg2ImgPipeline.prepare_latents (image not yet latents, add_noise=True) with `dtype` latents.
    `encode(image) -> moments` (e.g. VAEEncoderRef.encode); `batch_size` already includes num_images_per_prompt."""
    image = image.to(dtype)
    pdt = torch.float32 if force_upcast else dtype            # the VAE (and so its posterior) is upcast to fp32
    image = image.to(pdt)
    if isinstance(generator, list):
        if len(generator) != batch_size:
            raise ValueError(f"got {len(generator)} generators for a batch of {batch_size}")
        if image.shape[0] < batch_size:
            if batch_size % image.shape[0]:
                raise ValueError("cannot duplicate the image batch to the prompt batch")
            image = torch.cat([image] * (batch_size // image.shape[0]), dim=0)
        lat = []
        for i in range(batch_size):
            mom = encode(image[i:i + 1]).to(pdt)
            eps = _randn((1, latent_channels) + tuple(mom.shape[2:]), generator[i], pdt).to(mom.device)
            lat.append(posterior_sample_ref(mom, eps))
        init = torch.cat(lat, dim=0)
    else:
        mom = encode(image).to(pdt)
        eps = _randn((mom.shape[0], latent_channels) + tuple(mom.shape[2:]), generator, pdt).to(mom.device)
        init = posterior_sample_ref(mom, eps)
    init = init.to(dtype)
    init = scaling_factor * init
    if batch_size > init.shape[0]:
        if batch_size % init.shape[0]:
            raise ValueError("cannot duplicate the image batch to the prompt batch")
        init = torch.cat([init] * (batch_size // init.shape[0]), dim=0)
    noise = _randn(init.shape, generator, dtype).to(init.device)
    return add_noise_ref(init, noise, sigma)


@torch.no_grad()
def img2img_denoise_loop(unet_fn: Callable, latents: torch.Tensor, prompt_embeds, neg_prompt_embeds, pooled, neg_pooled,
                         time_ids, num_inference_steps: int, strength: float, guidance_scale: float = 5.0,
                         set_scale: Optional[Callable[[float], None]] = None, conditioning_scale: float = 1.0,
                         control_guidance_start: float = 0.0, control_guidance_end: float = 1.0,
                         guidance_rescale: float = 0.0, denoising_end: Optional[float] = None,
                         callback: Optional[Callable] = None, callback_steps: int = 1,
                         trace: Optional[List[torch.Tensor]] = None) -> torch.Tensor:
    """The denoise loop over the truncated list: step i of the loop uses sigmas[t_start + i] (the scheduler's begin
    index); denoising_end keeps the leading entries of the TRUNCATED list; gating uses i / len(truncated list)."""
    timesteps, sigmas, _ = euler_tables(num_inference_steps)
    t_start, ts = img2img_timesteps(num_inference_steps, strength)
    if denoising_end is not None and isinstance(denoising_end, float) and 0 < denoising_end < 1:
        cutoff = int(round(1000 - denoising_end * 1000))
        ts = ts[:sum(1 for t in ts if t >= cutoff)]
    n_loop = len(ts)
    cfg = guidance_scale > 1.0
    if cfg:
        ehs = torch.cat([neg_prompt_embeds, prompt_embeds], dim=0)
        text_embeds = torch.cat([neg_pooled, pooled], dim=0)
        tids = torch.cat([time_ids, time_ids], dim=0)
    else:
        ehs, text_embeds, tids = prompt_embeds, pooled, time_ids
    for i in range(n_loop):
        k = t_start + i
        if set_scale is not None:
            off = (i / n_loop < control_guidance_start) or ((i + 1) / n_loop > control_guidance_end)
            set_scale(0.0 if off else conditioning_scale)
        sigma, sigma_next = float(sigmas[k]), float(sigmas[k + 1])
        x2 = torch.cat([latents] * 2) if cfg else latents
        x2 = (x2 / ((sigma ** 2 + 1) ** 0.5)).to(latents.dtype)
        noise = unet_fn(x2, float(timesteps[k]), ehs, text_embeds, tids)
        if cfg:
            u, c = noise.chunk(2)
            eps = u + guidance_scale * (c - u)
            if guidance_rescale > 0.0:
                eps = rescale_noise_cfg(eps, c, guidance_rescale)
        else:
            eps = noise
        x = latents.float()
        x0 = x - (sigma * eps.float()).to(eps.dtype).float()
        latents = (x + (x - x0) / sigma * (sigma_next - sigma)).to(eps.dtype)
        if trace is not None:
            trace.append(latents.clone())
        if callback is not None and i % callback_steps == 0:
            callback(i, float(ts[i]), latents)
    return latents


def posterior_noise_ref(moments_nhwc: torch.Tensor, eps: torch.Tensor, noise: torch.Tensor, channels: int,
                        scaling_factor: float, sigma: float) -> torch.Tensor:
    """The rounding points of ih_vae_posterior_noise_f16 (= prepare_img2img_latents after the encoder, fp16 latents)
    as torch ops on any device: moments NHWC [Bm, h, w, >= 2C]; image b uses moments[b % Bm] and eps[b % Be]."""
    C = channels
    B, Bm, Be = noise.shape[0], moments_nhwc.shape[0], eps.shape[0]
    m = moments_nhwc.half().float().permute(0, 3, 1, 2)
    im = torch.arange(B, device=noise.device) % Bm
    ie = torch.arange(B, device=noise.device) % Be
    mean, logvar = m[im, :C], m[im, C:2 * C]
    if eps.dtype == torch.float32:                     # fp32 posterior (upcast VAE)
        z = posterior_sample_ref(torch.cat([mean, logvar], dim=1), eps[ie])
    else:                                              # fp16 posterior: every op rounds to fp16
        z = posterior_sample_ref(torch.cat([mean, logvar], dim=1).half(), eps[ie].half())
    z = scaling_factor * z.half()
    return add_noise_ref(z, noise.half(), sigma)
