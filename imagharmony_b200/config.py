"""Architecture description of the SDXL-base UNet the reference drives (custom_pipelines.py:338-345) plus the
IMAGHarmony adapter hyper-parameters (test.py:12-15, ip_adapter.py:99-123). [3P] values are the public
stabilityai/stable-diffusion-xl-base-1.0 unet/config.json restated in SURVEY.md appendix A.1."""
from __future__ import annotations

from dataclasses import dataclass, field, fields, replace
from typing import Optional, Tuple


@dataclass(frozen=True)
class UNetConfig:
    in_channels: int = 4
    out_channels: int = 4
    block_out_channels: Tuple[int, ...] = (320, 640, 1280)
    layers_per_block: int = 2
    # transformer depth per resolution level; 0 = no attention at that level (DownBlock2D / UpBlock2D)
    transformer_layers_per_block: Tuple[int, ...] = (0, 2, 10)
    attention_head_dim: int = 64
    cross_attention_dim: int = 2048
    norm_num_groups: int = 32
    addition_time_embed_dim: int = 256
    pooled_embed_dim: int = 1280          # text_embeds width (projection_class_embeddings_input_dim = 6*256 + 1280)
    sample_size: int = 128
    # IMAGHarmony / IP-Adapter
    num_ip_tokens: int = 4
    ip_target_substring: str = "down_blocks.2.attentions.1"   # ip_adapter.py:117 (hard-coded in the reference)
    # transformer depth of the mid block; None = the last level's depth (SDXL-base: 10)
    mid_block_layers: Optional[int] = None
    # micro-conditioning ids: 6 = (original size, crop, target size); 5 = (original size, crop, aesthetic score) for
    # models that require an aesthetics score (the SDXL refiner)
    num_time_ids: int = 6

    @property
    def time_embed_dim(self) -> int:
        return self.block_out_channels[0] * 4

    @property
    def add_embed_in(self) -> int:
        return self.num_time_ids * self.addition_time_embed_dim + self.pooled_embed_dim

    @property
    def mid_depth(self) -> int:
        return self.transformer_layers_per_block[-1] if self.mid_block_layers is None else self.mid_block_layers

    def heads(self, channels: int) -> int:
        return channels // self.attention_head_dim


SDXL_BASE = UNetConfig()

# A structurally identical miniature (same block types, skip wiring, IP layer placement) used by the CPU-side tests
# and the golden fixtures; channels stay multiples of 64 so every sm_90a kernel path is exercised.
TINY = UNetConfig(
    block_out_channels=(64, 128, 256),
    transformer_layers_per_block=(0, 1, 2),
    cross_attention_dim=128,
    addition_time_embed_dim=32,
    pooled_embed_dim=64,
    sample_size=32,
)

# [3P] public stabilityai/stable-diffusion-xl-refiner-1.0 unet/config.json, recalled and not checked against the file:
# block_out_channels [384, 768, 1536, 1536]; down blocks DownBlock2D, CrossAttnDownBlock2D x2, DownBlock2D;
# transformer_layers_per_block 4 (so the mid block has depth 4); attention_head_dim [6, 12, 24, 24] (head counts: 64
# wide at every level); cross_attention_dim 1280; addition_time_embed_dim 256; projection_class_embeddings_input_dim
# 2560 = 5 * 256 + 1280 (model_index.json: requires_aesthetics_score = true); use_linear_projection; 32 groups;
# layers_per_block 2; sample_size 128.  The IMAGHarmony adapter is trained for the base: no image-prompt tokens.
SDXL_REFINER = UNetConfig(
    block_out_channels=(384, 768, 1536, 1536),
    transformer_layers_per_block=(0, 4, 4, 0),
    mid_block_layers=4,
    cross_attention_dim=1280,
    addition_time_embed_dim=256,
    pooled_embed_dim=1280,
    num_time_ids=5,
    num_ip_tokens=0,
)

# the refiner's structure in miniature (four levels, attention-free first and last levels, a mid block deeper than the
# last level, five time ids, text-only cross-attention) with a cross_attention_dim that differs from TINY's
TINY_REFINER = UNetConfig(
    block_out_channels=(64, 128, 256, 256),
    transformer_layers_per_block=(0, 1, 2, 0),
    mid_block_layers=1,
    cross_attention_dim=192,
    addition_time_embed_dim=32,
    pooled_embed_dim=64,
    sample_size=32,
    num_time_ids=5,
    num_ip_tokens=0,
)


@dataclass(frozen=True)
class ControlNetConfig(UNetConfig):
    """[3P] diffusers ControlNetModel config of an SDXL ControlNet (e.g. diffusers/controlnet-canny-sdxl-1.0
    config.json): the UNet's encoder half (same block fields as UNetConfig) plus the conditioning-image embedding
    (SURVEY appendix A.7).  `global_pool_conditions` models are not supported (IHError at construction)."""
    conditioning_channels: int = 3
    conditioning_embedding_out_channels: Tuple[int, ...] = (16, 32, 96, 256)
    controlnet_conditioning_channel_order: str = "rgb"
    global_pool_conditions: bool = False


SDXL_CONTROLNET = ControlNetConfig()
# TINY's encoder with the SDXL embedding's small widths 16/32/96 (the direct small-channel conv path); the last width
# is 128 so that the embedding's conv_out (-> 64) runs on the implicit-GEMM conv as SDXL's 256 -> 320 does
TINY_CONTROLNET = ControlNetConfig(
    block_out_channels=TINY.block_out_channels,
    transformer_layers_per_block=TINY.transformer_layers_per_block,
    cross_attention_dim=TINY.cross_attention_dim,
    addition_time_embed_dim=TINY.addition_time_embed_dim,
    pooled_embed_dim=TINY.pooled_embed_dim,
    sample_size=TINY.sample_size,
    conditioning_embedding_out_channels=(16, 32, 96, 128),
)


@dataclass(frozen=True)
class T2IAdapterConfig:
    """[3P] diffusers 0.30.0 T2IAdapter config (e.g. TencentARC/t2i-adapter-canny-sdxl-1.0 config.json):
    `full_adapter_xl` with one feature per UNet injection point (imagharmony_b200.t2i_adapter)."""
    in_channels: int = 3
    channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    num_res_blocks: int = 2
    downscale_factor: int = 16
    adapter_type: str = "full_adapter_xl"


SDXL_T2I_ADAPTER = T2IAdapterConfig()
# the same architecture at TINY's widths (its three UNet levels and mid block)
TINY_T2I_ADAPTER = T2IAdapterConfig(channels=(64, 128, 256, 256))


# diffusers config.json fields the native UNet / ControlNet build only with these values (absent = the default)
_REQUIRED = {
    "addition_embed_type": ("text_time",),
    "use_linear_projection": (True,),
    "mid_block_type": ("UNetMidBlock2DCrossAttn",),
    "act_fn": ("silu",),
    "time_embedding_type": ("positional",),
    "flip_sin_to_cos": (True,),
    "freq_shift": (0,),
    "norm_eps": (1e-5,),
    "resnet_time_scale_shift": ("default",),
    "conv_in_kernel": (3,),
    "conv_out_kernel": (3,),
    "downsample_padding": (1,),
    "mid_block_scale_factor": (1, 1.0),
    "resnet_out_scale_factor": (1, 1.0),
    "center_input_sample": (False,),
    "upcast_attention": (None, False),
    "only_cross_attention": (False,),
    "dual_cross_attention": (False,),
    "mid_block_only_cross_attention": (None, False),
    "attention_type": ("default",),
    "class_embed_type": (None,),
    "num_class_embeds": (None,),
    "encoder_hid_dim": (None,),
    "encoder_hid_dim_type": (None,),
    "time_cond_proj_dim": (None,),
    "time_embedding_dim": (None,),
    "time_embedding_act_fn": (None,),
    "timestep_post_act": (None,),
    "cross_attention_norm": (None,),
    "reverse_transformer_layers_per_block": (None,),
    "class_embeddings_concat": (False,),
}


def config_from_diffusers(meta: dict, cls=UNetConfig, requires_aesthetics_score: bool = False):
    """A diffusers UNet2DConditionModel / ControlNetModel `config.json` (as a dict) -> `cls` (UNetConfig or
    ControlNetConfig), starting from cls's defaults (SDXL-base).  IHError for a model the native blocks cannot build.

    * `attention_head_dim` is a head count per level in diffusers' SDXL configs (`num_attention_heads` wins when set);
      the native attention is 64 wide, so block_out_channels[i] / heads[i] must be 64 at every level.
    * `transformer_layers_per_block` (an int or one entry per level) is taken per level, then zeroed at the DownBlock2D
      levels; the mid block's depth is its last entry before that (4 for the refiner, 10 for the base).
    * `num_time_ids` is 5 when the pipeline's model_index.json sets `requires_aesthetics_score`, else 6: the UNet config
      alone cannot tell, because projection_class_embeddings_input_dim = 2560 reads as 5 * 256 + 1280 and as 6 * 256 +
      1024.  pooled_embed_dim = projection_class_embeddings_input_dim - num_time_ids * addition_time_embed_dim.
    * A 5-id (aesthetic-score) UNet gets no image-prompt tokens: the IMAGHarmony adapter is trained for the base."""
    from ._lib import IHError
    for k, ok in _REQUIRED.items():
        if k in meta and meta[k] not in ok:
            raise IHError(f"diffusers config: {k} = {meta[k]!r} is not supported (supported: {list(ok)})")
    names = {f.name for f in fields(cls)}
    base = cls()
    upd = {k: (tuple(v) if isinstance(v, list) else v) for k, v in meta.items()
           if k in names and k not in ("attention_head_dim", "transformer_layers_per_block")}
    boc = upd.get("block_out_channels", base.block_out_channels)
    n = len(boc)
    if not isinstance(upd.get("layers_per_block", base.layers_per_block), int):
        raise IHError(f"diffusers config: layers_per_block must be one int, got {upd['layers_per_block']!r}")
    tl = meta.get("transformer_layers_per_block", list(base.transformer_layers_per_block))
    tl = [tl] * n if isinstance(tl, int) else list(tl)
    if len(tl) != n or not all(isinstance(d, int) and d >= 0 for d in tl):
        raise IHError(f"diffusers config: transformer_layers_per_block {tl!r} must be an int or one int per level")
    mid = tl[-1]
    dbt = meta.get("down_block_types")
    if dbt is not None:
        if len(dbt) != n or any(t not in ("DownBlock2D", "CrossAttnDownBlock2D") for t in dbt):
            raise IHError(f"diffusers config: down_block_types {dbt!r} (one DownBlock2D / CrossAttnDownBlock2D per level)")
        tl = [d if t == "CrossAttnDownBlock2D" else 0 for t, d in zip(dbt, tl)]
        ubt = meta.get("up_block_types")
        if ubt is not None and list(ubt) != [t.replace("Down", "Up") for t in reversed(dbt)]:
            raise IHError(f"diffusers config: up_block_types {ubt!r} do not mirror down_block_types {dbt!r}")
    upd["transformer_layers_per_block"] = tuple(tl)
    upd["mid_block_layers"] = None if mid == tl[-1] else mid
    heads = meta.get("num_attention_heads") or meta.get("attention_head_dim")
    if heads is not None:
        heads = [heads] * n if isinstance(heads, int) else list(heads)
        if len(heads) != n or any(not isinstance(h, int) or h <= 0 or c != 64 * h for c, h in zip(boc, heads)):
            raise IHError(f"diffusers config: block_out_channels {list(boc)} with {heads} heads: the native attention "
                          "needs heads of width 64 at every level")
    upd["num_time_ids"] = 5 if requires_aesthetics_score else 6
    if "projection_class_embeddings_input_dim" in meta:
        pooled = int(meta["projection_class_embeddings_input_dim"]) - upd["num_time_ids"] * int(
            upd.get("addition_time_embed_dim", base.addition_time_embed_dim))
        if pooled <= 0:
            raise IHError(f"diffusers config: projection_class_embeddings_input_dim "
                          f"{meta['projection_class_embeddings_input_dim']} leaves no pooled text embedding")
        upd["pooled_embed_dim"] = pooled
    if requires_aesthetics_score:
        upd["num_ip_tokens"] = 0
    try:
        return replace(base, **upd)
    except TypeError as e:
        raise IHError(f"diffusers config: {e}") from None


@dataclass(frozen=True)
class HarmonyConfig:
    """HarmonyAttention hyper-parameters (train.py:189-197; shipped values run.sh:17-20, test.py:12-15)."""
    image_hidden_size: int = 1280
    text_context_dim: int = 2048
    inter_dim: int = 2560
    cross_heads: int = 8
    reshape_blocks: int = 8
    cross_value_dim: int = 64
    scale: float = 1.0


HARMONY_DEFAULT = HarmonyConfig()
HARMONY_TINY = HarmonyConfig(image_hidden_size=64, text_context_dim=128, inter_dim=256, cross_heads=4,
                             reshape_blocks=4, cross_value_dim=16)


@dataclass(frozen=True)
class VAEConfig:
    """[3P] diffusers AutoencoderKL of SDXL (decoder half): vae/config.json of stabilityai/stable-diffusion-xl-base-1.0."""
    latent_channels: int = 4
    out_channels: int = 3
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    layers_per_block: int = 2
    norm_num_groups: int = 32
    scaling_factor: float = 0.13025
    sample_size: int = 1024               # tiling: tiles of sample_size pixels (= sample_size / 8 latents), 25 % overlap
    tile_overlap_factor: float = 0.25
    force_upcast: bool = True             # vae/config.json of SDXL-base: the reference upcasts the VAE to fp32 (custom_pipelines.py:366-371)

    @property
    def tile_latent_min_size(self) -> int:
        return int(self.sample_size / (2 ** (len(self.block_out_channels) - 1)))

    @property
    def decoder_channels(self) -> Tuple[int, ...]:
        return tuple(reversed(self.block_out_channels))


SDXL_VAE = VAEConfig()
# miniature with the same block structure (mid attention, a channel-changing shortcut); channels stay multiples of 64
# because the implicit-GEMM conv kernel needs Cin % 64 == 0
TINY_VAE = VAEConfig(block_out_channels=(64, 64, 128, 128), layers_per_block=1, norm_num_groups=8, sample_size=64)


@dataclass(frozen=True)
class TinyVAEConfig:
    """[3P] diffusers AutoencoderTiny (decoder half) with the defaults of the published TAESD-XL config.json
    (madebyollin/taesdxl): ReLU, nearest 2x upsampling, 64 channels throughout, blocks (3, 3, 3, 1)."""
    latent_channels: int = 4
    out_channels: int = 3
    decoder_block_out_channels: Tuple[int, ...] = (64, 64, 64, 64)
    num_decoder_blocks: Tuple[int, ...] = (3, 3, 3, 1)
    scaling_factor: float = 1.0


TAESDXL = TinyVAEConfig()
