"""SDXL LoRA adapters merged into the native UNet and CLIP text towers.

A LoRA adds f * up @ down to a weight W [N, K'] (K' = Cin * kh * kw for a conv: the canonical flattening of an OIHW
weight).  Here that delta is merged into the canonical fp16 parameters on the device and the kernel-layout weights are
re-derived (`SDXLEncoderModel.finalize()`), so a denoise step runs exactly the kernels it runs without a LoRA.

Loader (`parse_lora`).  Accepted key formats:
  * kohya / sd-scripts: `lora_unet_<flat>.lora_down.weight`, `.lora_up.weight`, `.alpha`; text towers `lora_te1_<flat>`
    and `lora_te2_<flat>`.  `<flat>` is a module name with dots replaced by underscores, SGM-named
    (`input_blocks_4_1_transformer_blocks_0_attn1_to_q`) or diffusers-named (`down_blocks_1_attentions_0_...`).
  * diffusers / PEFT: `unet.<name>.lora_A.weight` (down) / `.lora_B.weight` (up), `text_encoder.` / `text_encoder_2.`
    with transformers names (`text_model.encoder.layers.N.self_attn.q_proj`, `mlp.fc1`, ...).
The scaling of a module is alpha / r when its `.alpha` key exists, else 1.  Names resolve by exact lookup in tables
built from the native model's module tree (`unet_name_table`, `text_name_table`); the SGM numbering is derived from the
UNetConfig level structure.  Everything else raises IHError naming the keys, before any weight changes: LyCORIS
variants (LoHa `hada_`, LoKr `lokr_`), DoRA (`dora_scale`), Tucker `lora_mid`, full diffs (`.diff`, `.diff_b`), legacy
diffusers attention-processor keys, modules the native model does not have or cannot target (conv_in, conv_out, the
time / added embeddings, norms), and text-tower keys for a tower the pipeline's prompt encoder does not have.

Merge (`LoraWeights`).  The original fp16 tensor of every parameter (or q|k|v row slice) an adapter touches is kept on
the device, and every merge recomputes live = orig + sum_k f_k * up_k @ down_k from it, one `ops.linear` launch (the
library's tensor-core GEMM with alpha and a residual, `ih_gemm_scaled_f16`) per term:
    f_k = fp32(s * w_k * alpha_k / r_k)   (evaluated left to right in fp32; s the per-call scale, w_k the adapter weight)
The rank is zero-padded to a multiple of 64 (exact).  Each term costs one fp16 rounding of fp32(f_k * up_k down_k + prev);
several terms chain orig -> scratch / live -> ... -> live so that a launch's residual and output never alias.  A term
with f_k = 0 is skipped, and a tensor without terms is copied back from its original bit for bit.
"""
from __future__ import annotations

import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from . import ops
from ._lib import IHError

UNET, TE1, TE2 = "unet", "text_encoder", "text_encoder_2"
COMPONENTS = (UNET, TE1, TE2)
DEFAULT_WEIGHT_NAME = "pytorch_lora_weights.safetensors"

_KOHYA_PREFIX = {"lora_unet_": UNET, "lora_te1_": TE1, "lora_te2_": TE2}
_PEFT_PREFIX = {"unet.": UNET, "text_encoder.": TE1, "text_encoder_2.": TE2}
_KOHYA_SUFFIX = {".lora_down.weight": "down", ".lora_up.weight": "up", ".alpha": "alpha"}
_PEFT_SUFFIX = {".lora_A.weight": "down", ".lora_B.weight": "up", ".alpha": "alpha"}
_VARIANTS = ("hada_", "lokr_", "dora_scale", "lora_mid")
_SHOW = 5


# ---------------------------------------------------------------------------------------------------------------------
# name tables
# ---------------------------------------------------------------------------------------------------------------------
_RES_SGM = {"conv1": "in_layers.2", "time_emb_proj": "emb_layers.1", "conv2": "out_layers.3",
            "conv_shortcut": "skip_connection"}


def _transformer_leaves(t) -> List[str]:
    leaves = ["proj_in", "proj_out"]
    for i in range(len(t.transformer_blocks)):
        b = f"transformer_blocks.{i}."
        for a in ("attn1", "attn2"):
            leaves += [f"{b}{a}.to_q", f"{b}{a}.to_k", f"{b}{a}.to_v", f"{b}{a}.to_out.0"]
        leaves += [f"{b}ff.net.0.proj", f"{b}ff.net.2"]
    return leaves


def _resnet_leaves(r) -> List[str]:
    return [n for n in _RES_SGM if getattr(r, n) is not None]


def unet_name_table(unet) -> Dict[str, str]:
    """{native (diffusers) module name: SGM name} for every LoRA-targetable module of the native UNet: the Linear and
    Conv layers of each Transformer2DModel and ResnetBlock2D and the down/upsampler convs.  The SGM numbering
    (input_blocks / middle_block / output_blocks) follows the UNetConfig level structure, so it holds for any number of
    levels, attention-free levels and mid-block depth."""
    cfg = unet.config
    lpb = cfg.layers_per_block
    sgm_of_block: Dict[str, str] = {}
    for i, blk in enumerate(unet.down_blocks):
        for j in range(lpb):
            idx = 1 + i * (lpb + 1) + j
            sgm_of_block[f"down_blocks.{i}.resnets.{j}"] = f"input_blocks.{idx}.0"
            if blk.has_attn:
                sgm_of_block[f"down_blocks.{i}.attentions.{j}"] = f"input_blocks.{idx}.1"
        if blk.has_down:
            sgm_of_block[f"down_blocks.{i}.downsamplers.0"] = f"input_blocks.{1 + i * (lpb + 1) + lpb}.0"
    sgm_of_block["mid_block.resnets.0"] = "middle_block.0"
    sgm_of_block["mid_block.attentions.0"] = "middle_block.1"
    sgm_of_block["mid_block.resnets.1"] = "middle_block.2"
    for u, blk in enumerate(unet.up_blocks):
        for j in range(lpb + 1):
            idx = u * (lpb + 1) + j
            sgm_of_block[f"up_blocks.{u}.resnets.{j}"] = f"output_blocks.{idx}.0"
            if blk.has_attn:
                sgm_of_block[f"up_blocks.{u}.attentions.{j}"] = f"output_blocks.{idx}.1"
        if blk.has_up:
            sgm_of_block[f"up_blocks.{u}.upsamplers.0"] = f"output_blocks.{u * (lpb + 1) + lpb}.{2 if blk.has_attn else 1}"
    from .unet import Resample, ResnetBlock2D, Transformer2DModel
    table: Dict[str, str] = {}
    for name, m in unet.named_modules():
        if name not in sgm_of_block:
            continue
        sgm = sgm_of_block[name]
        if isinstance(m, Transformer2DModel):
            for leaf in _transformer_leaves(m):
                table[f"{name}.{leaf}"] = f"{sgm}.{leaf}"
        elif isinstance(m, ResnetBlock2D):
            for leaf in _resnet_leaves(m):
                table[f"{name}.{leaf}"] = f"{sgm}.{_RES_SGM[leaf]}"
        elif isinstance(m, Resample):
            table[f"{name}.conv"] = f"{sgm}.conv" if m.up else f"{sgm}.op"
    return table


def text_name_table(num_layers: int) -> List[str]:
    """transformers module names of the targetable layers of a CLIP text tower: q/k/v/out projections, fc1, fc2."""
    out = []
    for i in range(num_layers):
        p = f"text_model.encoder.layers.{i}."
        out += [p + f"self_attn.{n}_proj" for n in ("q", "k", "v", "out")] + [p + "mlp.fc1", p + "mlp.fc2"]
    return out


def _lookup(names: Dict[str, str]) -> Dict[str, str]:
    """{alias: native name} with every alias also flattened with underscores; raises on an ambiguous alias."""
    out: Dict[str, str] = {}
    for alias, native in names.items():
        for a in (alias, alias.replace(".", "_")):
            if out.setdefault(a, native) != native:
                raise IHError(f"LoRA name table: {a!r} names both {out[a]!r} and {native!r}")
    return out


# ---------------------------------------------------------------------------------------------------------------------
# targets: the tensors a LoRA may change
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class Target:
    """One [N, K'] weight view a LoRA term is merged into; `kernel` is (kh, kw) for a conv, None for a linear."""
    live: torch.Tensor
    kernel: Optional[Tuple[int, int]]
    cin: int


def unet_targets(unet) -> Dict[str, Target]:
    """{native name: Target} of every targetable UNet module (the canonical parameter, flattened to [N, K'])."""
    mods = dict(unet.named_modules())
    out = {}
    for name in unet_name_table(unet):
        w = mods[name].weight.detach()
        kernel = tuple(w.shape[2:]) if w.dim() == 4 else None
        out[name] = Target(w.view(w.shape[0], -1), kernel, w.shape[1])
    return out


def tower_targets(tower) -> Dict[str, Target]:
    """{transformers name: Target} of a ClipTextTower: q / k / v are row slices of the fused [3C, C] q|k|v weight."""
    out = {}
    C = tower.cfg.hidden_size
    names = text_name_table(len(tower.enc.layers))
    for i, L in enumerate(tower.enc.layers):
        views = [L.w_qkv[:C], L.w_qkv[C:2 * C], L.w_qkv[2 * C:], L.w_o, L.w_fc1, L.w_fc2]
        for n, v in zip(names[6 * i:6 * i + 6], views):
            out[n] = Target(v, None, v.shape[1])
    return out


def prompt_towers(prompt_encoder) -> Dict[str, object]:
    """{component: ClipTextTower} of a pipeline's prompt encoder: both towers, tower 2 alone (the refiner's single-tower
    mode) or none (a prompt encoder without native CLIP towers)."""
    towers = list(getattr(prompt_encoder, "text_encoders", None) or [])
    if not towers:
        return {}
    return {TE2: towers[-1]} if len(towers) == 1 else {TE1: towers[0], TE2: towers[1]}


# ---------------------------------------------------------------------------------------------------------------------
# loader
# ---------------------------------------------------------------------------------------------------------------------
def read_state_dict(src, weight_name: Optional[str] = None) -> Dict[str, torch.Tensor]:
    """A state dict as is, or the tensors of a `.safetensors` / `.bin` file, or of `weight_name` (default
    pytorch_lora_weights.safetensors) inside a directory."""
    if isinstance(src, dict):
        return src
    path = str(src)
    if os.path.isdir(path):
        path = os.path.join(path, weight_name or DEFAULT_WEIGHT_NAME)
    if not os.path.isfile(path):
        raise FileNotFoundError(f"no LoRA weights at {path}")
    if path.endswith(".safetensors"):
        from safetensors.torch import load_file
        return load_file(path)
    return torch.load(path, map_location="cpu", weights_only=True)


def _refuse(what: str, keys: List[str]) -> None:
    if keys:
        more = f" (and {len(keys) - _SHOW} more)" if len(keys) > _SHOW else ""
        raise IHError(f"LoRA: {what}: {keys[:_SHOW]}{more}")


def _split_key(key: str):
    """-> (component, module alias, part) of a kohya or PEFT key, or None."""
    for prefixes, suffixes in ((_KOHYA_PREFIX, _KOHYA_SUFFIX), (_PEFT_PREFIX, _PEFT_SUFFIX)):
        for pre, comp in prefixes.items():
            if not key.startswith(pre):
                continue
            for suf, part in suffixes.items():
                if key.endswith(suf) and len(key) > len(pre) + len(suf):
                    return comp, key[len(pre):-len(suf)], part
    return None


def parse_lora(sd: Dict[str, torch.Tensor], tables: Dict[str, Dict[str, str]],
               targets: Dict[str, Dict[str, Target]]) -> Dict[str, Dict[str, Tuple[torch.Tensor, torch.Tensor, float]]]:
    """state dict -> {component: {native module name: (up [N, r] fp32, down [r, K'] fp32, alpha)}} (alpha = r when the
    file has no `.alpha`, so that alpha / r = 1).  `tables[c]` maps every accepted alias of component c to its native
    name, `targets[c]` gives the shapes.  IHError, naming the keys, for anything that cannot be merged exactly."""
    keys = sorted(sd)
    _refuse("LyCORIS / DoRA / Tucker variants are not supported (keys)",
            [k for k in keys if any(v in k for v in _VARIANTS)])
    _refuse("full weight differences are not supported (keys)", [k for k in keys if k.endswith((".diff", ".diff_b"))])
    _refuse("legacy diffusers attention-processor keys are not supported (keys)",
            [k for k in keys if ".processor." in k or "_lora.down." in k or "_lora.up." in k])
    split = {k: _split_key(k) for k in keys}
    _refuse("keys of no known LoRA format", [k for k in keys if split[k] is None])
    _refuse("the pipeline's prompt encoder has no such text tower (keys)",
            [k for k in keys if split[k][0] != UNET and split[k][0] not in tables])
    _refuse("keys for modules the native model does not have or cannot target",
            [k for k in keys if split[k][1] not in tables[split[k][0]]])
    parts: Dict[Tuple[str, str], Dict[str, Tuple[str, torch.Tensor]]] = {}
    dup = []
    for k in keys:
        comp, alias, part = split[k]
        slot = parts.setdefault((comp, tables[comp][alias]), {})
        if part in slot:
            dup += [slot[part][0], k]
        slot[part] = (k, sd[k])
    _refuse("several keys name the same module", dup)
    out: Dict[str, Dict[str, Tuple[torch.Tensor, torch.Tensor, float]]] = {}
    bad = []
    for (comp, name), slot in sorted(parts.items()):
        t = targets[comp][name]
        if "up" not in slot or "down" not in slot:
            bad += [k for k, _ in slot.values()]
            continue
        (ku, up), (kd, down) = slot["up"], slot["down"]
        up, down = up.detach().float(), down.detach().float()
        r = down.shape[0]
        N, Kp = t.live.shape
        if t.kernel is None:
            ok = up.shape == (N, r) and down.shape == (r, Kp)
        else:
            ok = up.shape == (N, r, 1, 1) and down.shape == (r, t.cin) + t.kernel
        if not ok:
            bad += [ku, kd]
            continue
        alpha = float(slot["alpha"][1]) if "alpha" in slot else float(r)
        out.setdefault(comp, {})[name] = (up.reshape(N, r), down.reshape(r, Kp), alpha)
    _refuse("keys without their up / down partner or with shapes that do not fit the module", bad)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# merge
# ---------------------------------------------------------------------------------------------------------------------
def term_factor(s: float, w: float, alpha: float, r: int) -> float:
    """f = fp32(s * w * alpha / r), evaluated left to right with a float32 rounding after each operation."""
    f32 = np.float32
    return float(f32(f32(f32(s) * f32(w)) * f32(alpha)) / f32(r))


@dataclass
class _Term:
    up: torch.Tensor       # [N, rp] with the rank zero-padded to a multiple of 64
    down_t: torch.Tensor   # [K', rp]
    alpha: float
    rank: int


@dataclass
class Adapter:
    name: str
    terms: Dict[str, Dict[str, _Term]] = field(default_factory=dict)    # component -> module -> term


def _pad_term(up: torch.Tensor, down: torch.Tensor, alpha: float, like: torch.Tensor) -> _Term:
    N, r = up.shape
    rp = (r + 63) // 64 * 64
    u = torch.zeros((N, rp), dtype=like.dtype, device=like.device)
    u[:, :r] = up.to(like.dtype)
    d = torch.zeros((down.shape[1], rp), dtype=like.dtype, device=like.device)
    d[:, :r] = down.t().to(like.dtype)
    return _Term(u, d, alpha, r)


class LoraWeights:
    """The adapters loaded into one pipeline and the merge state of its UNet and text towers.

    `sync(component, factors)` makes every tensor of that component equal orig + the listed terms: it merges only the
    tensors whose (adapter, f) list changed, and re-derives the UNet's kernel-layout weights (`finalize()`, which also
    bumps graph_epoch) only when a UNet tensor changed.  An unchanged state launches nothing."""

    def __init__(self, unet, towers: Dict[str, object]):
        self.unet = unet
        self.towers = towers
        self.targets: Dict[str, Dict[str, Target]] = {UNET: unet_targets(unet)}
        self.tables: Dict[str, Dict[str, str]] = {}
        table = unet_name_table(unet)
        self.tables[UNET] = _lookup({**{n: n for n in table}, **{s: n for n, s in table.items()}})
        for comp, tower in towers.items():
            self.targets[comp] = tower_targets(tower)
            self.tables[comp] = _lookup({n: n for n in self.targets[comp]})
        self.adapters: Dict[str, Adapter] = {}
        self.orig: Dict[Tuple[str, str], torch.Tensor] = {}
        self.merged: Dict[Tuple[str, str], tuple] = {}       # (component, module) -> ((adapter, f), ...) merged now

    def add(self, name: str, sd: Dict[str, torch.Tensor]) -> Adapter:
        parsed = parse_lora(sd, self.tables, self.targets)
        if not parsed:
            raise IHError(f"LoRA {name!r}: the state dict holds no LoRA weights")
        ad = Adapter(name)
        for comp, mods in parsed.items():
            for mod, (up, down, alpha) in mods.items():
                live = self.targets[comp][mod].live
                ad.terms.setdefault(comp, {})[mod] = _pad_term(up, down, alpha, live)
        for comp, mods in ad.terms.items():
            for mod in mods:
                if (comp, mod) not in self.orig:
                    self.orig[(comp, mod)] = self.targets[comp][mod].live.clone()
                    self.merged[(comp, mod)] = ()
        self.adapters[name] = ad
        return ad

    def remove(self, name: str) -> None:
        """Drop an adapter; call `sync` afterwards, then `release()` frees the originals nothing touches any more."""
        del self.adapters[name]

    def components(self, name: str) -> List[str]:
        return [c for c in COMPONENTS if c in self.adapters[name].terms]

    def sync(self, comp: str, factors: Dict[str, Tuple[float, float]]) -> int:
        """factors: {adapter name: (s, w)} of the active adapters for this component.  -> number of tensors merged."""
        want: Dict[str, list] = {}
        for name, (s, w) in factors.items():
            for mod, t in self.adapters[name].terms.get(comp, {}).items():
                f = term_factor(s, w, t.alpha, t.rank)
                if f != 0.0:
                    want.setdefault(mod, []).append((name, f, t))
        changed = 0
        for (c, mod), have in self.merged.items():
            if c != comp:
                continue
            terms = want.get(mod, [])
            sig = tuple((n, f) for n, f, _ in terms)
            if sig == have:
                continue
            self._merge(self.targets[comp][mod].live, self.orig[(comp, mod)], [(f, t) for _, f, t in terms])
            self.merged[(comp, mod)] = sig
            changed += 1
        if changed and comp == UNET:
            self.unet.finalize()
        return changed

    def release(self) -> None:
        """Forget the originals of tensors no loaded adapter touches (sync has already restored them)."""
        used = {(c, m) for ad in self.adapters.values() for c, mods in ad.terms.items() for m in mods}
        for key in [k for k in self.orig if k not in used]:
            if self.merged[key]:
                raise IHError(f"LoRA: {key} still holds merged terms")
            del self.orig[key], self.merged[key]

    @staticmethod
    def _merge(live: torch.Tensor, orig: torch.Tensor, terms) -> None:
        if not terms:
            live.copy_(orig)
            return
        scratch = torch.empty_like(live) if len(terms) > 1 else None
        prev = orig
        for k, (f, t) in enumerate(terms):
            out = live if (len(terms) - 1 - k) % 2 == 0 else scratch
            ops.linear(t.up, t.down_t, alpha=f, residual=prev, out=out)
            prev = out

    def kept_bytes(self) -> int:
        return sum(t.numel() * t.element_size() for t in self.orig.values())
