"""Restatement of what the LoRA tests compare against: random LoRAs written in the kohya (SGM or diffusers names) and
diffusers / PEFT key formats, the fp64 merge, and PEFT's unfused LoRA forward ([3P] peft.tuners.lora.Linear / Conv2d:
base(x) + f * lora_B(lora_A(x)), f = scale * weight * alpha / r) attached to the oracle UNet and to transformers' CLIP
text models with forward hooks."""
import torch
import torch.nn.functional as F

KOHYA = {"unet": "lora_unet_", "text_encoder": "lora_te1_", "text_encoder_2": "lora_te2_"}
PEFT = {"unet": "unet.", "text_encoder": "text_encoder.", "text_encoder_2": "text_encoder_2."}


def module_shapes(model, names):
    """{name: weight shape} of the named Linear / Conv2d modules of any module tree."""
    mods = dict(model.named_modules())
    return {n: tuple(mods[n].weight.shape) for n in names}


def random_lora(shapes, rank, seed, rel=0.1, alpha=None, fp16=True):
    """{name: (up [N, r] or [N, r, 1, 1], down [r, K] or [r, Cin, kh, kw], alpha)} with up @ down of about rel / sqrt(K')
    per element (a delta of ~rel |W| for weights drawn U(+-1/sqrt(K')))."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name, sh in shapes.items():
        N, kdim = sh[0], int(torch.tensor(sh[1:]).prod())
        r = min(rank, N, kdim)
        down = torch.randn((r,) + tuple(sh[1:]), generator=g) / kdim ** 0.5
        up = torch.randn((N, r) + ((1, 1) if len(sh) == 4 else ()), generator=g) * rel / r ** 0.5 * (3.0 / kdim) ** 0.5
        if fp16:
            up, down = up.half().float(), down.half().float()
        out[name] = (up, down, float(r) if alpha is None else float(alpha))
    return out


def to_kohya(lora, component, names=None):
    """kohya keys; `names` maps a native name to the alias to write (e.g. its SGM name), dots flattened to '_'."""
    sd = {}
    for n, (up, down, alpha) in lora.items():
        flat = KOHYA[component] + (names[n] if names else n).replace(".", "_")
        sd[flat + ".lora_up.weight"], sd[flat + ".lora_down.weight"] = up, down
        sd[flat + ".alpha"] = torch.tensor(alpha)
    return sd


def to_peft(lora, component):
    sd = {}
    for n, (up, down, alpha) in lora.items():
        sd[PEFT[component] + n + ".lora_B.weight"], sd[PEFT[component] + n + ".lora_A.weight"] = up, down
        sd[PEFT[component] + n + ".alpha"] = torch.tensor(alpha)
    return sd


def delta64(up, down):
    """up @ down in fp64 in the canonical [N, K'] layout."""
    return up.double().reshape(up.shape[0], -1) @ down.double().reshape(down.shape[0], -1)


def merged64(orig, terms):
    """orig + sum f * up @ down in fp64; terms = [(f, up, down)]."""
    w = orig.double().reshape(orig.shape[0], -1).clone()
    for f, up, down in terms:
        w += f * delta64(up, down)
    return w


def attach_unfused(model, lora, factor):
    """PEFT's unfused forward on `model`: each named module's output gains factor(alpha, r) * up(down(x)).  Returns the
    hook handles."""
    mods = dict(model.named_modules())
    handles = []
    for name, (up, down, alpha) in lora.items():
        m = mods[name]
        f = factor(alpha, down.shape[0])

        def hook(mod, inp, out, up=up, down=down, f=f):
            x = inp[0]
            u, d = up.to(x.dtype).to(x.device), down.to(x.dtype).to(x.device)
            if isinstance(mod, torch.nn.Conv2d):
                y = F.conv2d(F.conv2d(x, d, None, mod.stride, mod.padding), u)
            else:
                y = F.linear(F.linear(x, d), u)
            return out + f * y
        handles.append(m.register_forward_hook(hook))
    return handles
