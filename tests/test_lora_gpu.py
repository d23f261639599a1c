"""GPU tests of merged LoRA adapters: the merge GEMMs at SDXL-base shapes against the fp64 merge, exact re-derivation of
the kernel-layout weights, graph re-capture through a pipeline, parity of the merged native UNet and CLIP text towers
with PEFT's unfused forward (tests/lora_ref.py) under the bar of SURVEY section 7, an unchanged launch list per step, and
the pipeline surface (IPAdapterXL, cross_attention_kwargs, ControlNet)."""
import pytest
import torch

import census
from lora_ref import attach_unfused, merged64, module_shapes, random_lora, to_kohya, to_peft
from test_kernels_gpu import ops  # noqa: F401  (fixture: TF32 off for the census' fp32 references)
from test_unet_census_gpu import plan

pytestmark = pytest.mark.gpu


def _fp16_ulp(x):
    return torch.pow(2.0, torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -14))) - 10)


def test_merge_accuracy_at_sdxl_shapes():
    """attn q / out (1280^2), attn2 k / v (K = 2048), GEGLU (10240 x 1280), FF-out (1280 x 5120), packed 3x3 convs and the
    1x1 shortcut, two adapters of rank 64 and 128: every merged weight is within one fp16 ulp per term of the fp64 merge."""
    from imagharmony_b200.lora import LoraWeights, _pad_term, term_factor
    shapes = {"q": (1280, 1280), "out": (1280, 1280), "attn2.k": (1280, 2048), "geglu": (10240, 1280), "ff_out": (1280, 5120),
              "conv": (1280, 1280, 3, 3), "conv_in320": (640, 320, 3, 3), "shortcut": (640, 320, 1, 1)}
    g = torch.Generator().manual_seed(0)
    a = random_lora(shapes, 64, 1, rel=0.1, alpha=32)
    b = random_lora(shapes, 128, 2, rel=0.1)
    for name, sh in shapes.items():
        kdim = int(torch.tensor(sh[1:]).prod())
        orig = ((torch.rand(sh[0], kdim, generator=g) * 2 - 1) / kdim ** 0.5).half().cuda()
        live = orig.clone()
        terms = [(term_factor(0.7, 1.0, a[name][2], a[name][1].shape[0]), a[name]),
                 (term_factor(0.7, -0.5, b[name][2], b[name][1].shape[0]), b[name])]
        LoraWeights._merge(live, orig, [(f, _pad_term(u.reshape(sh[0], -1), d.reshape(d.shape[0], -1), al, orig))
                                        for f, (u, d, al) in terms])
        torch.cuda.synchronize()
        t64 = [(f, u, d) for f, (u, d, _) in terms]
        want = merged64(orig.cpu(), t64)
        mag = orig.cpu().double().abs() + sum(abs(f) * (u.double().reshape(sh[0], -1) @ d.double().reshape(d.shape[0], -1)).abs()
                                              for f, u, d in t64)
        err = (live.cpu().double() - want).abs() / _fp16_ulp(mag)
        print(f"[merge {name} {tuple(sh)}] max err {err.max().item():.3f} ulp (2 terms)")
        assert err.max().item() <= 2.0, name


def _tiny_native(seed=0):
    """TINY native UNet with random IP weights, and the state dicts it was built from."""
    from imagharmony_b200.config import TINY
    from imagharmony_b200.unet import UNet2DConditionModel
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from oracle.unet_ref import UNetRef
    with torch.device("meta"):
        shapes = shapes_of(UNetRef(TINY))
    sd = random_state_dict(shapes, seed)
    native = UNet2DConditionModel.from_state_dict(TINY, sd, device="cuda")
    procs = torch.nn.ModuleList(native.attn_processors.values())
    ip_sd = random_state_dict(shapes_of(procs), seed + 1)
    procs.load_state_dict({k: v.cuda() for k, v in ip_sd.items()})
    native.finalize()
    return native, sd, ip_sd


def _unet_lora(unet, rank=16, seed=3, rel=0.1):
    from imagharmony_b200.lora import unet_name_table
    return random_lora(module_shapes(unet, unet_name_table(unet)), rank, seed, rel=rel, alpha=rank / 2)


def _inputs(cfg, n, lat, seed=3):
    g = torch.Generator("cpu").manual_seed(seed)
    B = 2 * n
    return (torch.randn(B, 4, lat, lat, generator=g).half(),
            torch.randn(B, 77 + cfg.num_ip_tokens, cfg.cross_attention_dim, generator=g).half(),
            torch.randn(B, cfg.pooled_embed_dim, generator=g).half(),
            torch.tensor([[lat * 8., lat * 8., 0., 0., lat * 8., lat * 8.]] * B))


def test_rederivation_is_exact():
    """A UNet built by from_state_dict from the merged canonical parameters computes bit for bit what the LoRA-merged
    UNet computes: one step and a 10-step graph-replayed trajectory."""
    from imagharmony_b200.config import TINY
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.lora import LoraWeights
    from imagharmony_b200.unet import UNet2DConditionModel
    native, sd, ip_sd = _tiny_native()
    lw = LoraWeights(native, {})
    lw.add("a", to_peft(_unet_lora(native), "unet"))
    lw.sync("unet", {"a": (0.9, 1.0)})
    merged = {k: v.clone() for k, v in native.state_dict().items() if ".processor." not in k}
    fresh = UNet2DConditionModel.from_state_dict(TINY, merged, device="cuda")
    torch.nn.ModuleList(fresh.attn_processors.values()).load_state_dict({k: v.cuda() for k, v in ip_sd.items()})
    fresh.finalize()
    x = _inputs(TINY, 1, 32)
    s, e, te, tid = (v.cuda() for v in x)
    t = torch.full((2,), 500.0, device="cuda")
    with torch.no_grad():
        o1, o2 = native(s, t, e, te, tid), fresh(s, t, e, te, tid)
    assert torch.equal(o1, o2)
    _, e, te, tid = x
    lat = torch.randn(1, 4, 32, 32, generator=torch.Generator().manual_seed(1)).half()
    args = (lat, e[1:], e[:1], te[1:], te[:1], tid[:1], 10)
    r1 = DenoiseEngine(native).run(*args, guidance_scale=5.0, ip_scale=0.7)
    r2 = DenoiseEngine(fresh).run(*args, guidance_scale=5.0, ip_scale=0.7)
    torch.cuda.synchronize()
    assert torch.equal(r1, r2)


def _t2i(pipe, **kw):
    gen = torch.Generator("cpu").manual_seed(9)
    D, P = pipe.unet.config.cross_attention_dim, pipe.unet.config.pooled_embed_dim
    return pipe(prompt_embeds=torch.randn(1, 77, D, generator=gen).half(),
                negative_prompt_embeds=torch.randn(1, 77, D, generator=gen).half(),
                pooled_prompt_embeds=torch.randn(1, P, generator=gen).half(),
                negative_pooled_prompt_embeds=torch.randn(1, P, generator=gen).half(), height=256, width=256,
                num_inference_steps=4, generator=torch.Generator("cuda").manual_seed(3), output_type="latent",
                **kw).images


def test_graphs_recapture_through_load_and_unload():
    from imagharmony_b200.config import TINY
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    pipe = StableDiffusionXLCustomPipeline.from_random(TINY, seed=2)
    sd = to_kohya(_unet_lora(pipe.unet), "unet")
    r0 = _t2i(pipe)
    pipe.load_lora_weights(sd)
    r1 = _t2i(pipe)
    pipe.unload_lora_weights()
    r2 = _t2i(pipe)
    fresh = StableDiffusionXLCustomPipeline.from_random(TINY, seed=2)
    fresh.load_lora_weights(sd)
    r3 = _t2i(fresh)
    torch.cuda.synchronize()
    assert torch.equal(r0, r2) and not torch.equal(r0, r1) and torch.equal(r1, r3)


def _parity(tag, native, ref32, eager16, x, t, merged32=None):
    """SURVEY section 7 against the unfused fp32 oracle.  With `merged32` (the fp32 oracle holding the merged fp16
    weights) the bar also admits the merge's own error, |merged32 - ref32|: rounding W + f up down to fp16 once is what
    a merged (fused) LoRA is, and at full coverage it can outweigh the eager path's activation roundings."""
    s, e, te, tid = x
    with torch.no_grad():
        r = ref32(s.float(), t, e.float(), te.float(), tid).float().cpu()
        eg = eager16(s.cuda(), t, e.cuda(), te.cuda(), tid.cuda())
        o = native(s.cuda(), torch.full((s.shape[0],), t, device="cuda"), e.cuda(), te.cuda(), tid.cuda())
        m = merged32(s.float(), t, e.float(), te.float(), tid).float().cpu() if merged32 is not None else r
    torch.cuda.synchronize()
    e_nat, e_eag, mx = ((o.float().cpu() - r).abs().max().item(), (eg.float().cpu() - r).abs().max().item(),
                        r.abs().max().item())
    e_mrg, e_nat_m = (m - r).abs().max().item(), (o.float().cpu() - m).abs().max().item()
    print(f"[{tag}] native max|err| {e_nat:.3e}  eager-fp16 {e_eag:.3e}  fp16 merge {e_mrg:.3e}  "
          f"native vs merged oracle {e_nat_m:.3e}  max|ref| {mx:.3e}")
    bar = max(2.0 * e_eag, 2e-3 * mx)
    assert torch.isfinite(o).all() and e_nat <= e_mrg + bar, (e_nat, e_mrg, e_eag, mx)
    if merged32 is not None:          # the kernels on the merged weights: the plain section 7 bar
        assert e_nat_m <= bar, (e_nat_m, e_eag, mx)


def _oracles(cfg, sd, ip_sd, lora, factor, eager=True):
    from oracle import adapter_ref as A
    from oracle.unet_ref import UNetRef

    def oracle(device, dtype):
        with torch.device("meta"):
            ref = UNetRef(cfg)
        ref = ref.to_empty(device=device)
        ref.load_state_dict({k: v.to(device=device, dtype=dtype) for k, v in sd.items()})
        with torch.device("meta"):
            pr = A.install_processors(ref, cfg)
        for p in pr.values():
            p.to_empty(device=device)
        torch.nn.ModuleList(pr.values()).load_state_dict({k: v.to(device=device, dtype=dtype) for k, v in ip_sd.items()})
        attach_unfused(ref, lora, factor)
        return ref.to(dtype).eval()
    return oracle("cpu", torch.float32), (oracle("cuda", torch.float16) if eager else None)


def test_parity_with_unfused_forward_tiny_and_trajectory():
    from imagharmony_b200.config import TINY
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.lora import LoraWeights, term_factor
    from oracle.scheduler_ref import denoise_loop, euler_tables, prepare_latents
    native, sd, ip_sd = _tiny_native(4)
    lora = _unet_lora(native, rank=64, seed=5)
    lw = LoraWeights(native, {})
    lw.add("a", to_kohya(lora, "unet"))
    lw.sync("unet", {"a": (1.0, 1.0)})
    factor = lambda alpha, r: term_factor(1.0, 1.0, alpha, r)  # noqa: E731
    ref32, eager16 = _oracles(TINY, sd, ip_sd, lora, factor)
    x = _inputs(TINY, 1, 32)
    _parity("lora unet tiny", native, ref32, eager16, x, 500.0)
    T, n = 4, 1
    _, _, ins = euler_tables(T)
    latents = prepare_latents(n, 4, 32, 32, [42], ins)
    _, ehs, te, tid = x

    def run_oracle(m, dev, dt):
        procs = [p for p in m.attn_processors.values() if hasattr(p, "to_k_ip")]

        def set_scale(sc):
            for p in procs:
                p.scale = sc
        fn = lambda s_, t_, e_, te_, ti_: m(s_.to(dt), t_, e_, te_, ti_).to(torch.float16)  # noqa: E731
        with torch.no_grad():
            return denoise_loop(fn, latents.to(dev), ehs[1:].to(dev, dt), ehs[:1].to(dev, dt), te[1:].to(dev, dt),
                                te[:1].to(dev, dt), tid[:1].to(dev), T, guidance_scale=5.0, set_scale=set_scale,
                                conditioning_scale=1.0)
    r4, e4 = run_oracle(ref32, "cpu", torch.float32).float().cpu(), run_oracle(eager16, "cuda", torch.float16).float().cpu()
    o4 = DenoiseEngine(native).run(latents, ehs[1:], ehs[:1], te[1:], te[:1], tid[:1], T, guidance_scale=5.0,
                                   ip_scale=1.0).float().cpu()
    e_nat, e_eag, mx = (o4 - r4).abs().max().item(), (e4 - r4).abs().max().item(), r4.abs().max().item()
    print(f"[lora tiny trajectory] native {e_nat:.3e} eager-fp16 {e_eag:.3e} max|ref| {mx:.3e}")
    assert e_nat <= max(2.0 * e_eag, 2e-3 * mx), (e_nat, e_eag, mx)


@pytest.fixture(scope="module")
def sdxl_lora():
    """SDXL-base (random init) with a full-coverage rank-64 LoRA whose deltas are about 0.1 |W|."""
    from imagharmony_b200.config import SDXL_BASE as cfg
    from imagharmony_b200.lora import LoraWeights
    from imagharmony_b200.unet import UNet2DConditionModel
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from oracle.unet_ref import UNetRef
    with torch.device("meta"):
        shapes = shapes_of(UNetRef(cfg))
    sd = random_state_dict(shapes, 0, device="cuda")
    native = UNet2DConditionModel.from_state_dict(cfg, sd, device="cuda")
    procs = torch.nn.ModuleList(native.attn_processors.values())
    ip_sd = random_state_dict(shapes_of(procs), 1, device="cuda")
    procs.load_state_dict(ip_sd)
    native.finalize()
    lora = _unet_lora(native, rank=64, seed=6)
    lw = LoraWeights(native, {})
    yield cfg, native, sd, ip_sd, lora, lw
    del native, sd, lw
    torch.cuda.empty_cache()


def test_census_step_ops_unchanged_with_lora(ops, sdxl_lora, monkeypatch):  # noqa: F811
    """One SDXL-base 1024^2 CFG forward calls the identical op list (tests/census.py: every op, keyed by op, tensor
    shapes / strides / dtypes, flags and the execution plan, in first-call order with call counts), each key within its
    bar on the LoRA-merged weights, and a graph-replayed step launches as many kernels, with and without a LoRA."""
    from imagharmony_b200.denoise import DenoiseEngine
    cfg, native, _, _, lora, lw = sdxl_lora
    x = _inputs(cfg, 1, 128)

    def record(title):
        c = census.Census(ops, check_all=False, plan=plan).install(monkeypatch)
        s, e, te, tid = (v.cuda() for v in x)
        with torch.no_grad():
            native(s, torch.full((2,), 500.0, device="cuda"), e, te, tid)
        monkeypatch.undo()
        torch.cuda.synchronize()
        print("\n" + c.report(title))
        bad = c.failures()
        assert not bad, [(r["op"], r["shape"], r["worst"]) for r in bad]
        _, e, te, tid = x
        eng = DenoiseEngine(native)
        lat = torch.randn(1, 4, 128, 128, generator=torch.Generator().manual_seed(0)).half()
        eng.run(lat, e[1:], e[:1], te[1:], te[:1], tid[:1], 1, guidance_scale=5.0, ip_scale=1.0)
        torch.cuda.synchronize()
        return [(k, r["calls"]) for k, r in c.rows.items()], eng.last_launches_per_step
    base_ops, base_launches = record("SDXL-base 1024^2 CFG, no LoRA")
    lw.add("census", to_kohya(lora, "unet"))
    try:
        lw.sync("unet", {"census": (1.0, 1.0)})
        lora_ops, lora_launches = record("SDXL-base 1024^2 CFG, rank-64 LoRA merged")
    finally:
        lw.sync("unet", {})
        lw.remove("census")
        lw.release()
    print(f"[lora census] {sum(n for _, n in base_ops)} op calls, {base_launches} launches per step")
    assert lora_ops == base_ops and lora_launches == base_launches > 0


def test_parity_with_unfused_forward_sdxl_base_512(sdxl_lora):
    from imagharmony_b200.lora import term_factor
    cfg, native, sd, ip_sd, lora, lw = sdxl_lora
    lw.add("parity", to_kohya(lora, "unet"))
    lw.sync("unet", {"parity": (1.0, 1.0)})
    ref32, eager16 = _oracles(cfg, sd, ip_sd, lora, lambda alpha, r: term_factor(1.0, 1.0, alpha, r))
    merged = {k: v for k, v in native.state_dict().items() if ".processor." not in k}
    merged32, _ = _oracles(cfg, merged, ip_sd, {}, None, eager=False)
    try:
        _parity("lora unet SDXL-base 512^2 B2", native, ref32, eager16, _inputs(cfg, 1, 64, seed=13), 601.0, merged32)
    finally:
        del ref32, eager16, merged32
        lw.sync("unet", {})
        lw.remove("parity")
        lw.release()


@pytest.mark.parametrize("name,with_proj", [("TEXT_L", False), ("TEXT_BIGG", True)])
def test_text_tower_with_lora_matches_transformers(name, with_proj):
    from imagharmony_b200.clip import ClipTextTower
    from imagharmony_b200.lora import LoraWeights, TE2, term_factor, text_name_table
    from oracle import clip_ref as R
    kw = getattr(R, name)
    hf = R.hf_text_model(11, with_proj, **kw)
    tower = ClipTextTower.from_hf(hf, device="cuda")
    lora = random_lora(module_shapes(hf, text_name_table(kw["num_hidden_layers"])), 32, 4, rel=0.1, alpha=16)
    native, _, _ = _tiny_native()
    lw = LoraWeights(native, {TE2: tower})
    lw.add("t", to_kohya(lora, TE2))
    lw.sync(TE2, {"t": (0.8, 1.0)})
    attach_unfused(hf, lora, lambda alpha, r: term_factor(0.8, 1.0, alpha, r))
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(0, 49406, (2, 77), generator=g)
    ids[0, 9:], ids[1, 17:] = 49407, 49407
    with torch.no_grad():
        want = hf(ids, output_hidden_states=True).hidden_states[-2]
        eag = hf.half().cuda()(ids.cuda(), output_hidden_states=True).hidden_states[-2]
    got = tower(ids).penultimate
    torch.cuda.synchronize()
    err, e_eag, mx = ((got.float().cpu() - want).abs().max().item(), (eag.float().cpu() - want).abs().max().item(),
                      want.abs().max().item())
    print(f"[lora {name} hidden_states[-2]] native {err:.3e} hf-fp16 {e_eag:.3e} max|ref| {mx:.3e}")
    assert err <= max(2.0 * e_eag, 2e-3 * mx), (err, e_eag, mx)


def _ip_model(pipe):
    from imagharmony_b200.weights import random_state_dict, shapes_of
    from ip_adapter import IPAdapterXL
    ip = IPAdapterXL(pipe, None, None, "cuda", num_tokens=4, inference=True)
    ip.image_proj_model.load_state_dict({k: v.cuda() for k, v in random_state_dict(shapes_of(ip.image_proj_model), 3).items()})
    procs = torch.nn.ModuleList(pipe.unet.attn_processors.values())
    procs.load_state_dict({k: v.cuda() for k, v in random_state_dict(shapes_of(procs), 5).items()})
    pipe.unet.finalize()
    return ip


def _generate(ip, **kw):
    img = torch.randn(1, ip.pipe.unet.config.pooled_embed_dim, generator=torch.Generator("cpu").manual_seed(5)).half()
    return ip.generate(pil_image=None, clip_image_embeds=img, prompt="lions", negative_prompt="blurry", scale=0.8,
                       num_samples=1, num_inference_steps=3, seed=[42], output_type="latent", height=256, width=256, **kw)


def test_ip_adapter_generate_with_lora():
    from imagharmony_b200.config import TINY
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    pipe = StableDiffusionXLCustomPipeline.from_random(TINY, seed=4)
    sd = to_peft(_unet_lora(pipe.unet, seed=8), "unet")
    ip = _ip_model(pipe)
    base = _generate(ip)
    ip.pipe.load_lora_weights(sd, adapter_name="style")
    zero = _generate(ip, cross_attention_kwargs={"scale": 0.0})
    half = _generate(ip, cross_attention_kwargs={"scale": 0.6})
    full_after = _generate(ip)
    ip.pipe.set_adapters(["style"], [0.6])
    half_w = _generate(ip)
    torch.cuda.synchronize()
    assert torch.equal(zero, base) and torch.equal(half, half_w) and not torch.equal(half, base)
    # loading before building the adapter gives the same latents as loading after it
    pipe2 = StableDiffusionXLCustomPipeline.from_random(TINY, seed=4)
    pipe2.load_lora_weights(sd, adapter_name="style")
    full_before = _generate(_ip_model(pipe2))
    torch.cuda.synchronize()
    assert torch.equal(full_before, full_after)


def test_controlnet_pipeline_with_lora_leaves_controlnet_weights():
    from imagharmony_b200.config import TINY, TINY_CONTROLNET
    from ip_adapter.custom_pipelines import StableDiffusionXLControlNetPipeline
    pipe = StableDiffusionXLControlNetPipeline.from_random(TINY, TINY_CONTROLNET, seed=0)
    before = {k: v.clone() for k, v in pipe.controlnet.state_dict().items()}
    img = torch.rand(1, 3, 256, 256, generator=torch.Generator().manual_seed(0))
    gen = torch.Generator("cpu").manual_seed(9)
    D, P = TINY.cross_attention_dim, TINY.pooled_embed_dim
    emb = dict(prompt_embeds=torch.randn(1, 77, D, generator=gen).half(),
               negative_prompt_embeds=torch.randn(1, 77, D, generator=gen).half(),
               pooled_prompt_embeds=torch.randn(1, P, generator=gen).half(),
               negative_pooled_prompt_embeds=torch.randn(1, P, generator=gen).half())
    run = lambda **kw: pipe(image=img, num_inference_steps=3, generator=torch.Generator("cuda").manual_seed(3),  # noqa: E731
                            output_type="latent", **emb, **kw).images
    r0 = run()
    pipe.load_lora_weights(to_kohya(_unet_lora(pipe.unet, seed=9), "unet"))
    r1 = run(cross_attention_kwargs={"scale": 0.5})
    torch.cuda.synchronize()
    assert torch.isfinite(r1).all() and not torch.equal(r0, r1)
    assert all(torch.equal(v, before[k]) for k, v in pipe.controlnet.state_dict().items())
