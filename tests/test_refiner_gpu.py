"""GPU tests of the SDXL refiner: the native refiner UNet (TINY_REFINER and the full-size refiner at 1024^2) against the
fp32 oracle (tests/refiner_ref.py) with test_unet_gpu.py's bar, the graph-replayed image-to-image handoff against eager
and the restated trajectory, and the base -> refiner ensemble end to end at 1024^2 with random weights."""
import pytest
import torch

from refiner_ref import begin_step_ref, ensemble_loop, unet_ref

pytestmark = pytest.mark.gpu


def _make_pair(cfg, seed=0):
    """(native unet on cuda fp16, oracle on cpu fp32, oracle on cuda fp16) with identical parameters."""
    from imagharmony_b200.unet import UNet2DConditionModel
    from imagharmony_b200.weights import random_state_dict, shapes_of
    with torch.device("meta"):
        shapes = shapes_of(unet_ref(cfg))
    sd = random_state_dict(shapes, seed)
    native = UNet2DConditionModel.from_state_dict(cfg, sd, device="cuda")

    def oracle(device, dtype):
        m = unet_ref(cfg)
        m.load_state_dict({k: v.float() for k, v in sd.items()})
        return m.to(device=device, dtype=dtype).eval()
    return native, oracle("cpu", torch.float32), oracle("cuda", torch.float16)


def _inputs(cfg, B, lat, seed):
    g = torch.Generator("cpu").manual_seed(seed)
    res = lat * 8.0
    return (torch.randn(B, 4, lat, lat, generator=g).half(),
            torch.randn(B, 77, cfg.cross_attention_dim, generator=g).half(),
            torch.randn(B, cfg.pooled_embed_dim, generator=g).half(),
            torch.tensor([[res, res, 0.0, 0.0, 2.5]] * (B // 2) + [[res, res, 0.0, 0.0, 6.0]] * (B - B // 2)))


def _check(tag, native_out, r, e):
    ref = r.float().cpu()
    e_nat = (native_out.float().cpu() - ref).abs().max().item()
    e_eag = (e.float().cpu() - ref).abs().max().item()
    mx = ref.abs().max().item()
    rms = lambda a: ((a.float().cpu() - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()  # noqa: E731
    print(f"[{tag}] native max|err| {e_nat:.3e} rel-RMS {rms(native_out):.3e} | eager-fp16 max|err| {e_eag:.3e} "
          f"rel-RMS {rms(e):.3e} | max|ref| {mx:.3e}")
    assert torch.isfinite(native_out).all()
    assert e_nat <= max(2.0 * e_eag, 2e-3 * mx), (e_nat, e_eag, mx)
    assert rms(native_out) <= max(2.0 * rms(e), 1e-3)


@pytest.mark.parametrize("which,lat,t", [("TINY_REFINER", 32, 500.0), ("SDXL_REFINER", 128, 181.0)])
def test_refiner_forward_matches_oracle(which, lat, t):
    from imagharmony_b200 import config
    cfg = getattr(config, which)
    native, ref32, eager16 = _make_pair(cfg)
    x, ehs, te, tid = _inputs(cfg, 2, lat, 17)
    with torch.no_grad():
        r = ref32(x.float(), t, ehs.float(), te.float(), tid)
        e = eager16(x.cuda(), t, ehs.cuda(), te.cuda(), tid.cuda())
        o = native(x.cuda(), torch.full((2,), t, device="cuda"), ehs.cuda(), te.cuda(), tid.cuda())
    torch.cuda.synchronize()
    _check(f"{which} forward {8 * lat}^2 B2", o, r, e)


def test_refiner_handoff_graph_replay_matches_eager_and_restated_loop():
    from imagharmony_b200.config import TINY_REFINER as cfg
    from ip_adapter.custom_pipelines import StableDiffusionXLImg2ImgPipeline
    pipe = StableDiffusionXLImg2ImgPipeline.from_random(cfg, seed=5, device="cuda")
    T, d, gs, lat = 8, 0.7, 5.0, 32
    k = begin_step_ref(T, d)
    g = torch.Generator("cpu").manual_seed(2)
    start = (torch.randn(1, 4, lat, lat, generator=g) * 3).half()
    pe, ne = (torch.randn(1, 77, cfg.cross_attention_dim, generator=g).half() for _ in "ab")
    pp, npool = (torch.randn(1, cfg.pooled_embed_dim, generator=g).half() for _ in "ab")
    kw = dict(prompt_embeds=pe, negative_prompt_embeds=ne, pooled_prompt_embeds=pp, negative_pooled_prompt_embeds=npool,
              image=start.cuda(), num_inference_steps=T, denoising_start=d, guidance_scale=gs, output_type="latent")
    graph = pipe(**kw).images
    assert pipe.engine.use_cuda_graph and pipe.engine.graphs_captured > 0
    pipe.engine.use_cuda_graph = False
    eager = pipe(**kw).images
    torch.cuda.synchronize()
    assert torch.equal(graph, eager), (graph.float() - eager.float()).abs().max()

    _, ref32, eager16 = _make_pair(cfg, seed=0)
    ref32.load_state_dict({n: v.float().cpu() for n, v in pipe.unet.state_dict().items()})
    eager16.load_state_dict({n: v.cuda() for n, v in pipe.unet.state_dict().items()})
    tid = torch.tensor([[256.0, 256.0, 0.0, 0.0, 2.5], [256.0, 256.0, 0.0, 0.0, 6.0]])

    def restated(m, dev, dt):
        cond = (torch.cat([ne, pe]).to(dev, dt), torch.cat([npool, pp]).to(dev, dt), tid.to(dev))
        fn = lambda s_, t_, e_, te_, ti_: m(s_.to(dt), t_, e_, te_, ti_).to(torch.float16)  # noqa: E731
        return ensemble_loop(fn, cond, fn, cond, k, start.to(dev), T, gs, begin=k)
    _check(f"refiner handoff TINY, steps {k}..{T}", graph, restated(ref32, "cpu", torch.float32),
           restated(eager16, "cuda", torch.float16))


def test_ensemble_end_to_end_1024():
    """IPAdapterXL.generate on the base with denoising_end=0.8, output_type="latent", then the refiner's image-to-image
    with denoising_start=0.8 on those latents: random weights, finite latents of the right shape."""
    from imagharmony_b200.config import SDXL_BASE, SDXL_REFINER
    from ip_adapter import IPAdapterXL
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline, StableDiffusionXLImg2ImgPipeline
    base = StableDiffusionXLCustomPipeline.from_random(SDXL_BASE, seed=0, device="cuda")
    ip = IPAdapterXL(base, None, None, "cuda", num_tokens=4)
    emb = torch.randn(1, SDXL_BASE.pooled_embed_dim, generator=torch.Generator().manual_seed(1))
    mid = ip.generate(clip_image_embeds=emb, prompt="eight sheep", num_samples=1, seed=3, num_inference_steps=10,
                      denoising_end=0.8, output_type="latent", height=1024, width=1024)
    assert mid.shape == (1, 4, 128, 128) and torch.isfinite(mid.float()).all()
    refiner = StableDiffusionXLImg2ImgPipeline.from_random(SDXL_REFINER, seed=1, device="cuda")
    out = refiner(prompt="eight sheep", image=mid, denoising_start=0.8, num_inference_steps=10,
                  generator=torch.Generator().manual_seed(3), output_type="latent").images
    torch.cuda.synchronize()
    assert out.shape == (1, 4, 128, 128) and torch.isfinite(out.float()).all()
    assert not torch.equal(out, mid)
    assert refiner.engine.last_launches_per_step > 0
