"""DenoiseEngine.run refuses an invalid call before it does any work: no kernel launch, no new static buffer and no new
cross-attention K/V buffer, for every option clash and every range and shape check, at a shape the engine has not
seen.  A refused call therefore leaves nothing behind that a later call or a captured graph could depend on."""
import dataclasses

import pytest
import torch

from test_controlnet_cpu import _image
from test_multi_controlnet_cpu import _pipe, mcp  # noqa: F401  (fixture)
from test_wiring_cpu import _Empty32, _inputs, patched  # noqa: F401  (fixture)

# option -> the options it cannot be combined with
EXCLUDES = {
    "dpm": ("begin_step", "inpaint", "unet_cond", "start_step", "stop_after"),
    "unet_cond": ("inpaint", "start_step", "stop_after"),
    "controlnet": ("begin_step", "inpaint", "unet_cond", "start_step", "stop_after"),
    "inpaint": ("start_step", "stop_after"),
    "begin_step": ("start_step", "stop_after"),
}


def _kv_buffers(models):
    """(attention module, processor, buffer key) of every K/V buffer the models' processors hold."""
    keys = set()
    for m in models:
        for name, p in m.attn_processors.items():
            for q in [p] + list(getattr(p, "_text", {}).values()):     # a ControlNet's per-module text processors
                keys |= {(name, id(q), k) for k in getattr(q, "_kv_bufs", {})}
    return keys


def _refused_calls(T, n, lat, nets):
    """(scheduler, run keywords, words the message must contain) of every call run refuses."""
    from imagharmony_b200.config import TINY_CONTROLNET
    from imagharmony_b200.controlnet import ControlNetCall, ControlNetModel
    x, mask = torch.zeros(n, 4, lat, lat), torch.zeros(n, 1, lat, lat)
    img = _image(n, 8 * lat)
    a, b = (ControlNetCall(m, img, 1.0, False) for m in nets)
    value = {"begin_step": 1, "inpaint": (x, x, mask), "unet_cond": (mask, x), "start_step": 1, "stop_after": 2,
             "controlnet": [a, b]}
    calls = []
    for option, excluded in EXCLUDES.items():
        for other in excluded:
            if option == "dpm":
                calls.append(("dpm", {other: value[other]}, "EulerAncestralDiscreteScheduler"))
            else:
                calls.append(("euler", {option: value[option], other: value[other]}, option))
    with torch.device("meta"):
        wide = ControlNetModel(dataclasses.replace(TINY_CONTROLNET, block_out_channels=(64, 128, 128)))
    calls += [
        ("euler", dict(negative_prompt_embeds=None), "negative"),
        ("euler", dict(num_loop_steps=0), "num_loop_steps"),
        ("euler", dict(num_loop_steps=T + 1), "num_loop_steps"),
        ("euler", dict(start_step=-1), "start_step"),
        ("euler", dict(start_step=T + 1), "start_step"),
        ("euler", dict(begin_step=-1), "begin_step"),
        ("euler", dict(begin_step=T), "begin_step"),
        ("euler", dict(inpaint=(x, x, x)), "mask"),
        ("euler", dict(unet_cond=(mask, x)), "9-channel"),
        ("euler_a", dict(generator=[torch.Generator()] * (n + 1)), "generators"),
        ("euler", dict(controlnet=[]), "1 .. 8"),
        ("euler", dict(controlnet=[a] * 9), "1 .. 8"),
        ("euler", dict(controlnet=[a, ControlNetCall(b.model, img, 1.0, True)]), "guess_mode"),
        ("euler", dict(controlnet=[a, ControlNetCall(wide, img, 1.0, False)]), "block_out_channels"),
        ("euler", dict(controlnet=ControlNetCall(a.model, img, 1.0, False, [1.0] * (T - 1))), "keep"),
        ("euler", dict(controlnet=[a, ControlNetCall(b.model, _image(n, 8 * lat + 8), 1.0, False)]), "image"),
        ("euler", dict(latents=torch.zeros(n, 4, lat + 2, lat)), "latent size"),    # the stride-2 convs need h % 4 == 0
    ]
    return calls


def test_refused_calls_do_no_work(mcp):  # noqa: F811
    from imagharmony_b200 import ops
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.controlnet import ControlNetCall
    from imagharmony_b200.denoise import DenoiseEngine
    from imagharmony_b200.scheduler import (DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler,
                                            EulerDiscreteScheduler)
    pipe = _pipe(2)
    models = [pipe.unet] + list(pipe.controlnet.nets)
    T, n, lat = 4, 1, 8
    latents, ehs, te, tid = _inputs(pipe.unet.config, n, lat)
    args = dict(latents=latents[:n], prompt_embeds=ehs[n:, :77], negative_prompt_embeds=ehs[:n, :77],
                pooled=te[n:], negative_pooled=te[:n], time_ids=tid[:n], num_inference_steps=T)
    schedulers = {"euler": EulerDiscreteScheduler, "euler_a": EulerAncestralDiscreteScheduler,
                  "dpm": DPMSolverMultistepScheduler}
    engines = {k: DenoiseEngine(pipe.unet, use_cuda_graph=False, scheduler=s()) for k, s in schedulers.items()}
    calls = _refused_calls(T, n, lat, pipe.controlnet.nets)
    assert len(calls) == sum(len(v) for v in EXCLUDES.values()) + 17
    kv = _kv_buffers(models)
    for kind, kw, words in calls:
        eng = engines[kind]
        launches = ops.launch_count()
        with pytest.raises(IHError, match=words):
            eng.run(**{**args, **kw})
        assert ops.launch_count() == launches, (kind, list(kw))
        assert not eng._pool and not eng._schedules, (kind, list(kw))
        assert _kv_buffers(models) == kv, (kind, list(kw))

    # a valid call at that shape does all three kinds of work, so the checks above would see it
    launches = ops.launch_count()
    with _Empty32():
        engines["euler"].run(**args, controlnet=ControlNetCall(pipe.controlnet.nets[0], _image(n, 8 * lat), 1.0, False))
    assert ops.launch_count() > launches and engines["euler"]._pool and _kv_buffers(models) > kv


@pytest.mark.parametrize("height,width,error", [(1001, 1024, ValueError), (1000, 1000, "IHError"),
                                                (1016, 1024, "IHError")])
def test_pipeline_refuses_sizes_the_unet_cannot_run(patched, height, width, error):  # noqa: F811
    """Text-to-image at a size that is not a multiple of 8 is a ValueError (as diffusers' check_inputs), and at a
    multiple of 8 that is not one of 32 (the UNet's two stride-2 convs halve the latent twice) an IHError from the
    engine, before it launches anything or allocates a static buffer."""
    from imagharmony_b200 import ops
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.config import TINY
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    pipe = StableDiffusionXLCustomPipeline.from_random(TINY, seed=0, device="cpu")
    pe, pooled = torch.randn(1, 81, TINY.cross_attention_dim).half(), torch.randn(1, TINY.pooled_embed_dim).half()
    launches = ops.launch_count()
    with pytest.raises(IHError if error == "IHError" else error, match="divisible by"):
        pipe(prompt_embeds=pe, negative_prompt_embeds=pe, pooled_prompt_embeds=pooled,
             negative_pooled_prompt_embeds=pooled, num_inference_steps=4, output_type="latent", height=height,
             width=width)
    assert ops.launch_count() == launches
    assert not pipe.engine._pool and not pipe.engine._schedules
