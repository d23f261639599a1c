"""CPU tests of LoRA loading and merging (imagharmony_b200/lora.py and the pipeline surface): the SGM <-> diffusers name
table, the kohya / PEFT key formats and the refused ones, the conv (LoCon) delta, the adapter state machine against the
fp64 merge, and PEFT's unfused forward (tests/lora_ref.py) on the oracle UNet and transformers' CLIP text models against
the merged native models, all on the plain-PyTorch stand-in ops."""
import pytest
import torch

from lora_ref import attach_unfused, merged64, module_shapes, random_lora, to_kohya, to_peft
from test_wiring_cpu import _build, _inputs, patched  # noqa: F401  (fixture)


def _targetable(model):
    """Linear / Conv2d modules a LoRA may target, found independently of lora.py: every one outside conv_in, conv_out,
    the time / added embeddings and the attention processors."""
    skip = ("conv_in", "conv_out", "time_embedding.", "add_embedding.")
    return {n for n, m in model.named_modules() if isinstance(m, (torch.nn.Linear, torch.nn.Conv2d))
            and not n.startswith(skip) and ".processor" not in n}


@pytest.mark.parametrize("name", ["TINY", "SDXL_BASE", "SDXL_REFINER"])
def test_name_table_is_a_bijection_onto_targetable_modules(name):
    import imagharmony_b200.config as C
    from imagharmony_b200.lora import unet_name_table
    from imagharmony_b200.unet import UNet2DConditionModel
    with torch.device("meta"):
        m = UNet2DConditionModel(getattr(C, name))
    table = unet_name_table(m)
    assert set(table) == _targetable(m)
    assert len(set(table.values())) == len(table)
    flat = {s.replace(".", "_") for s in table.values()} | {n.replace(".", "_") for n in table}
    assert len(flat) == 2 * len(table)
    if name == "SDXL_BASE":
        want = {
            "down_blocks.0.resnets.1.conv1": "input_blocks.2.0.in_layers.2",
            "down_blocks.0.downsamplers.0.conv": "input_blocks.3.0.op",
            "down_blocks.1.resnets.0.conv_shortcut": "input_blocks.4.0.skip_connection",
            "down_blocks.1.attentions.1.transformer_blocks.1.attn2.to_k": "input_blocks.5.1.transformer_blocks.1.attn2.to_k",
            "down_blocks.1.downsamplers.0.conv": "input_blocks.6.0.op",
            "down_blocks.2.attentions.0.proj_in": "input_blocks.7.1.proj_in",
            "mid_block.resnets.0.time_emb_proj": "middle_block.0.emb_layers.1",
            "mid_block.attentions.0.transformer_blocks.9.ff.net.0.proj": "middle_block.1.transformer_blocks.9.ff.net.0.proj",
            "mid_block.resnets.1.conv2": "middle_block.2.out_layers.3",
            "up_blocks.0.attentions.2.transformer_blocks.0.attn1.to_out.0": "output_blocks.2.1.transformer_blocks.0.attn1.to_out.0",
            "up_blocks.0.upsamplers.0.conv": "output_blocks.2.2.conv",
            "up_blocks.1.resnets.0.conv_shortcut": "output_blocks.3.0.skip_connection",
            "up_blocks.1.upsamplers.0.conv": "output_blocks.5.2.conv",
            "up_blocks.2.resnets.2.conv2": "output_blocks.8.0.out_layers.3",
        }
        assert {k: table[k] for k in want} == want
    if name == "SDXL_REFINER":      # an attention-free last level: its upsampler is the block's second module
        assert table["up_blocks.0.upsamplers.0.conv"] == "output_blocks.2.1.conv"
        assert table["down_blocks.3.resnets.1.conv2"] == "input_blocks.11.0.out_layers.3"
        assert "down_blocks.3.downsamplers.0.conv" not in table


# ---------------------------------------------------------------------------------------------------------------------
# loader
# ---------------------------------------------------------------------------------------------------------------------
def _towers():
    from imagharmony_b200.clip import ClipTextTower, ClipTowerConfig
    from oracle.clip_ref import hf_text_model
    kw = dict(vocab_size=100, eos_token_id=99, hidden_size=64, intermediate_size=128, num_hidden_layers=2,
              num_attention_heads=2)
    hf1 = hf_text_model(3, False, hidden_act="quick_gelu", **kw)
    hf2 = hf_text_model(4, True, hidden_act="gelu", projection_dim=64, **kw)
    # towers from copies: an fp32 CPU tower would otherwise share the HF model's tensors, and a merge would change both
    return hf1, hf2, *(ClipTextTower(ClipTowerConfig.from_hf(m.config), {k: v.clone() for k, v in m.state_dict().items()},
                                     device="cpu") for m in (hf1, hf2))


def _tiny_unet(seed=0, dtype=torch.float16):
    from imagharmony_b200.config import TINY
    from imagharmony_b200.unet import UNet2DConditionModel
    from imagharmony_b200.weights import random_state_dict, shapes_of
    with torch.device("meta"):
        m = UNet2DConditionModel(TINY)
    m.load_state_dict({k: v.to(dtype) for k, v in random_state_dict(shapes_of(m), seed).items()}, assign=True)
    m.requires_grad_(False)
    m.install_default_processors()
    m.finalize()
    return m


def _random_loras(unet, t1=None, t2=None, rank=4, seed=0):
    from imagharmony_b200.lora import text_name_table, unet_name_table
    out = {"unet": random_lora(module_shapes(unet, unet_name_table(unet)), rank, seed, alpha=rank / 2)}
    for comp, hf, s in (("text_encoder", t1, 1), ("text_encoder_2", t2, 2)):
        if hf is not None:
            names = text_name_table(hf.config.num_hidden_layers)
            out[comp] = random_lora(module_shapes(hf, names), rank, seed + s, alpha=rank)
    return out


def test_three_formats_load_identically(patched):  # noqa: F811
    from imagharmony_b200.lora import LoraWeights, parse_lora, unet_name_table
    unet = _tiny_unet()
    hf1, hf2, t1, t2 = _towers()
    lw = LoraWeights(unet, {"text_encoder": t1, "text_encoder_2": t2})
    loras = _random_loras(unet, hf1, hf2)
    sgm = unet_name_table(unet)
    forms = [
        {**to_kohya(loras["unet"], "unet", sgm), **to_kohya(loras["text_encoder"], "text_encoder"),
         **to_kohya(loras["text_encoder_2"], "text_encoder_2")},
        {**to_kohya(loras["unet"], "unet"), **to_kohya(loras["text_encoder"], "text_encoder"),
         **to_kohya(loras["text_encoder_2"], "text_encoder_2")},
        {k: v for c in loras for k, v in to_peft(loras[c], c).items()},
    ]
    parsed = [parse_lora(sd, lw.tables, lw.targets) for sd in forms]
    for comp, mods in loras.items():
        assert set(parsed[0][comp]) == set(mods)
        for p in parsed:
            for n, (up, down, alpha) in mods.items():
                u, d, a = p[comp][n]
                assert a == alpha and torch.equal(u, up.reshape(u.shape)) and torch.equal(d, down.reshape(d.shape))


_GOOD = "lora_unet_input_blocks_4_1_transformer_blocks_0_attn1_to_q"


@pytest.mark.parametrize("bad", [
    {"lora_unet_input_blocks_4_1_proj_in.hada_w1_a": 1}, {"lora_unet_input_blocks_4_1_proj_in.lokr_w1": 1},
    {_GOOD + ".dora_scale": 1}, {"lora_unet_input_blocks_1_0_in_layers_2.lora_mid.weight": 1},
    {"lora_unet_input_blocks_4_1_proj_in.diff": 1}, {"lora_unet_input_blocks_4_1_proj_in.diff_b": 1},
    {"down_blocks.1.attentions.0.transformer_blocks.0.attn1.processor.to_q_lora.down.weight": 1},
    {"lora_unet_conv_in.lora_down.weight": 1, "lora_unet_conv_in.lora_up.weight": 1},
    {"unet.time_embedding.linear_1.lora_A.weight": 1, "unet.time_embedding.linear_1.lora_B.weight": 1},
    {"lora_unet_input_blocks_4_1_norm.lora_down.weight": 1},
    {"unet.up_blocks.0.attentions.0.transformer_blocks.0.norm1.lora_A.weight": 1},
    {"lora_te1_text_model_encoder_layers_0_mlp_fc1.lora_down.weight": 1},          # the refiner has no tower 1
    {"lora_unet_" + "input_blocks_4_1_transformer_blocks_0_attn1_to_k.lora_down.weight": torch.zeros(4, 7)},  # shape
])
def test_refused_formats_raise_and_leave_weights_untouched(patched, bad):  # noqa: F811
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.lora import LoraWeights, unet_name_table
    unet = _tiny_unet()
    _, hf2, _, t2 = _towers()
    lw = LoraWeights(unet, {"text_encoder_2": t2})
    good = to_kohya(_random_loras(unet)["unet"], "unet", unet_name_table(unet))
    bad = {k: (v if isinstance(v, torch.Tensor) else torch.zeros(4, 4)) for k, v in bad.items()}
    before = {k: v.clone() for k, v in unet.state_dict().items()}
    epoch = unet.graph_epoch
    with pytest.raises(IHError) as e:
        lw.add("x", {**good, **bad})
    assert next(iter(bad)) in str(e.value)
    assert not lw.adapters and not lw.orig and unet.graph_epoch == epoch
    assert all(torch.equal(v, before[k]) for k, v in unet.state_dict().items())


def test_conv_delta_is_the_composition(patched):  # noqa: F811
    """A LoCon term on a 3x3 conv (and the 1x1 shortcut) changes the conv by exactly F.conv2d(x, down) then the 1x1 up."""
    import torch.nn.functional as F
    from imagharmony_b200.lora import LoraWeights, unet_name_table
    unet = _tiny_unet(dtype=torch.float32)
    names = ["down_blocks.1.resnets.0.conv1", "down_blocks.1.resnets.0.conv_shortcut", "down_blocks.0.downsamplers.0.conv"]
    lora = random_lora(module_shapes(unet, names), 8, 5, rel=1.0, alpha=4)
    lw = LoraWeights(unet, {})
    mods = dict(unet.named_modules())
    orig = {n: mods[n].weight.detach().clone() for n in names}
    lw.add("a", to_kohya(lora, "unet", unet_name_table(unet)))
    lw.sync("unet", {"a": (1.0, 1.0)})
    g = torch.Generator().manual_seed(0)
    for n in names:
        m, (up, down, alpha) = mods[n], lora[n]
        x = torch.randn(2, m.in_channels, 9, 9, generator=g).double()
        got = F.conv2d(x, (m.weight - orig[n]).double(), None, m.stride, m.padding)
        want = 0.5 * F.conv2d(F.conv2d(x, down.double(), None, m.stride, m.padding), up.double())
        assert torch.allclose(got, want, rtol=1e-5, atol=1e-5 * want.abs().max().item()), (n, (got - want).abs().max())


# ---------------------------------------------------------------------------------------------------------------------
# state machine
# ---------------------------------------------------------------------------------------------------------------------
class _Tok:
    """Stand-in tokenizer: the prompt's characters as ids below the toy vocabulary's end token 99, then 99s."""
    model_max_length = 77

    def __call__(self, prompts, padding=None, max_length=77, truncation=True, return_tensors="pt"):
        from types import SimpleNamespace
        ids = torch.full((len(prompts), max_length), 99, dtype=torch.long)
        for i, p in enumerate(prompts):
            codes = [ord(c) % 98 for c in p][:max_length - 1]
            ids[i, :len(codes)] = torch.tensor(codes, dtype=torch.long)
        return SimpleNamespace(input_ids=ids)


def _pipe():
    from ip_adapter.custom_pipelines import StableDiffusionXLCustomPipeline
    from ip_adapter.encoders import ClipPromptEncoder
    unet = _tiny_unet()
    hf1, hf2, t1, t2 = _towers()
    pipe = StableDiffusionXLCustomPipeline(unet, prompt_encoder=ClipPromptEncoder(_Tok(), _Tok(), t1, t2, device="cpu"))
    return pipe, hf1, hf2


def _live(pipe):
    """{(component, module): tensor} of every weight a LoRA may touch."""
    from imagharmony_b200.lora import prompt_towers, tower_targets, unet_targets
    out = {("unet", n): t.live for n, t in unet_targets(pipe.unet).items()}
    for comp, tower in prompt_towers(pipe.prompt_encoder).items():
        out.update({(comp, n): t.live for n, t in tower_targets(tower).items()})
    return out


def _fp16_ulp(x):
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -14)))
    return torch.pow(2.0, e - 10)


def _check(pipe, base, loras, factors, what):
    """Every weight equals its original plus sum_k f_k up_k down_k (fp64) within one fp16 ulp per term; weights no term
    touches are bit-identical to their original."""
    from imagharmony_b200.lora import term_factor
    for key, live in _live(pipe).items():
        comp, mod = key
        terms = [(term_factor(s, w, loras[a][comp][mod][2], loras[a][comp][mod][1].shape[0]),) + loras[a][comp][mod][:2]
                 for a, (s, w) in factors.get(comp, {}).items() if mod in loras[a].get(comp, {})]
        terms = [t for t in terms if t[0] != 0.0]
        if not terms:
            assert torch.equal(live, base[key]), (what, key)
            continue
        want = merged64(base[key], terms)
        ulp = _fp16_ulp(want.abs() + sum(abs(f) * (u.double().reshape(u.shape[0], -1) @ d.double().reshape(d.shape[0], -1)).abs()
                                         for f, u, d in terms))
        err = (live.double().reshape(want.shape) - want).abs()
        assert bool((err <= len(terms) * ulp).all()), (what, key, (err / ulp).max().item())


def test_state_machine_matches_fp64_merge(patched, monkeypatch):  # noqa: F811
    from imagharmony_b200._lib import IHError
    from imagharmony_b200.lora import unet_name_table
    pipe, hf1, hf2 = _pipe()
    base = {k: v.clone() for k, v in _live(pipe).items()}
    ptrs = {k: v.data_ptr() for k, v in _live(pipe).items()}
    la = _random_loras(pipe.unet, hf1, hf2, rank=4, seed=0)
    lb = _random_loras(pipe.unet, None, hf2, rank=8, seed=7)
    lb["unet"] = {n: v for i, (n, v) in enumerate(lb["unet"].items()) if i % 2}   # B touches half the UNet, no tower 1
    loras = {"A": la, "B": lb}
    sd_a = {**to_kohya(la["unet"], "unet", unet_name_table(pipe.unet)), **to_kohya(la["text_encoder"], "text_encoder"),
            **to_kohya(la["text_encoder_2"], "text_encoder_2")}
    sd_b = {k: v for c in lb for k, v in to_peft(lb[c], c).items()}
    every = lambda f: {c: f for c in ("unet", "text_encoder", "text_encoder_2")}  # noqa: E731

    pipe.load_lora_weights(sd_a, adapter_name="A")
    assert pipe.get_active_adapters() == ["A"]
    _check(pipe, base, loras, every({"A": (1.0, 1.0)}), "load A")
    pipe.load_lora_weights(sd_b)
    assert pipe.get_active_adapters() == ["default_1"]
    loras["default_1"] = loras.pop("B")
    assert pipe.get_list_adapters() == {"unet": ["A", "default_1"], "text_encoder": ["A"],
                                        "text_encoder_2": ["A", "default_1"]}
    _check(pipe, base, loras, every({"default_1": (1.0, 1.0)}), "load B")
    pipe.set_adapters(["A", "default_1"], [0.5, -0.75])
    two = every({"A": (1.0, 0.5), "default_1": (1.0, -0.75)})
    _check(pipe, base, loras, two, "set_adapters")
    snap = {k: v.clone() for k, v in _live(pipe).items()}
    with pytest.raises(ValueError):
        pipe.set_adapters(["nope"])
    pipe.disable_lora()
    _check(pipe, base, loras, {}, "disable")
    pipe.enable_lora()
    assert all(torch.equal(v, snap[k]) for k, v in _live(pipe).items())
    pipe.encode_prompt(None, prompt_embeds=torch.zeros(1, 77, 128), pooled_prompt_embeds=torch.zeros(1, 64),
                       negative_prompt_embeds=torch.zeros(1, 77, 128), negative_pooled_prompt_embeds=torch.zeros(1, 64),
                       lora_scale=0.25)                      # the towers do not run: their weights stay as they are
    assert all(torch.equal(v, snap[k]) for k, v in _live(pipe).items())
    pipe.encode_prompt("a cat", negative_prompt="blurry", lora_scale=0.25)
    _check(pipe, base, loras, {"unet": two["unet"], **{c: {"A": (0.25, 0.5), "default_1": (0.25, -0.75)}
                                                       for c in ("text_encoder", "text_encoder_2")}}, "lora_scale")
    pipe.fuse_lora(lora_scale=0.5)
    fused = every({"A": (0.5, 0.5), "default_1": (0.5, -0.75)})
    _check(pipe, base, loras, fused, "fuse")
    with pytest.raises(IHError):
        pipe.set_adapters(["A"])
    from imagharmony_b200.denoise import DenoiseEngine
    monkeypatch.setattr(DenoiseEngine, "run", lambda engine, latents, *a, **k: latents.clone())
    pipe(prompt_embeds=torch.zeros(1, 77, 128), pooled_prompt_embeds=torch.zeros(1, 64), height=64, width=64,
         num_inference_steps=2, output_type="latent", cross_attention_kwargs={"scale": 3.0})
    _check(pipe, base, loras, fused, "per-call scale while fused")
    pipe.unfuse_lora()
    assert all(torch.equal(v, snap[k]) for k, v in _live(pipe).items())
    pipe(prompt_embeds=torch.zeros(1, 77, 128), pooled_prompt_embeds=torch.zeros(1, 64), height=64, width=64,
         num_inference_steps=2, output_type="latent", cross_attention_kwargs={"scale": -2.0})
    _check(pipe, base, loras, {"unet": {"A": (-2.0, 0.5), "default_1": (-2.0, -0.75)},      # embeddings given: the
                               **{c: two[c] for c in ("text_encoder", "text_encoder_2")}},    # towers keep scale 1
           "cross_attention_kwargs")
    pipe.delete_adapters("A")
    assert pipe.get_active_adapters() == ["default_1"] and pipe.get_list_adapters() == {
        "unet": ["default_1"], "text_encoder_2": ["default_1"]}
    _check(pipe, base, {"default_1": loras["default_1"]}, every({"default_1": (1.0, -0.75)}), "delete A")
    pipe.unload_lora_weights()
    assert pipe.get_list_adapters() == {} and pipe.get_active_adapters() == []
    for k, v in _live(pipe).items():
        assert v.data_ptr() == ptrs[k] and torch.equal(v, base[k]), k


def test_unchanged_state_does_no_merge(patched, monkeypatch):  # noqa: F811
    import imagharmony_b200.ops as ops
    from imagharmony_b200.denoise import DenoiseEngine
    pipe, hf1, hf2 = _pipe()
    la = _random_loras(pipe.unet, hf1, hf2)
    pipe.load_lora_weights({k: v for c in la for k, v in to_peft(la[c], c).items()})
    calls = []
    inner = ops.linear
    monkeypatch.setattr(ops, "linear", lambda *a, **k: calls.append(1) or inner(*a, **k))
    monkeypatch.setattr(DenoiseEngine, "run", lambda engine, latents, *a, **k: latents.clone())

    def call(**kw):
        pipe(prompt_embeds=torch.zeros(1, 77, 128), pooled_prompt_embeds=torch.zeros(1, 64), height=64, width=64,
             num_inference_steps=2, output_type="latent", **kw)
    epoch = pipe.unet.graph_epoch
    call()
    call(cross_attention_kwargs={"scale": 1.0})
    pipe.set_adapters("default_0", 1.0)
    assert not calls and pipe.unet.graph_epoch == epoch
    call(cross_attention_kwargs={"scale": 0.5})      # a new scale: one merge per UNet tensor, one finalize
    assert len(calls) == len(la["unet"]) and pipe.unet.graph_epoch == epoch + 1
    calls.clear()
    call(cross_attention_kwargs={"scale": 0.5})
    assert not calls and pipe.unet.graph_epoch == epoch + 1
    pipe.encode_prompt("a cat", lora_scale=0.5)       # the towers run: merged once for the new scale
    n_text = len(la["text_encoder"]) + len(la["text_encoder_2"])
    assert len(calls) == n_text + 2 * 4 * 2           # + the towers' own GEMMs (4 per layer, 2 layers, 2 towers)
    calls.clear()
    pipe.encode_prompt("a cat", lora_scale=0.5)
    assert len(calls) == 2 * 4 * 2 and pipe.unet.graph_epoch == epoch + 1


def test_fuse_and_load_edge_cases(patched):  # noqa: F811
    from imagharmony_b200._lib import IHError
    pipe, hf1, hf2 = _pipe()
    epoch = pipe.unet.graph_epoch
    pipe.fuse_lora()                                   # nothing loaded: nothing to bake, loading still works
    pipe.unfuse_lora()
    assert pipe._lora_fused is None and pipe.unet.graph_epoch == epoch
    la = _random_loras(pipe.unet, hf1, hf2)
    sd = {k: v for c in la for k, v in to_peft(la[c], c).items()}
    with pytest.raises(IHError):
        pipe.load_lora_weights(sd, cache_dir="/tmp")    # hub / loading options are refused, not ignored
    with pytest.raises(IHError):
        pipe.load_lora_weights(sd, subfolder="x")       # a subfolder of a state dict
    pipe.load_lora_weights(sd)
    base = {k: v.clone() for k, v in _live(pipe).items()}
    pipe.disable_lora()
    with pytest.raises(IHError):
        pipe.fuse_lora()                               # disabled: no active set to bake
    pipe.enable_lora()
    pipe.fuse_lora(lora_scale=0.5)
    pipe.unfuse_lora(unfuse_unet=False)               # the towers follow the active set again, the UNet stays fused
    assert set(pipe._lora_fused) == {"unet"}
    pipe.unfuse_lora()
    assert pipe._lora_fused is None and all(torch.equal(v, base[k]) for k, v in _live(pipe).items())


def test_load_from_directory_and_subfolder(patched, tmp_path):  # noqa: F811
    from safetensors.torch import save_file
    pipe, hf1, hf2 = _pipe()
    la = _random_loras(pipe.unet, hf1, hf2)
    sd = {k: v.contiguous() for c in la for k, v in to_peft(la[c], c).items()}
    (tmp_path / "style").mkdir()
    save_file(sd, str(tmp_path / "style" / "pytorch_lora_weights.safetensors"))
    save_file(sd, str(tmp_path / "other.safetensors"))
    pipe.load_lora_weights(str(tmp_path), subfolder="style", adapter_name="a")
    merged = {k: v.clone() for k, v in _live(pipe).items()}
    pipe.unload_lora_weights()
    pipe.load_lora_weights(str(tmp_path), weight_name="other.safetensors", adapter_name="b")
    assert all(torch.equal(v, merged[k]) for k, v in _live(pipe).items())


# ---------------------------------------------------------------------------------------------------------------------
# unfused forward (PEFT) vs merged native model
# ---------------------------------------------------------------------------------------------------------------------
def test_unfused_unet_forward_matches_merged_native(patched):  # noqa: F811
    from imagharmony_b200.config import TINY
    from imagharmony_b200.lora import LoraWeights, term_factor, unet_name_table
    native, ref = _build(TINY, 0)
    names = unet_name_table(native)
    lora = random_lora(module_shapes(ref, names), 8, 3, alpha=4, fp16=False)
    lw = LoraWeights(native, {})
    lw.add("a", to_kohya(lora, "unet", names))
    lw.sync("unet", {"a": (0.8, 1.25)})
    attach_unfused(ref, lora, lambda alpha, r: term_factor(0.8, 1.25, alpha, r))
    sample, ehs, te, tid = _inputs(TINY, 1, 16)
    with torch.no_grad():
        r = ref(sample, 321.0, ehs, te, tid)
        o = native(sample, torch.full((2,), 321.0), ehs, te, tid)
    assert torch.allclose(o, r, rtol=1e-4, atol=1e-4), (o - r).abs().max()
    lw.sync("unet", {})
    with torch.no_grad():
        o0 = native(sample, torch.full((2,), 321.0), ehs, te, tid)
    assert (o0 - o).abs().max() > 1e-2             # the LoRA matters at this size


def test_unfused_text_towers_match_merged_native(patched, monkeypatch):  # noqa: F811
    import imagharmony_b200.clip as clip
    from imagharmony_b200.lora import LoraWeights, term_factor
    monkeypatch.setattr(clip, "_DTYPE", [torch.float32])
    hf1, hf2, t1, t2 = _towers()
    loras = _random_loras(_tiny_unet(), hf1, hf2, rank=8, seed=9)
    lw = LoraWeights(_tiny_unet(dtype=torch.float32), {"text_encoder": t1, "text_encoder_2": t2})
    lw.add("a", {k: v for c in ("text_encoder", "text_encoder_2") for k, v in to_kohya(loras[c], c).items()})
    for comp, hf, tower in (("text_encoder", hf1, t1), ("text_encoder_2", hf2, t2)):
        lw.sync(comp, {"a": (0.6, 1.0)})
        attach_unfused(hf, loras[comp], lambda alpha, r: term_factor(0.6, 1.0, alpha, r))
        ids = torch.randint(0, 98, (2, 77), generator=torch.Generator().manual_seed(1))
        ids[:, 20:] = 99
        with torch.no_grad():
            want = hf(ids, output_hidden_states=True)
        got = tower(ids)
        assert torch.allclose(got.penultimate, want.hidden_states[-2], atol=5e-5), \
            (comp, (got.penultimate - want.hidden_states[-2]).abs().max())
