"""Every entry point of include/ih_api.h is either called directly by a named GPU parity test or exempt for a stated
reason, so a new entry point cannot land without a direct test (model-level goldens run one shape per model and do not
count).  A test "calls" an entry point when its body (or a helper function of its module that it calls) references
the symbol through the library handle, or calls `ops.<wrapper>` for an imagharmony_b200.ops function that does."""
import ast
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

EXEMPT = {
    "ih_version": "version query, checked by test_abi.py",
    "ih_last_error": "error message accessor, checked by test_abi.py",
    "ih_launch_count": "launch counter, a diagnostic with no arithmetic",
    "ih_launch_count_reset": "launch counter, a diagnostic with no arithmetic",
    "ih_gemm_set_trace": "debug timestamps, not on the product path",
    "ih_gemm_prefetch_next": "L2 prefetch hint; results never depend on it",
    "ih_attention_set_split_policy": "test aid that selects the KV-split plan of ih_attention_ws_f16",
    "ih_attention_set_kernel": "test aid that selects the multi-block attention kernel of ih_attention_ws_f16",
}

REGISTRY = {
    "ih_gemm_f16": ["test_kernels_gpu::test_gemm_plain", "test_kernel_edges_gpu::test_gemm_epilogue_matrix"],
    "ih_gemm_ln_f16": ["test_kernels_gpu::test_gemm_layernorm_fold", "test_kernel_edges_gpu::test_gemm_epilogue_matrix",
                       "test_kernel_edges_gpu::test_layernorm_fold_accuracy_envelope"],
    "ih_gemm_scaled_f16": ["test_kernel_edges_gpu::test_gemm_alpha_with_residual_and_gelu",
                           "test_kernel_edges_gpu::test_relu_epilogue_propagates_nan_and_inf"],
    "ih_conv2d_f16": ["test_kernels_gpu::test_conv3x3", "test_kernel_edges_gpu::test_conv3x3_rowbias_every_tile"],
    "ih_conv2d_shortcut_f16": ["test_kernels_gpu::test_conv3x3_fused_shortcut"],
    "ih_conv2d_scaled_f16": ["test_kernel_edges_gpu::test_conv2d_scaled_stride2_residual",
                             "test_kernel_edges_gpu::test_relu_epilogue_propagates_nan_and_inf"],
    "ih_conv2d_down_f16": ["test_img2img_gpu::test_conv_down_kernel"],
    "ih_attention_workspace_bytes": ["test_kernels_gpu::test_attention_kv_split",
                                     "test_planted_gpu::test_attention_planted"],
    "ih_attention_ws_f16": ["test_kernels_gpu::test_attention", "test_kernels_gpu::test_attention_kv_split",
                            "test_kernel_edges_gpu::test_attention_ws_f16_without_workspace",
                            "test_planted_gpu::test_attention_planted",
                            "test_planted_gpu::test_attention_two_segment_planted"],
    "ih_groupnorm_workspace_bytes": ["test_kernel_edges_gpu::test_groupnorm_workspace_reuse_and_graph_replay"],
    "ih_groupnorm_f16": ["test_kernel_edges_gpu::test_groupnorm_group_counts",
                         "test_kernel_edges_gpu::test_groupnorm_large_group_means",
                         "test_kernel_edges_gpu::test_groupnorm_workspace_reuse_and_graph_replay",
                         "test_planted_gpu::test_groupnorm_planted"],
    "ih_layernorm_f16": ["test_kernels_gpu::test_layernorm", "test_kernel_edges_gpu::test_layernorm_large_mean",
                         "test_planted_gpu::test_layernorm_planted"],
    "ih_linear_small_f16": ["test_kernel_edges_gpu::test_linear_small_edges"],
    "ih_attention_small_f16": ["test_kernel_edges_gpu::test_attention_small_key_tails",
                               "test_kernel_edges_gpu::test_attention_small_rejects_ragged_warp_count"],
    "ih_sinusoid_f16": ["test_kernels_gpu::test_sinusoid"],
    "ih_add_bcast_f16": ["test_kernel_edges_gpu::test_add_bcast"],
    "ih_mean_tokens_f16": ["test_kernel_edges_gpu::test_mean_tokens"],
    "ih_softmax_rows_masked_f16": ["test_vae_gpu::test_softmax_rows_kernel",
                                   "test_vae_gpu::test_softmax_rows_masked_kernel",
                                   "test_planted_gpu::test_softmax_rows_masked_planted"],
    "ih_upsample2x_f16": ["test_kernels_gpu::test_upsample", "test_kernel_edges_gpu::test_upsample2x_odd"],
    "ih_concat_f16": ["test_kernel_edges_gpu::test_concat_channels"],
    "ih_im2col3x3_nchw_f16": ["test_inpaint9_gpu::test_im2col_cat_kernel_equals_im2col_of_the_concatenation"],
    "ih_im2col3x3_nchw_cat_f16": ["test_inpaint9_gpu::test_im2col_cat_kernel_equals_im2col_of_the_concatenation"],
    "ih_nhwc_to_nchw_f16": ["test_kernel_edges_gpu::test_nhwc_to_nchw"],
    "ih_vae_posterior_noise_f16": ["test_img2img_gpu::test_posterior_noise_kernel"],
    "ih_euler_cfg_step": ["test_kernels_gpu::test_euler_cfg_step"],
    "ih_euler_step_ex": ["test_kernels_gpu::test_euler_step_ex", "test_planted_gpu::test_step_kernels_rescale_planted"],
    "ih_euler_inpaint_step": ["test_inpaint_gpu::test_euler_inpaint_step_kernel",
                              "test_planted_gpu::test_step_kernels_rescale_planted"],
    "ih_dpm_solver_step": ["test_dpm_gpu::test_dpm_solver_step_kernel",
                           "test_planted_gpu::test_step_kernels_rescale_planted"],
    "ih_euler_ancestral_step": ["test_euler_a_gpu::test_euler_ancestral_step_kernel",
                                "test_planted_gpu::test_step_kernels_rescale_planted"],
    "ih_euler_ancestral_scale_input": ["test_euler_a_gpu::test_first_input_equals_torch_scale_model_input"],
    "ih_scale_model_input_ex": ["test_kernels_gpu::test_euler_cfg_step",
                                "test_kernel_edges_gpu::test_scale_model_input_entry"],
    "ih_attention_generic_f16": ["test_clip_gpu::test_attention_generic"],
    "ih_embed_tokens_f16": ["test_kernel_edges_gpu::test_embed_tokens_clamps_ids"],
    "ih_resize_patchify_f16": ["test_clip_gpu::test_embed_quickgelu_resize_kernels"],
    "ih_conv3x3_small_f16": ["test_kernel_edges_gpu::test_conv3x3_small_edges"],
    "ih_controlnet_add_residuals_f16": ["test_controlnet_gpu::test_injection_kernel_bit_exact_sdxl_shapes"],
    "ih_controlnet_add_residuals_multi_f16": ["test_multi_controlnet_gpu::test_multi_kernel_bit_exact_sdxl_shapes"],
}


def _header_symbols():
    txt = open(os.path.join(ROOT, "include", "ih_api.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return set(re.findall(r"\b(ih_[a-z0-9_]+)\s*\(", txt))


def _functions(path):
    return {n.name: n for n in ast.parse(open(path).read()).body if isinstance(n, ast.FunctionDef)}


def _attrs(fn):
    return {n.attr for n in ast.walk(fn) if isinstance(n, ast.Attribute)}


def _ops_calls(fn):
    """Names of the ops functions called as `ops.<name>(...)`."""
    return {n.func.attr for n in ast.walk(fn) if isinstance(n, ast.Call) and isinstance(n.func, ast.Attribute)
            and isinstance(n.func.value, ast.Name) and n.func.value.id == "ops"}


def _calls(fn):
    return {n.func.id for n in ast.walk(fn) if isinstance(n, ast.Call) and isinstance(n.func, ast.Name)}


def _reach(fns, name):
    """(ih_* attribute names, ops calls) of test `name` and of the module-level helpers it calls, transitively."""
    seen, todo, syms, opcalls = set(), [name], set(), set()
    while todo:
        f = todo.pop()
        if f in seen:
            continue
        seen.add(f)
        syms |= {a for a in _attrs(fns[f]) if a.startswith("ih_")}
        opcalls |= _ops_calls(fns[f])
        todo += [c for c in _calls(fns[f]) if c in fns]
    return syms, opcalls


def _wrappers():
    """ih_* symbol -> names of the imagharmony_b200.ops functions that call it."""
    out = {}
    for name, fn in _functions(os.path.join(ROOT, "imagharmony_b200", "ops.py")).items():
        for a in _attrs(fn):
            if a.startswith("ih_"):
                out.setdefault(a, set()).add(name)
    return out


def test_registry_and_exemptions_cover_the_header_exactly():
    declared = _header_symbols()
    assert not set(REGISTRY) & set(EXEMPT), set(REGISTRY) & set(EXEMPT)
    assert set(REGISTRY) | set(EXEMPT) == declared, {
        "declared but neither tested nor exempt": sorted(declared - set(REGISTRY) - set(EXEMPT)),
        "listed but not declared": sorted((set(REGISTRY) | set(EXEMPT)) - declared)}
    assert all(REGISTRY.values()) and all(EXEMPT.values())


def test_registered_gpu_tests_exist_and_call_their_entry_point():
    gpu_files = {os.path.basename(p)[:-3]: p for p in glob.glob(os.path.join(ROOT, "tests", "*_gpu.py"))}
    wrappers = _wrappers()
    modules = {}
    for symbol, tests in REGISTRY.items():
        for ref in tests:
            mod, name = ref.split("::")
            assert mod in gpu_files, f"{symbol}: {ref}: no tests/{mod}.py"
            fns = modules.setdefault(mod, _functions(gpu_files[mod]))
            assert name in fns and name.startswith("test_"), f"{symbol}: {ref} does not exist"
            syms, opcalls = _reach(fns, name)
            assert symbol in syms or opcalls & wrappers.get(symbol, set()), (
                f"{ref} neither references {symbol} nor calls ops.{sorted(wrappers.get(symbol, []))}")
