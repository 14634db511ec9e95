"""CPU: every __global__ kernel in yomitoku_b200/csrc/*.cu is tied to at least one test that reaches it, and every test
named here exists.  A new kernel fails this test until it gets a line in CENSUS; a renamed or deleted kernel or test
fails it until the line follows.  Kernels that only an end-to-end test reaches say why in their REASON line.

The kernel names are read from the sources (comments removed): the identifier before the parameter list that follows
`__global__ void`, with or without a `__launch_bounds__(...)` in between and whatever line breaks or template header
surround it.  The test names are read from the test files with ast, without importing them."""
import ast
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "yomitoku_b200", "csrc")

G = "tests/test_gpu_glue_kernels.py::"
DEC = "tests/test_gpu_decoder_kernels.py::"
DBK = "tests/test_gpu_dbnet_kernels.py::"
PQD = "tests/test_gpu_parseq_decode_kernels.py::"
RTS = "tests/test_gpu_rtdetr_stages.py::"

# kernel -> tests that reach it (op-level tests first)
CENSUS = {
    # rtdetr_ops.cu
    "pack_input_kernel": [G + "test_engine_input_and_fpn_wiring", RTS + "test_backbone_stages"],
    "avgpool2_kernel": [G + "test_avgpool2_vs_float64", RTS + "test_backbone_stages"],
    "upsample_nearest2_kernel": [G + "test_upsample_nearest2_bitwise", G + "test_engine_input_and_fpn_wiring"],
    "add_f16_kernel": [G + "test_add_f16_bitwise", G + "test_add_table_bitwise", G + "test_engine_input_and_fpn_wiring",
                       G + "test_engine_aifi_position_embedding", RTS + "test_encoder_stages",
                       RTS + "test_decoder_layer_stages"],
    "mask_invalid_rows_kernel": [G + "test_mask_invalid_exact", G + "test_engine_encoder_selection_wiring"],
    "enc_scores_kernel": [G + "test_enc_scores_exact", G + "test_engine_encoder_selection_wiring"],
    "topk_select_kernel": ["tests/test_gpu_cell_detector.py::test_topk_equals_stable_sort"],
    "gather_queries_kernel": [G + "test_gather_queries_exact", G + "test_engine_encoder_selection_wiring"],
    "ref_update_kernel": [G + "test_ref_update_vs_float64", RTS + "test_query_selection_stages",
                          RTS + "test_decoder_layer_stages"],
    "qpos_l0_kernel": [G + "test_qpos_l0_vs_float64", RTS + "test_decoder_layer_stages"],
    "deform_attn_kernel": [DEC + "test_deform_attn_vs_float64", RTS + "test_decoder_layer_stages"],
    "copy_cols_kernel": [G + "test_engine_encoder_selection_wiring", RTS + "test_decoder_layer_stages"],
    # parseq_ops.cu
    "patchify_u8_kernel": [G + "test_patchify_u8_exact"],
    "patchify_f32_kernel": [G + "test_patchify_f32_exact"],
    "layernorm_kernel": [DEC + "test_layernorm_vs_float64", RTS + "test_encoder_stages", RTS + "test_decoder_layer_stages"],
    "flash_attn_kernel": ["tests/test_gpu_kernels.py::test_attention_legacy_kernel_still_matches"],
    "single_query_attn_kernel": [DEC + "test_single_query_self_attn_vs_float64",
                                 DEC + "test_single_query_cross_attn_vs_float64"],
    "ar_control_kernel": [PQD + "test_ar_control_whole_decode"],
    "refine_embed_kernel": [PQD + "test_refine_embed_vs_reference"],
    "softmax_max_kernel": [PQD + "test_head_statistics_exact"],
    "rowmax_finalize_kernel": [PQD + "test_head_statistics_exact"],
    "apply_rep_cut_kernel": [PQD + "test_apply_rep_cut_exact"],
    "bcast_rows_kernel": ["tests/test_gpu_parseq.py::test_model_seam_vs_oracle"],
    "refine_seqs_kernel": ["tests/test_gpu_parseq.py::test_model_seam_vs_oracle"],
    "fill_i32_kernel": ["tests/test_gpu_parseq.py::test_repetition_stop_and_refine_off"],
    # attn_tc.cu, gemm_tc.cu
    "attn_tc_kernel": ["tests/test_gpu_kernels.py::test_attention_tc_vs_torch",
                       "tests/test_gpu_attention_units.py::test_unit_edges_all_head_dims",
                       RTS + "test_encoder_stages", RTS + "test_decoder_layer_stages"],
    "gemm_tc_kernel": ["tests/test_gpu_gemm_variants.py::test_linear_instance_all_activations",
                       "tests/test_gpu_gemm_variants.py::test_conv", RTS + "test_backbone_stages",
                       RTS + "test_encoder_stages", RTS + "test_decoder_layer_stages"],
    # dbnet_ops.cu
    "preprocess_kernel": [DBK + "test_preprocess_table_vs_float64"],
    "pack_nchw_kernel": ["tests/test_gpu_dbnet.py::test_reference_fixture_through_model_seam"],
    "maxpool3x3s2_kernel": [DBK + "test_maxpool_bitwise", RTS + "test_backbone_stages"],
    "upsample_bilinear_kernel": [DBK + "test_upsample_vs_float64"],
    "asf_pool_kernel": [DBK + "test_asf_vs_float64"],
    "asf_gate_kernel": [DBK + "test_asf_vs_float64"],
    "asf_cmean_kernel": [DBK + "test_asf_vs_float64"],
    "asf_apply_kernel": [DBK + "test_asf_vs_float64"],
    # dbpost_ops.cu
    "label_seed_kernel": ["tests/test_gpu_dbpost.py::test_runs_equal_scipy_twin"],
    "label_merge_kernel": ["tests/test_gpu_dbpost.py::test_runs_equal_scipy_twin"],
    "page_stats_kernel": ["tests/test_gpu_dbpost.py::test_runs_equal_scipy_twin"],
    "emit_runs_kernel": ["tests/test_gpu_dbpost.py::test_runs_equal_scipy_twin"],
    # crop_ops.cu, page_ops.cu, resample_ops.cu, table_ops.cu
    "crop_warp_kernel": ["tests/test_gpu_crops.py::test_device_crops_match_opencv_and_host_build_on_random_quads"],
    "crop_canvas_kernel": ["tests/test_gpu_crops.py::test_device_crops_match_opencv_and_host_build_on_random_quads"],
    "halve_pages_kernel": ["tests/test_gpu_mixed_batch.py::test_halve_table_equals_opencv_per_page"],
    "pack_pages_kernel": ["tests/test_gpu_device_pages.py::test_pack_equals_torch_gather"],
    "resample_first_kernel": ["tests/test_gpu_rtdetr_u8.py::test_resize_op_equals_pillow"],
    "resample_second_kernel": ["tests/test_gpu_rtdetr_u8.py::test_resize_op_equals_pillow"],
    "assign_best_overlap_kernel": ["tests/test_gpu_table_semantic.py::test_kernel_equals_oracle_bit_for_bit"],
}

# kernels no op-level test calls alone: why the listed tests are enough
REASON = {
    "pack_input_kernel": "a layout of the input with three real channels: the in-situ checks compare it exactly",
    "copy_cols_kernel": "a column copy of the logits: the in-situ checks compare pred_logits with it exactly",
    "flash_attn_kernel": "the legacy attention kernel, selected by impl 1; the engines run attn_tc_kernel",
    "bcast_rows_kernel": "a row copy seeding the refinement K/V cache: a wrong row changes the refined logits",
    "refine_seqs_kernel": "integer descriptors of the refinement attention: a wrong one changes the refined logits",
    "fill_i32_kernel": "an integer fill of the AR state: the repetition and refine-off paths depend on it",
    "pack_nchw_kernel": "the layout of the f32 model seam: the reference fixture through that seam compares its output",
    "label_seed_kernel": "one stage of the connected-component labelling, compared as a whole against a scipy twin",
    "label_merge_kernel": "one stage of the connected-component labelling, compared as a whole against a scipy twin",
    "page_stats_kernel": "one stage of the connected-component labelling, compared as a whole against a scipy twin",
    "emit_runs_kernel": "one stage of the connected-component labelling, compared as a whole against a scipy twin",
}

_KERNEL = re.compile(r"__global__\s+void\s+(?:__launch_bounds__\s*\((?:[^()]|\([^()]*\))*\)\s*)?([A-Za-z_]\w*)\s*\(")


def _strip_comments(src):
    return re.sub(r"//[^\n]*|/\*.*?\*/", "", src, flags=re.S)


def kernels_in(src):
    """names of the __global__ functions defined in C++/CUDA source text"""
    return set(_KERNEL.findall(_strip_comments(src)))


def source_kernels():
    found = {}
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu"))):
        for k in kernels_in(open(path).read()):
            found[k] = os.path.basename(path)
    return found


def test_parser_reads_every_declaration_form():
    src = """
    __global__ void plain_kernel(int a) {}
    __global__ void __launch_bounds__(256) bounded_kernel(int a) {}
    __global__ void __launch_bounds__(QT * 2, QT == 128 ? 2 : 3) nested_kernel(int a) {}
    __global__ void __launch_bounds__(kThreads, 1)
    next_line_kernel(const float* __restrict__ s) {}
    template <int P>
    __global__ void templated_kernel(const float* x) {}
    template <typename T, int N> __global__ void
        split_kernel(T* x) {}
    // __global__ void commented_kernel(int a) {}
    /* __global__ void block_commented_kernel(int a) {} */
    __device__ void device_fn(int a) {}
    """
    assert kernels_in(src) == {"plain_kernel", "bounded_kernel", "nested_kernel", "next_line_kernel",
                               "templated_kernel", "split_kernel"}


def test_every_kernel_has_a_test():
    found = source_kernels()
    assert len(found) >= 40
    missing = sorted(k for k in found if k not in CENSUS)
    assert not missing, "kernels without a test in CENSUS: %s" % ", ".join("%s (%s)" % (k, found[k]) for k in missing)


def test_every_census_entry_names_a_kernel():
    found = source_kernels()
    stale = sorted(k for k in CENSUS if k not in found)
    assert not stale, "CENSUS names kernels that no longer exist: %s" % ", ".join(stale)
    assert all(CENSUS[k] for k in CENSUS)
    assert set(REASON) <= set(CENSUS) and all(len(r) > 20 for r in REASON.values())


def _test_functions(path):
    tree = ast.parse(open(os.path.join(ROOT, path)).read())
    return {n.name for n in tree.body if isinstance(n, (ast.FunctionDef, ast.AsyncFunctionDef))}


def test_every_named_test_exists():
    bad = []
    cache = {}
    for kernel, tests in CENSUS.items():
        for t in tests:
            path, _, name = t.partition("::")
            if not name.startswith("test_") or not os.path.exists(os.path.join(ROOT, path)):
                bad.append("%s: %s" % (kernel, t))
                continue
            if path not in cache:
                cache[path] = _test_functions(path)
            if name not in cache[path]:
                bad.append("%s: %s" % (kernel, t))
    assert not bad, "CENSUS names tests that do not exist: %s" % "; ".join(bad)

