"""One small invocation of every CUDA path of the library (the GPU tests' own functions at their smallest shapes), meant to
be run under compute-sanitizer:
    compute-sanitizer --tool memcheck --error-exitcode 9 python tools/sanitize.py
    compute-sanitizer --tool racecheck --error-exitcode 9 python tools/sanitize.py ops
The parity assertions of the tests stay active, so a pass means: no invalid access and unchanged results."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)
import torch   # noqa: E402

what = sys.argv[1] if len(sys.argv) > 1 else "all"


def run(name, fn, *a):
    fn(*a)
    torch.cuda.synchronize()
    print("ok", name, a, flush=True)


import test_gpu_ops as T   # noqa: E402
run("gemm", T.test_gemm, 128, 256, 64, 0, 0, False, False, 0)
run("gemm", T.test_gemm, 300, 768, 768, 0, 0, True, False, 0)          # small-M path: 128-wide tiles
run("gemm", T.test_gemm, 257, 1024, 768, 1, 1, True, False, 0)
run("gemm", T.test_gemm, 513, 768, 1024, 0, 0, True, True, 0)
run("gemm", T.test_gemm, 200, 128, 192, 0, 0, True, False, 7)
run("gemm", T.test_gemm, 128 * 170, 2304, 768, 1, 0, True, False, 0)   # persistent tiles wrap, fp16 epilogue
run("attention", T.test_attention, 2, 30, None, 0)
run("attention", T.test_attention, 3, 100, "rand", 1)
run("attention", T.test_attention, 1, 300, None, 0)
run("attention", T.test_attention, 2, 257, "rand", 0)
run("attention", T.test_attention, 2, 1000, "blocks", 1)
run("layernorm", T.test_layernorm, 77, 0)
run("scheduler steps", T.test_fused_ddpm_and_pndm_steps)
import test_gpu_sample_noise as SN   # noqa: E402
run("keyed noise", SN.test_randn_keyed_matches_numpy_philox, 13, 1, 0)
run("keyed steps", SN.test_ddpm_step_with_keys_equals_step_fed_keyed_noise_and_table_form, 7, 0.6)
run("keyed bad args", SN.test_bad_keyed_step_arguments_are_rejected_and_launch_nothing)
import test_gpu_ddim as DD   # noqa: E402
run("ddim step", DD.test_step_matches_float64, 0, 10, False, 0.5)
run("ddim forms", DD.test_forms_agree_and_draw_the_ddpm_step_noise, 7, 0.6, 1)
run("ddim bad args", DD.test_bad_arguments_are_rejected_and_launch_nothing)
import test_gpu_dpm as DP   # noqa: E402
run("dpm step", DP.test_step_matches_float64, 10, "sde-dpmsolver++")
run("dpm forms", DP.test_eager_keyed_and_table_forms_agree, 7, 0.6)
run("dpm bad args", DP.test_bad_arguments_are_rejected_and_launch_nothing)
import test_gpu_completion as CO   # noqa: E402
run("replace known", CO.test_kernel_matches_float64, 18, 13, "random")
run("replace forms", CO.test_noise_forms_agree, 6, 7)
run("replace bad args", CO.test_bad_arguments_are_rejected_and_launch_nothing)
import test_gpu_repaint as RP   # noqa: E402
run("repaint step", RP.test_step_matches_float64_and_ddim, 18, 13, 0.8, "random")
run("repaint undo", RP.test_undo_is_the_fp32_chain_bit_for_bit, 50, 300)
run("repaint forms", RP.test_noise_forms_agree, 6, 7)
run("repaint bad args", RP.test_bad_arguments_are_rejected_and_launch_nothing)
import test_gpu_variation as VA   # noqa: E402
run("variation gather", VA.test_gather_is_the_torch_expression_bit_for_bit, 18, 50, 3.0)
run("variation keyed gather", VA.test_keyed_z_is_randn_keyed, 18, 13)
run("variation poisoned gather", VA.test_out_of_range_index_poisons_only_its_token)
run("variation fill", VA.test_fill_index_matches_oracle, 100, 50, True)
run("variation dedup index", VA.test_dedup_index_keeps_positions_and_mask, "duplicates", 3, 7)
run("variation bad args", VA.test_bad_arguments_are_rejected_and_launch_nothing)
if what != "ops-no-res1":
    run("gemm", T.test_gemm, 128 * 170 + 5, 768, 1024, 0, 0, True, True, 0)   # persistent tiles wrap, residual epilogue
if what == "all":
    import test_gpu_cascade as C
    import test_gpu_compaction as K
    import test_gpu_denoisers as D
    import test_gpu_post as P
    import test_gpu_vae as V
    run("denoiser golden", D.test_golden, "surfpos", True)
    run("denoiser golden", D.test_golden, "edgez", False)
    run("compaction", K.test_compact_equals_dense_on_valid_tokens, *K.CASES[0])
    run("dedup surfaces", C.test_dedup_surfaces_bit_exact, 3, 7)
    run("dedup edges", C.test_dedup_edges_bit_exact, 2, 9, 30)
    run("short cascade", C.test_short_cascade_matches_oracle, True, "ddpm")
    run("surface decoder", V.test_surface_decoder, 5, 2)
    run("edge decoder", V.test_edge_decoder, 37, 16)
    run("encoders", V.test_encoders_match_oracle)
    import test_gpu_vae_posterior as VP
    run("posterior tail", VP.test_moments_match_oracle_and_mean_equals_encode, "surf", 24)
    run("posterior tail", VP.test_moments_match_oracle_and_mean_equals_encode, "edge", 32)
    run("reconstruct", VP.test_posterior_z_kl_mse_match_fp64, "surf")
    run("reconstruct", VP.test_reconstruct_equals_unfused_entry_points, "edge")
    run("reconstruct graph", VP.test_graph_replayed_chunks_equal_eager, "edge", 29, 8)
    run("reconstruct bad args", VP.test_bad_arguments_are_reported_not_faulted)
    run("post topology", P.test_topology_and_edges_match_reference, list(P.CASES)[0])
    run("post joint optimize", P.test_joint_optimize_matches_reference, list(P.CASES)[0])
print("SANITIZE_DONE", flush=True)
