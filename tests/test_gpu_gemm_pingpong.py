"""The encoder-layer GEMM forms give the same bytes whichever kernel runs them: by default the fp32-output forms run on
the ping-pong kernel (gemm_pp_kernel), and BREPGEN_B200_GEMM_PINGPONG=0 sends every form to gemm_f16_kernel.  The fp16
forms (qkv, linear1) run on gemm_f16_kernel either way; they stay in the list so that moving a form between the kernels
stays checked.

Each case runs in this process through bg_op_gemm_f16_ex and, with the same seeded inputs, in a subprocess with the
knob set to 0; the SHA-256 digests of the whole output buffers must match.  The forms are those of denoiser.cu at
precisions 0, 1 and 2: qkv (fp16 out, a_kwrap and, at precision 1, n_short / k_short), out_proj and linear2 (in-place
fp32 residual, a_kwrap from precision 1 / 2), linear1 (ReLU, fp16 out), fc_out (fp32 out without residual; from precision
1 the compensated [x_hi | x_lo | x_hi] x [W_hi | W_hi | W_lo] product, a_kwrap 1536).  Row counts: 4000 (one sample of the edge
stage), 256 000 (the benchmark's B = 64), 77 777 (persistent CTAs wrap, partial last tile) and 3200 (a surface stage:
fewer 128 x 128 tiles than SMs for some forms).  Device row counts (token compaction) end inside a tile, on a tile
boundary, at 0 and past M; the rows from *m_dev on must keep their prior contents.

    python tests/test_gpu_gemm_pingpong.py OUT.json     writes the digests of every case (the subprocess side)
"""
import hashlib
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KNOB = "BREPGEN_B200_GEMM_PINGPONG"
D, FF = 768, 1024

# form: (N, A columns, output fp16, ReLU, in-place residual)
FORMS = {"qkv": (3 * D, D, True, 0, False), "out_proj": (D, D, False, 0, True),
         "linear1": (FF, D, True, 1, False), "linear2": (D, FF, False, 0, True), "fc_out": (D, D, False, 0, False)}


def a_cols_and_k(form, precision):
    """A columns and K of the form at a precision: split weights [W_hi | W_lo] double K over the same A (a_kwrap)"""
    a_cols = FORMS[form][1]
    if form == "fc_out":
        return (2 * D, 3 * D) if precision >= 1 else (D, D)
    split = precision >= 1 if form in ("qkv", "out_proj") else precision >= 2
    return a_cols, 2 * a_cols if split else a_cols


CASES = [(f, prec, M, None) for f in FORMS for prec in (0, 1, 2) for M in (4000, 256_000, 77_777, 3200)]
CASES += [(f, 1, 4000, m) for f in ("linear1", "out_proj", "qkv") for m in (0, 1000, 1024, 3999, 5000)]
CASES += [(f, 1, 256_000, m) for f in ("linear1", "out_proj") for m in (204_817, 204_800)]


def case_id(case):
    f, prec, M, m = case
    return f"{f}-p{prec}-M{M}" + ("" if m is None else f"-mdev{m}")


def run_case(case):
    """(output buffer after the GEMM, its contents before)"""
    from brepgen_b200 import _ffi
    f, prec, M, m_rows = case
    N, _, f16, relu, resid = FORMS[f]
    a_cols, K = a_cols_and_k(f, prec)
    g = torch.Generator(device="cuda").manual_seed(M + N + K + prec)
    A = torch.randn(M, a_cols, generator=g, device="cuda").half()
    W = (torch.randn(N, K, generator=g, device="cuda") / K ** 0.5).half()
    bias = torch.randn(N, generator=g, device="cuda")
    if resid:
        out = torch.randn(M, N, generator=g, device="cuda")
    else:
        out = torch.full((M, N), float("nan"), device="cuda", dtype=torch.float16 if f16 else torch.float32)
    init = out.clone()
    n_short, k_short = (2 * D, D) if (f == "qkv" and prec == 1) else (0, 0)
    m_dev = None if m_rows is None else torch.tensor([m_rows], dtype=torch.int32, device="cuda")
    o = out.data_ptr()
    _ffi.check(_ffi.lib().bg_op_gemm_f16_ex(A.data_ptr(), a_cols, W.data_ptr(), K, M, N, K, o, N, int(f16), relu,
                                            bias.data_ptr(), o if resid else None, N if resid else 0, None, 1, 0,
                                            a_cols if K > a_cols else 0, n_short, k_short, _ffi.ptr(m_dev), None,
                                            _ffi.current_stream()), case_id(case))
    torch.cuda.synchronize()
    return out, init


def digest(t):
    return hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy()).hexdigest()


@pytest.fixture(scope="module")
def legacy_digests(tmp_path_factory):
    path = tmp_path_factory.mktemp("pingpong") / "legacy.json"
    env = dict(os.environ, **{KNOB: "0"})
    r = subprocess.run([sys.executable, os.path.abspath(__file__), str(path)], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-3000:]
    with open(path) as fh:
        return json.load(fh)


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_pingpong_matches_legacy(case, legacy_digests):
    if os.environ.get(KNOB, "1").strip() == "0":
        pytest.skip(f"{KNOB}=0 in this process: both sides would run the legacy kernel")
    out, init = run_case(case)
    m_rows = case[3]
    if m_rows is not None:
        k = min(m_rows, case[2])
        assert torch.equal(out[k:].view(torch.uint8), init[k:].view(torch.uint8)), "rows past *m_dev were written"
    assert digest(out) == legacy_digests[case_id(case)], f"{case_id(case)}: outputs differ from the legacy kernel"


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    res = {}
    for c in CASES:
        out, _ = run_case(c)
        res[case_id(c)] = digest(out)
        del out
    with open(sys.argv[1], "w") as fh:
        json.dump(res, fh)
