"""Does a GEMM row come out bit-identical whatever M (and so the tile width the GEMM picks) and wherever it sits?

Per-sample noise makes sample k's inputs independent of the batch; its outputs are then bit-identical across batch sizes
only if every kernel computes a row the same way at every M.  The GEMM picks 128-wide column tiles when 256-wide ones would
leave SMs idle (csrc/gemm.cu), so at L = 4000 the edge stages run 128-wide tiles at B = 1 and 256-wide tiles at B = 64.
This compares the same A rows inside M = 4000 and inside M = 256 000 (at an offset that is not a multiple of the 128-row
tile) for the denoisers' N x K shapes, and one VAE decoder convolution (256 -> 256 channels, 3x3, 3 terms) over 2 and 1024
images.  Prints one line per case: tile widths and the number of differing elements.
    python tools/batch_invariance.py
"""
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from brepgen_b200 import _ffi as f  # noqa: E402


def gemm(A, W, bias, M, N, K):
    out = torch.empty(M, N, device="cuda")
    f.check(f.lib().bg_op_gemm_f16(A.data_ptr(), K, W.data_ptr(), K, M, N, K, out.data_ptr(), N, 0, 0, bias.data_ptr(),
                                   None, N, None, 1, N, f.current_stream()), "gemm")
    return out


def tile_width(M, N):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return 256 if N % 256 == 0 and ((M + 127) // 128) * (N // 256) >= sms else 128


def main():
    g = torch.Generator(device="cuda").manual_seed(0)
    Mbig, Msmall, r0 = 256_000, 4000, 123_457
    worst = 0
    for name, N, K in (("out_proj", 768, 768), ("linear1", 1024, 768), ("linear2", 768, 1024)):
        A = torch.randn(Mbig, K, generator=g, device="cuda").half()
        W = (torch.randn(N, K, generator=g, device="cuda") / math.sqrt(K)).half()
        bias = torch.randn(N, generator=g, device="cuda")
        big = gemm(A, W, bias, Mbig, N, K)
        small = gemm(A[r0:r0 + Msmall].contiguous(), W, bias, Msmall, N, K)
        head = gemm(A[:Msmall].contiguous(), W, bias, Msmall, N, K)
        torch.cuda.synchronize()
        d1 = int((big[r0:r0 + Msmall] != small).sum())
        d2 = int((big[:Msmall] != head).sum())
        worst = max(worst, d1, d2)
        print(f"gemm {name} N={N} K={K}: tiles M={Msmall} -> {tile_width(Msmall, N)}, M={Mbig} -> {tile_width(Mbig, N)}; "
              f"differing elements: rows at offset {r0}: {d1}, rows at 0: {d2} (of {Msmall * N})", flush=True)
        del A, big
    # one decoder convolution over 2 and over 1024 images (M = 512 vs 262 144 rows: 128- vs 256-wide tiles)
    C = Cout = 256
    H = Wd = 16
    taps, kw = 9, 3
    x32 = torch.randn(1024, H, Wd, C, generator=g, device="cuda")
    hi = x32.half()
    lo = (x32 - hi.float()).half()
    x = torch.cat([hi, lo], -1).contiguous()
    w32 = torch.randn(Cout, C, 3, 3, generator=g, device="cuda") / math.sqrt(C * taps)
    whi = w32.half()
    wlo = (w32 - whi.float()).half()
    pk = lambda t: t.permute(0, 2, 3, 1).reshape(Cout, taps * C)
    wbuf = torch.cat([pk(whi), pk(whi), pk(wlo)], 1).contiguous()
    bias = torch.randn(Cout, generator=g, device="cuda")

    def conv(n):
        out = torch.empty(n * H * Wd, Cout, device="cuda")
        f.check(f.lib().bg_op_conv_f16(x.data_ptr(), 2 * C, wbuf.data_ptr(), Cout, n, H, Wd, C, taps, kw, 1, 3, out.data_ptr(),
                                       Cout, bias.data_ptr(), None, Cout, f.current_stream()), "conv")
        return out
    big, small = conv(1024), conv(2)
    torch.cuda.synchronize()
    d = int((big[:small.shape[0]] != small).sum())
    worst = max(worst, d)
    print(f"conv 3x3 {C}->{Cout} {H}x{Wd}: tiles N=2 -> {tile_width(2 * H * Wd, Cout)}, N=1024 -> "
          f"{tile_width(1024 * H * Wd, Cout)}; differing elements: {d} (of {small.numel()})", flush=True)
    print("BIT_IDENTICAL" if worst == 0 else "NOT_BIT_IDENTICAL", flush=True)


if __name__ == "__main__":
    main()
