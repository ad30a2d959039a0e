"""GPU parity of the surface VAEs at the extents the C ABI accepts beyond the cascade's own (decoder latents 1 x 1, 2 x 2
and 3 x 3; encoder inputs 8 x 8 and 24 x 24), against the CPU fp32 oracle (oracle/vae.py) at the 1e-3 relative-L2 bar of
test_gpu_vae.py.  These are the only calls that reach the implicit convolution on 1 x 1 and 2 x 2 images (TMA boxes
{64, 1, 1, 128} and {64, 2, 2, 32}, 8 of 9 taps entirely in padding), the explicit im2col path at 3 / 6 / 12 / 24 and the
generic GroupNorm kernel at 9, 36, 144 and 576 positions.  As at the cascade's extents, the implicit and the explicit
(BREPGEN_B200_VAE_IM2COL=1) builds must give bit-identical outputs."""
import os

import pytest
import torch

from brepgen_b200.spec import surf_decoder_spec, surf_encoder_spec
from brepgen_b200.synth import synth_state_dict
from oracle import vae as V

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


def _run_both_builds(make, x):
    """the module's output with implicit convolutions and with the explicit im2col path (read at handle creation)"""
    outs = []
    for explicit in (0, 1):
        os.environ["BREPGEN_B200_VAE_IM2COL"] = str(explicit)
        try:
            m = make()
            m.use_graph = False
            with torch.no_grad():
                outs.append(m(x.cuda()).cpu())
            torch.cuda.synchronize()
        finally:
            os.environ.pop("BREPGEN_B200_VAE_IM2COL", None)
    return outs


@pytest.mark.parametrize("hw", [1, 2, 3])
def test_surface_decoder_small_latents(hw):
    from brepgen_b200.vae import AutoencoderKLFastDecode
    sd = synth_state_dict(surf_decoder_spec(), seed=5)

    def make():
        m = AutoencoderKLFastDecode()
        m.load_state_dict(sd, strict=False)
        return m.cuda().eval()

    N = 5
    z = torch.randn(N, 3, hw, hw, generator=torch.Generator().manual_seed(hw))
    implicit, explicit = _run_both_builds(make, z)
    with torch.no_grad():
        ref = V.surf_decode(sd, z)
    assert implicit.shape == (N, 3, 8 * hw, 8 * hw) and torch.isfinite(implicit).all()
    err = rel_l2(implicit, ref)
    print(f"surface decoder latent {hw}x{hw} rel_l2={err:.3e}")
    assert err < 1e-3, err
    assert torch.equal(implicit, explicit)


@pytest.mark.parametrize("hw", [8, 24])
def test_surface_encoder_small_inputs(hw):
    from brepgen_b200.vae import AutoencoderKLFastEncode
    sd = synth_state_dict(surf_encoder_spec(), seed=7)

    def make():
        m = AutoencoderKLFastEncode()
        m.load_state_dict(sd, strict=False)
        return m.cuda().eval()

    N = 3
    x = torch.rand(N, 3, hw, hw, generator=torch.Generator().manual_seed(hw)) * 2 - 1
    implicit, explicit = _run_both_builds(make, x)
    with torch.no_grad():
        ref = V.surf_encode(sd, x)
    assert implicit.shape == (N, 3, hw // 8, hw // 8) and torch.isfinite(implicit).all()
    err = rel_l2(implicit, ref)
    print(f"surface encoder {hw}x{hw} rel_l2={err:.3e}")
    assert err < 1e-3, err
    assert torch.equal(implicit, explicit)
