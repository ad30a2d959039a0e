"""CPU tests of the full auto-encoders' surface (brepgen_b200/vae.py AutoencoderKL / AutoencoderKL1D /
DiagonalGaussianDistribution), the posterior oracle (oracle/vae_posterior.py) and the VAE trainers' validation glue
(brepgen_b200/validation.py) against tests/golden/vae_val_golden.npz, the results of the reference's own statements
(tests/golden/make_golden_vae_val.py).  No compute call of the CUDA library is made here."""
import ctypes
import os

import numpy as np
import pytest
import torch

from brepgen_b200 import _ffi
from brepgen_b200 import validation as VAL
from brepgen_b200.spec import edge_decoder_spec, edge_encoder_spec, surf_decoder_spec, surf_encoder_spec
from make_golden_vae_val import SEEDS, OracleAutoencoder, full_state_dict
from oracle import vae_posterior as VP

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vae_val_golden.npz")
NEW_SYMBOLS = ("bg_vae_encode_moments", "bg_vae_posterior", "bg_vae_reconstruct", "bg_vae_reconstruct_workspace_bytes")


def test_posterior_symbols_are_declared_and_exported():
    hdr = open(os.path.join(os.path.dirname(GOLD), "..", "..", "include", "brepgen_b200.h")).read()
    lib = ctypes.CDLL(_ffi.LIB_PATH)
    for name in NEW_SYMBOLS:
        assert f"{name}(" in hdr and name in _ffi.SIGNATURES, name
        assert hasattr(lib, name), name


@pytest.mark.parametrize("kind", ["surf", "edge"])
def test_oracle_standin_reproduces_reference_statements(kind):
    g = np.load(GOLD)
    x = torch.from_numpy(g["surf_uv" if kind == "surf" else "edge_u"])
    model = OracleAutoencoder(full_state_dict(kind), kind == "surf")
    torch.manual_seed(SEEDS[kind])
    fn = VAL.surfvae_val_losses if kind == "surf" else VAL.edgevae_val_losses
    loss = fn(model, x)
    assert abs(loss - float(g[f"loss_{kind}"])) <= 1e-5 * abs(float(g[f"loss_{kind}"])), (loss, g[f"loss_{kind}"])
    # the loop helper: total_loss / total_count over one batch
    torch.manual_seed(SEEDS[kind])
    mse = VAL.vae_val_mse(model, [x], edge=kind == "edge")
    assert abs(mse - float(g[f"loss_{kind}"]) / int(g[f"count_{kind}"])) <= 1e-5 * mse
    # moments, the posterior draw and the KL terms of the trainers' statements
    xin = x.permute(0, 3, 1, 2) if kind == "surf" else x.permute(0, 2, 1)
    with torch.no_grad():
        post = model.encode(xin).latent_dist
    assert np.allclose(post.parameters.numpy(), g[f"moments_{kind}"], rtol=1e-5, atol=1e-6)
    torch.manual_seed(SEEDS[kind])
    assert np.allclose(post.sample().numpy(), g[f"z_{kind}"], rtol=1e-5, atol=1e-6)
    if kind == "surf":
        kl = post.kl().mean()
    else:
        kl = 0.5 * torch.sum(post.mean ** 2 + post.var - 1.0 - post.logvar, dim=[1, 2]).mean()
    assert abs(float(kl) - float(g[f"kl_{kind}"])) <= 1e-5 * abs(float(g[f"kl_{kind}"]))


def test_oracle_distribution_invariants():
    gen = torch.Generator().manual_seed(3)
    m = torch.randn(4, 6, 2, 2, generator=gen) * 2
    d = VP.DiagonalGaussianDistribution(m)
    assert torch.equal(d.sample(noise=torch.zeros(4, 3, 2, 2)), d.mode())
    assert torch.equal(d.mode(), m[:, :3])
    assert (d.kl() >= 0).all()
    assert torch.equal(VP.DiagonalGaussianDistribution(torch.zeros(2, 6, 2, 2)).kl(), torch.zeros(2))
    assert torch.allclose(d.kl(d), torch.zeros(4), atol=1e-6)
    ext = torch.zeros(1, 6, 1, 2)
    ext[0, 3:, 0, 0], ext[0, 3:, 0, 1] = -100.0, 100.0
    e = VP.DiagonalGaussianDistribution(ext)
    assert (e.logvar[..., 0] == -30.0).all() and (e.logvar[..., 1] == 20.0).all()
    assert torch.allclose(e.var[..., 1], torch.exp(torch.tensor(20.0)))
    det = VP.DiagonalGaussianDistribution(m, deterministic=True)
    assert torch.equal(det.sample(), det.mean) and float(det.kl()) == 0.0


def test_product_distribution_attributes_match_oracle():
    from brepgen_b200.vae import DiagonalGaussianDistribution
    m = torch.randn(3, 6, 4, generator=torch.Generator().manual_seed(4)) * 20
    a, b = DiagonalGaussianDistribution(m), VP.DiagonalGaussianDistribution(m)
    for k in ("mean", "logvar", "std", "var"):
        assert torch.equal(getattr(a, k), getattr(b, k)), k
    assert a.mode() is a.mean and a.parameters is m and a.deterministic is False
    with pytest.raises(IndexError):           # diffusers' kl() sums over dims [1, 2, 3]: a 1-D latent has no dim 3
        a.kl()
    with pytest.raises(RuntimeError):         # no CPU path
        DiagonalGaussianDistribution(torch.zeros(1, 6, 2, 2)).sample()
    det = DiagonalGaussianDistribution(m, deterministic=True)
    assert torch.equal(det.std, torch.zeros_like(det.mean)) and torch.equal(det.kl(), torch.Tensor([0.0]))


def test_randn_tensor_follows_diffusers():
    from brepgen_b200.vae import randn_tensor
    a = randn_tensor((2, 3, 4), generator=torch.Generator().manual_seed(9), device="cpu")
    assert torch.equal(a, torch.randn(2, 3, 4, generator=torch.Generator().manual_seed(9)))
    gens = [torch.Generator().manual_seed(s) for s in (1, 2)]
    b = randn_tensor((2, 3), generator=gens, device="cpu")
    assert torch.equal(b[1], torch.randn(1, 3, generator=torch.Generator().manual_seed(2))[0])


@pytest.mark.parametrize("kind", ["surf", "edge"])
def test_full_autoencoder_state_dict_and_config(kind):
    from brepgen_b200.vae import AutoencoderKL, AutoencoderKL1D
    if kind == "surf":
        m = AutoencoderKL(in_channels=3, out_channels=3, down_block_types=["DownEncoderBlock2D"] * 4,
                          up_block_types=["UpDecoderBlock2D"] * 4, block_out_channels=[128, 256, 512, 512],
                          layers_per_block=2, act_fn="silu", latent_channels=3, norm_num_groups=32, sample_size=512)
        spec = surf_encoder_spec() + surf_decoder_spec()
    else:
        m = AutoencoderKL1D(in_channels=3, out_channels=3, down_block_types=["DownBlock1D"] * 3,
                            up_block_types=["UpBlock1D"] * 3, block_out_channels=[128, 256, 512], layers_per_block=2,
                            act_fn="silu", latent_channels=3, norm_num_groups=32, sample_size=512)
        spec = edge_encoder_spec() + edge_decoder_spec()
    assert set(m.state_dict().keys()) == {k for k, _ in spec}
    assert len(m.state_dict()) == len(spec)
    m.load_state_dict(full_state_dict(kind), strict=True)          # a full checkpoint loads strictly
    m.enable_slicing()
    m.disable_slicing()
    with pytest.raises(NotImplementedError):
        m.enable_tiling()
    cls = type(m)
    with pytest.raises(NotImplementedError):
        cls(latent_channels=4)
    with pytest.raises(NotImplementedError):
        cls(block_out_channels=[64])
    with pytest.raises(NotImplementedError):
        cls(down_block_types=["DownEncoderBlock2D"])
