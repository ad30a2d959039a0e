"""GPU tests of the full auto-encoders: the fused encoder tail (quant_conv + posterior), bg_vae_posterior, bg_vae_reconstruct
(encoder -> posterior -> decoder -> per-sample MSE in one call), AutoencoderKL / AutoencoderKL1D and the VAE trainers'
validation against the oracle, fp64 restatements of the kernels' own arithmetic and tests/golden/vae_val_golden.npz."""
import os

import numpy as np
import pytest
import torch

from brepgen_b200 import _ffi
from brepgen_b200 import validation as VAL
from make_golden_vae_val import SEEDS, full_state_dict
from oracle import vae as V
from oracle import vae_posterior as VP

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vae_val_golden.npz")


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm())


def _model(kind):
    from brepgen_b200.vae import AutoencoderKL, AutoencoderKL1D
    m = AutoencoderKL() if kind == "surf" else AutoencoderKL1D()
    m.load_state_dict(full_state_dict(kind), strict=True)
    return m.cuda().eval()


def _input(kind, N, hw=32, seed=0):
    g = torch.Generator().manual_seed(seed)
    shape = (N, 3, hw, hw) if kind == "surf" else (N, 3, 32)
    return torch.rand(*shape, generator=g) * 2 - 1


def _ws(nbytes):
    return torch.empty(nbytes, dtype=torch.uint8, device="cuda")


def _encode_mode(m, x):
    """bg_vae_encode (the mode) through the module's own encoder handle"""
    N, hw = x.shape[0], x.shape[-1]
    out = torch.empty((N, 3) + tuple(s // 8 for s in x.shape[2:]), device="cuda")
    ws = _ws(_ffi.lib().bg_vae_workspace_bytes(m._handle, N))
    _ffi.check(_ffi.lib().bg_vae_encode(m._handle, x.data_ptr(), N, hw, out.data_ptr(), ws.data_ptr(), ws.numel(),
                                        _ffi.current_stream()), "bg_vae_encode")
    return out


def _reconstruct(m, x, noise):
    """one bg_vae_reconstruct call with every output requested"""
    N, hw = x.shape[0], x.shape[-1]
    lat = tuple(s // 8 for s in x.shape[2:])
    mom, z = torch.empty((N, 6) + lat, device="cuda"), torch.empty((N, 3) + lat, device="cuda")
    kl, dec, mse = torch.empty(N, device="cuda"), torch.empty_like(x), torch.empty(N, device="cuda")
    ws = _ws(_ffi.lib().bg_vae_reconstruct_workspace_bytes(m._handle, m._dec, N))
    _ffi.check(_ffi.lib().bg_vae_reconstruct(m._handle, m._dec, x.data_ptr(), N, hw, _ffi.ptr(noise), mom.data_ptr(),
                                             z.data_ptr(), kl.data_ptr(), dec.data_ptr(), mse.data_ptr(), ws.data_ptr(),
                                             ws.numel(), _ffi.current_stream()), "bg_vae_reconstruct")
    return mom, z, kl, dec, mse


@pytest.mark.parametrize("kind,hw", [("surf", 8), ("surf", 16), ("surf", 24), ("surf", 32), ("edge", 32)])
def test_moments_match_oracle_and_mean_equals_encode(kind, hw):
    m = _model(kind)
    x = _input(kind, 5, hw, seed=hw)
    sd = full_state_dict(kind)
    with torch.no_grad():
        post = m.encode(x.cuda()).latent_dist
        ref = (VP.surf_moments if kind == "surf" else VP.edge_moments)(sd, x)
        mode = _encode_mode(m, x.cuda())
    torch.cuda.synchronize()
    assert post.parameters.shape == ref.shape
    err = rel_l2(post.parameters, ref)
    print(f"{kind} moments {hw}: rel_l2={err:.3e}")
    assert err < 1e-3, err
    assert torch.equal(post.mean, mode)          # the fused tail's mean half is bg_vae_encode's output, bit for bit


@pytest.mark.parametrize("kind", ["surf", "edge"])
def test_posterior_z_kl_mse_match_fp64(kind):
    m = _model(kind)
    N = 7
    x = _input(kind, N, seed=1).cuda()
    lat = (4, 4) if kind == "surf" else (4,)
    noise = torch.randn((N, 3) + lat, generator=torch.Generator().manual_seed(2)).cuda()
    with torch.no_grad():
        m.encode(x)                               # packs the handles
        mom, z, kl, dec, mse = _reconstruct(m, x, noise)
    torch.cuda.synchronize()
    md = mom.double().cpu()
    mean, logvar = md[:, :3], md[:, 3:].clamp(-30, 20)
    z64 = mean + torch.exp(0.5 * logvar) * noise.double().cpu()
    kl64 = 0.5 * (mean ** 2 + torch.exp(logvar) - 1.0 - logvar).flatten(1).sum(1)
    mse64 = ((dec.double() - x.double()) ** 2).flatten(1).mean(1).cpu()
    ez = float((z.double().cpu() - z64).abs().max() / z64.abs().max())
    ekl = float(((kl.double().cpu() - kl64).abs() / kl64.abs()).max())
    emse = float(((mse.double().cpu() - mse64).abs() / mse64).max())
    print(f"{kind}: z {ez:.2e}  kl {ekl:.2e}  mse {emse:.2e}")
    assert ez <= 1e-6 and ekl <= 1e-5 and emse <= 1e-6, (ez, ekl, emse)
    # deterministic posterior (diffusers: std = var = 0): z = mean, kl = 0
    zd, kld = torch.empty_like(z), torch.empty_like(kl)
    _ffi.check(_ffi.lib().bg_vae_posterior(mom.data_ptr(), noise.data_ptr(), N, z[0, 0].numel(), 1, zd.data_ptr(),
                                           kld.data_ptr(), _ffi.current_stream()), "bg_vae_posterior")
    torch.cuda.synchronize()
    assert torch.equal(zd, mom[:, :3]) and torch.equal(kld, torch.zeros_like(kld))


@pytest.mark.parametrize("kind", ["surf", "edge"])
def test_reconstruct_equals_unfused_entry_points(kind):
    m = _model(kind)
    N = 6
    x = _input(kind, N, seed=3).cuda()
    lat = (4, 4) if kind == "surf" else (4,)
    noise = torch.randn((N, 3) + lat, generator=torch.Generator().manual_seed(4)).cuda()
    lib, st = _ffi.lib(), _ffi.current_stream()
    with torch.no_grad():
        m.encode(x)
        fused = _reconstruct(m, x, noise)
        mom = torch.empty_like(fused[0])
        ws = _ws(max(lib.bg_vae_workspace_bytes(m._handle, N), lib.bg_vae_workspace_bytes(m._dec, N)))
        _ffi.check(lib.bg_vae_encode_moments(m._handle, x.data_ptr(), N, 32, mom.data_ptr(), ws.data_ptr(), ws.numel(), st),
                   "bg_vae_encode_moments")
        z, kl = torch.empty_like(fused[1]), torch.empty_like(fused[2])
        _ffi.check(lib.bg_vae_posterior(mom.data_ptr(), noise.data_ptr(), N, z[0, 0].numel(), 0, z.data_ptr(), kl.data_ptr(),
                                        st), "bg_vae_posterior")
        dec = torch.empty_like(x)
        _ffi.check(lib.bg_vae_decode_hw(m._dec, z.data_ptr(), N, 4, dec.data_ptr(), ws.data_ptr(), ws.numel(), st),
                   "bg_vae_decode")
        kl_api = m.encode(x).latent_dist.kl() if kind == "surf" else None
    torch.cuda.synchronize()
    for name, a, b in zip(("moments", "z", "kl", "dec"), fused[:4], (mom, z, kl, dec)):
        assert torch.equal(a, b), name
    if kl_api is not None:
        assert torch.equal(kl_api, kl)


@pytest.mark.parametrize("kind,N,chunk", [("surf", 11, 3), ("edge", 29, 8)])
def test_graph_replayed_chunks_equal_eager(kind, N, chunk):
    m = _model(kind)
    m.chunk = chunk                               # >= 3 full chunks plus a remainder
    x = _input(kind, N, 16 if kind == "surf" else 32, seed=5).cuda()
    outs = []
    with torch.no_grad():
        for use_graph in (False, True, True):
            m.use_graph = use_graph
            dec, mse = m.reconstruct(x, sample_posterior=True, generator=torch.Generator(device="cuda").manual_seed(6))
            mom = m.encode(x).latent_dist.parameters
            outs.append((dec, mse, mom, m.decode(mom[:, :3]).sample))
    torch.cuda.synchronize()
    assert len(m._graphs) == 3                    # reconstruct, encode and decode each captured once, then re-used
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)
    for a, b in zip(outs[1], outs[2]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("kind", ["surf", "edge"])
def test_forward_matches_oracle_chain(kind):
    m = _model(kind)
    sd = full_state_dict(kind)
    x = _input(kind, 3, seed=7)
    lat = (4, 4) if kind == "surf" else (4,)
    noise = torch.randn((3, 3) + lat, generator=torch.Generator().manual_seed(8))
    moments = (VP.surf_moments if kind == "surf" else VP.edge_moments)(sd, x)
    decode = V.surf_decode if kind == "surf" else V.edge_decode
    with torch.no_grad():
        ref_s = decode(sd, VP.DiagonalGaussianDistribution(moments).sample(noise=noise))
        ref_m = decode(sd, moments[:, :3])
        y_s = m(x.cuda(), sample_posterior=True, generator=torch.Generator().manual_seed(8)).sample
        y_m = m(x.cuda(), return_dict=False)[0]
        # the posterior object alone: sample() with the same CPU generator, kl() against the oracle
        post = m.encode(x.cuda()).latent_dist
        z = post.sample(generator=torch.Generator().manual_seed(8))
        y_d = m.decode(z).sample
        ref_z = decode(sd, z.cpu())                   # the oracle decoder on the kernels' own latents
    torch.cuda.synchronize()
    e_s, e_m, e_d = rel_l2(y_s, ref_s), rel_l2(y_m, ref_m), rel_l2(y_d, ref_s)
    e_z, e_dz = rel_l2(z, VP.DiagonalGaussianDistribution(moments).sample(noise=noise)), rel_l2(y_d, ref_z)
    print(f"{kind} forward: sampled {e_s:.3e}  mode {e_m:.3e}  encode/sample/decode {e_d:.3e}  "
          f"(z {e_z:.3e}, decoder on the same z {e_dz:.3e})")
    assert torch.equal(y_s, y_d)                      # fused forward == encode -> sample -> decode, bit for bit
    assert e_z < 1e-3 and e_dz < 1e-3                 # each stage at the parity bar
    assert e_s < 1e-3 and e_m < 1e-3 and e_d < 1e-3   # and the whole chain
    if kind == "surf":
        assert rel_l2(post.kl(), VP.DiagonalGaussianDistribution(moments).kl()) < 1e-3


@pytest.mark.parametrize("kind", ["surf", "edge"])
def test_validation_matches_reference_statements(kind):
    g = np.load(GOLD)
    m = _model(kind)
    x = torch.from_numpy(g["surf_uv" if kind == "surf" else "edge_u"]).cuda()
    fn = VAL.surfvae_val_losses if kind == "surf" else VAL.edgevae_val_losses
    torch.manual_seed(SEEDS[kind])
    loss = fn(m, x, rng_device="cpu")            # the posterior noise from the CPU generator, as the golden drew it
    ref = float(g[f"loss_{kind}"])
    torch.manual_seed(SEEDS[kind])
    mse = VAL.vae_val_mse(m, [x.cpu()], edge=kind == "edge", device="cuda", rng_device="cpu")
    with torch.no_grad():
        post = m.encode(x.permute(0, 3, 1, 2) if kind == "surf" else x.permute(0, 2, 1)).latent_dist
        kl = post.kl().mean() if kind == "surf" else \
            0.5 * torch.sum(post.mean ** 2 + post.var - 1.0 - post.logvar, dim=[1, 2]).mean()
    e_loss, e_kl = abs(loss - ref) / ref, abs(float(kl) - float(g[f"kl_{kind}"])) / abs(float(g[f"kl_{kind}"]))
    e_mom = rel_l2(post.parameters, torch.from_numpy(g[f"moments_{kind}"]))
    print(f"{kind} validation: loss {e_loss:.2e}  kl {e_kl:.2e}  moments {e_mom:.2e}")
    assert e_loss < 1e-3 and e_kl < 1e-3 and e_mom < 1e-3
    assert abs(mse - ref / int(g[f"count_{kind}"])) <= 1e-3 * mse


def test_bad_arguments_are_reported_not_faulted():
    from brepgen_b200.vae import AutoencoderKL, AutoencoderKL1D
    s, e = _model("surf"), _model("edge")
    assert isinstance(s, AutoencoderKL) and isinstance(e, AutoencoderKL1D)
    lib, st = _ffi.lib(), _ffi.current_stream()
    x = _input("surf", 2).cuda()
    with torch.no_grad():
        s.encode(x)
        e.encode(_input("edge", 2).cuda())
    out, dec, mse = torch.empty(2, 6, 4, 4, device="cuda"), torch.empty_like(x), torch.empty(2, device="cuda")
    ws = _ws(lib.bg_vae_reconstruct_workspace_bytes(s._handle, s._dec, 2))

    def recon(enc, dcd, hw):
        return lib.bg_vae_reconstruct(enc, dcd, x.data_ptr(), 2, hw, None, None, None, None, dec.data_ptr(), mse.data_ptr(),
                                      ws.data_ptr(), ws.numel(), st)
    assert recon(s._handle, e._dec, 32) == -1        # surface encoder with the edge decoder
    assert recon(s._dec, s._handle, 32) == -1        # decoder in the encoder slot
    assert recon(s._handle, s._dec, 12) == -1        # an extent the handles do not take
    assert lib.bg_vae_encode_moments(s._dec, x.data_ptr(), 2, 32, out.data_ptr(), ws.data_ptr(), ws.numel(), st) == -1
    assert lib.bg_vae_posterior(None, None, 2, 16, 0, None, None, st) == -1
    with pytest.raises(RuntimeError, match="status -1"):
        _ffi.check(recon(e._handle, s._dec, 32), "bg_vae_reconstruct")
    torch.cuda.synchronize()
    assert recon(s._handle, s._dec, 32) == 0         # the handles still work
    torch.cuda.synchronize()
    assert torch.isfinite(dec).all() and torch.isfinite(mse).all()
