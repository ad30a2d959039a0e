"""GPU parity of the drop-in VAE decoders against the CPU fp32 oracle (oracle/vae.py; parity unpinned at the diffusers
boundary, see its header).  Tolerance: 1e-3 relative L2 (fp16 tensor-core operands, fp32 accumulation / norms)."""
import pytest
import torch

from brepgen_b200.spec import edge_decoder_spec, surf_decoder_spec
from brepgen_b200.synth import synth_state_dict
from oracle import vae as V

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("N,chunk", [(1, 1024), (5, 2)])
def test_surface_decoder(N, chunk):
    from brepgen_b200.vae import AutoencoderKLFastDecode
    sd = synth_state_dict(surf_decoder_spec(), seed=5)
    m = AutoencoderKLFastDecode(in_channels=3, out_channels=3, block_out_channels=[128, 256, 512, 512], layers_per_block=2,
                                act_fn="silu", latent_channels=3, norm_num_groups=32, sample_size=512)
    missing = m.load_state_dict({**sd, "encoder.conv_in.bias": torch.zeros(128)}, strict=False)
    assert not missing.missing_keys and missing.unexpected_keys == ["encoder.conv_in.bias"]
    m = m.cuda().eval()
    m.chunk = chunk
    z = torch.randn(N, 3, 4, 4, generator=torch.Generator().manual_seed(N))
    with torch.no_grad():
        ref = V.surf_decode(sd, z)
        y = m(z.cuda()).cpu()
    assert y.shape == (N, 3, 32, 32) and torch.isfinite(y).all()
    err = rel_l2(y, ref)
    print(f"surface decoder N={N} rel_l2={err:.3e}")
    assert err < 1e-3, err


@pytest.mark.parametrize("N,chunk", [(3, 32768), (37, 16)])
def test_edge_decoder(N, chunk):
    from brepgen_b200.vae import AutoencoderKL1DFastDecode
    sd = synth_state_dict(edge_decoder_spec(), seed=6)
    m = AutoencoderKL1DFastDecode(in_channels=3, out_channels=3, block_out_channels=[128, 256, 512], layers_per_block=2,
                                  act_fn="silu", latent_channels=3, norm_num_groups=32, sample_size=512)
    m.load_state_dict(sd, strict=False)
    m = m.cuda().eval()
    m.chunk = chunk
    z = torch.randn(N, 3, 4, generator=torch.Generator().manual_seed(N))
    with torch.no_grad():
        ref = V.edge_decode(sd, z)
        y = m(z.cuda()).cpu()
    assert y.shape == (N, 3, 32) and torch.isfinite(y).all()
    err = rel_l2(y, ref)
    print(f"edge decoder N={N} rel_l2={err:.3e}")
    assert err < 1e-3, err


def test_cascade_with_decode_shapes():
    from brepgen_b200.models import NETS
    from brepgen_b200.sampler import Cascade, CascadeConfig
    from brepgen_b200.spec import denoiser_spec
    from brepgen_b200.vae import build_synthetic_decoders
    ms = {}
    for kind in NETS:
        m = NETS[kind](False)
        m.load_state_dict(synth_state_dict(denoiser_spec(kind, False), seed=11))
        ms[kind] = m.cuda().eval()
    sv, ev = build_synthetic_decoders("cuda")
    cfg = CascadeConfig(batch_size=2, num_surfaces=3, num_edges=4, schedule="ddpm", ddpm_steps=2, seed=1)
    out = Cascade(ms, sv, ev).run(cfg)
    assert out["surf_ncs"].shape == (2, 6, 32, 32, 3) and out["edge_ncs"].shape == (2, 6, 4, 32, 3)
    assert torch.isfinite(out["surf_ncs"]).all() and torch.isfinite(out["edge_ncs"]).all()


def test_encoders_match_oracle():
    from brepgen_b200.spec import edge_encoder_spec, surf_encoder_spec
    from brepgen_b200.vae import AutoencoderKL1DFastEncode, AutoencoderKLFastEncode
    g = torch.Generator().manual_seed(21)
    sds, sde = synth_state_dict(surf_encoder_spec(), seed=7), synth_state_dict(edge_encoder_spec(), seed=8)
    es = AutoencoderKLFastEncode(block_out_channels=[128, 256, 512, 512])
    es.load_state_dict({**sds, "decoder.conv_in.bias": torch.zeros(512)}, strict=False)
    ee = AutoencoderKL1DFastEncode(block_out_channels=[128, 256, 512])
    ee.load_state_dict(sde, strict=False)
    es, ee = es.cuda().eval(), ee.cuda().eval()
    for hw in (16, 32):
        x = torch.rand(3, 3, hw, hw, generator=g) * 2 - 1
        with torch.no_grad():
            ref, y = V.surf_encode(sds, x), es(x.cuda()).cpu()
        assert y.shape == (3, 3, hw // 8, hw // 8)
        err = rel_l2(y, ref)
        print(f"surface encoder {hw}x{hw} rel_l2={err:.3e}")
        assert err < 1e-3, err
    x = torch.rand(5, 3, 32, generator=g) * 2 - 1
    with torch.no_grad():
        ref, y = V.edge_encode(sde, x), ee(x.cuda()).cpu()
    err = rel_l2(y, ref)
    print(f"edge encoder rel_l2={err:.3e}")
    assert y.shape == (5, 3, 4) and err < 1e-3, err


def test_config1_roundtrip():
    """BASELINE.json configs[0]: surface VAE encode -> decode round trip, batch 4 of 16x16x3 grids (and the edge
    analogue, batch 4 of 32x3), through the drop-in classes vs the oracle, U(-1,1) inputs seed 0 (SURVEY 8d item 1)."""
    from brepgen_b200.spec import edge_encoder_spec, surf_encoder_spec
    from brepgen_b200.vae import (AutoencoderKL1DFastDecode, AutoencoderKL1DFastEncode, AutoencoderKLFastDecode,
                                  AutoencoderKLFastEncode)
    g = torch.Generator().manual_seed(0)
    full_s = {**synth_state_dict(surf_encoder_spec(), 9), **synth_state_dict(surf_decoder_spec(), 9)}   # a "full AE" checkpoint
    full_e = {**synth_state_dict(edge_encoder_spec(), 9), **synth_state_dict(edge_decoder_spec(), 9)}
    mods = []
    for cls, sd in ((AutoencoderKLFastEncode, full_s), (AutoencoderKLFastDecode, full_s),
                    (AutoencoderKL1DFastEncode, full_e), (AutoencoderKL1DFastDecode, full_e)):
        m = cls()
        m.load_state_dict(sd, strict=False)
        mods.append(m.cuda().eval())
    es, ds, ee, de = mods
    x = torch.rand(4, 3, 16, 16, generator=g) * 2 - 1
    with torch.no_grad():
        ref = V.surf_decode_any(full_s, V.surf_encode(full_s, x))
        y = ds(es(x.cuda())).cpu()
    assert y.shape == (4, 3, 16, 16)
    e1 = rel_l2(y, ref)
    xe = torch.rand(4, 3, 32, generator=g) * 2 - 1
    with torch.no_grad():
        refe = V.edge_decode(full_e, V.edge_encode(full_e, xe))
        ye = de(ee(xe.cuda())).cpu()
    e2 = rel_l2(ye, refe)
    print(f"config-1 round trip: surface 16x16 rel_l2={e1:.3e}  edge rel_l2={e2:.3e}")
    assert e1 < 1e-3 and e2 < 1e-3


def test_training_side_latent_pass():
    """the frozen-encoder pass that feeds LDM training (trainer.py:518-524, 918-928): surfPnt (B,S,32,32,3) -> surfZ (B,S,48),
    edgePnt (B,S,E,32,3) -> edgeZ (B,S,E,12), with the reference's reshapes around the drop-in encoders; against the same
    statements around the oracle encoders"""
    from brepgen_b200.spec import edge_encoder_spec, surf_encoder_spec
    from brepgen_b200.vae import (AutoencoderKL1DFastEncode, AutoencoderKLFastEncode, encode_edge_latents,
                                  encode_surface_latents)
    g = torch.Generator().manual_seed(4)
    sd_s, sd_e = synth_state_dict(surf_encoder_spec(), 5), synth_state_dict(edge_encoder_spec(), 5)
    es, ee = AutoencoderKLFastEncode(), AutoencoderKL1DFastEncode()
    es.load_state_dict(sd_s, strict=False)
    ee.load_state_dict(sd_e, strict=False)
    es, ee = es.cuda().eval(), ee.cuda().eval()
    B, S, E, zs = 2, 3, 4, 1.0
    surfPnt = torch.rand(B, S, 32, 32, 3, generator=g) * 2 - 1
    edgePnt = torch.rand(B, S, E, 32, 3, generator=g) * 2 - 1
    with torch.no_grad():
        surfZ = encode_surface_latents(es, surfPnt.cuda(), zs).cpu()
        edgeZ = encode_edge_latents(ee, edgePnt.cuda(), zs).cpu()
        # the reference's statements (trainer.py:919-928) around the oracle encoders
        sz = V.surf_encode(sd_s, surfPnt.flatten(0, 1).permute(0, 3, 1, 2))
        sz = sz.unflatten(0, (B, -1)).flatten(-2, -1).permute(0, 1, 3, 2).flatten(-2, -1) * zs
        ez = V.edge_encode(sd_e, edgePnt.flatten(0, 1).flatten(0, 1).permute(0, 2, 1))
        ez = ez.unflatten(0, (-1, E)).unflatten(0, (B, -1)).permute(0, 1, 2, 4, 3).flatten(-2, -1) * zs
    assert surfZ.shape == (B, S, 48) and edgeZ.shape == (B, S, E, 12)
    e1, e2 = rel_l2(surfZ, sz), rel_l2(edgeZ, ez)
    print(f"training-side latent pass: surfZ rel_l2={e1:.3e} edgeZ rel_l2={e2:.3e}")
    assert e1 < 1e-3 and e2 < 1e-3


def test_decoders_graph_replay_equals_eager():
    """many chunks per call: one chunk is captured in a CUDA graph and replayed (vae.py); results identical to eager chunks"""
    from brepgen_b200.vae import build_synthetic_decoders
    sv, ev = build_synthetic_decoders(torch.device("cuda"))
    sv.chunk, ev.chunk = 3, 8
    zs = torch.randn(14, 3, 4, 4, generator=torch.Generator().manual_seed(1)).cuda()     # 4 full chunks + 2
    ze = torch.randn(43, 3, 4, generator=torch.Generator().manual_seed(2)).cuda()        # 5 full chunks + 3
    with torch.no_grad():
        sv.use_graph = ev.use_graph = False
        a_s, a_e = sv(zs), ev(ze)
        sv.use_graph = ev.use_graph = True
        b_s, b_e = sv(zs), ev(ze)
        c_s = sv(zs)                                  # second call re-uses the captured chunk
    torch.cuda.synchronize()
    assert len(sv._graphs) == 1 and len(ev._graphs) == 1
    assert torch.equal(a_s, b_s) and torch.equal(a_e, b_e) and torch.equal(b_s, c_s)


def test_implicit_convolutions_equal_explicit_im2col():
    """the implicit-GEMM convolutions (TMA boxes of the image per tap) and the explicit im2col gather + GEMM run the same
    k-block order through the same MMA, so the decoders' and the encoders' outputs are bit-identical; the switch is read at
    handle creation"""
    import os
    from brepgen_b200.spec import edge_encoder_spec, surf_encoder_spec
    from brepgen_b200.vae import AutoencoderKL1DFastEncode, AutoencoderKLFastEncode, build_synthetic_decoders
    dev = torch.device("cuda")
    zs = torch.randn(37, 3, 4, 4, generator=torch.Generator().manual_seed(3)).cuda()      # 37 * 16 rows: a ragged last tile
    ze = torch.randn(203, 3, 4, generator=torch.Generator().manual_seed(4)).cuda()
    g = torch.Generator().manual_seed(5)
    xs = (torch.rand(37, 3, 32, 32, generator=g) * 2 - 1).cuda()   # 4 x 4 at the encoder's conv_out: 37 * 16 rows again
    xe = (torch.rand(203, 3, 32, generator=g) * 2 - 1).cuda()
    outs = []
    for explicit in (0, 1):
        os.environ["BREPGEN_B200_VAE_IM2COL"] = str(explicit)
        try:
            sv, ev = build_synthetic_decoders(dev)
            es, ee = AutoencoderKLFastEncode(), AutoencoderKL1DFastEncode()
            es.load_state_dict(synth_state_dict(surf_encoder_spec(), seed=7), strict=False)
            ee.load_state_dict(synth_state_dict(edge_encoder_spec(), seed=8), strict=False)
            mods = (sv, ev, es.to(dev).eval(), ee.to(dev).eval())
            for m in mods:
                m.use_graph = False
            with torch.no_grad():
                outs.append([m(x) for m, x in zip(mods, (zs, ze, xs, xe))])
            torch.cuda.synchronize()
        finally:
            os.environ.pop("BREPGEN_B200_VAE_IM2COL", None)
    for implicit, explicit in zip(*outs):
        assert torch.isfinite(implicit).all()
        assert torch.equal(implicit, explicit)
