"""State-dict specifications (key -> shape) of the hot-path networks.

These are the reference's checkpoint layouts, which are part of the drop-in boundary
(SURVEY.md §8b): `sample.py:56-70` does `Net(use_cf).load_state_dict(torch.load(path))`.

  denoisers : network.py:1066-1105 (SurfPosNet), :1129-1174 (SurfZNet),
              :1203-1255 (EdgePosNet), :1289-1355 (EdgeZNet); encoder = nn.TransformerEncoder
              (12 pre-norm layers d=768, 12 heads, FFN 1024) + final LayerNorm.
"""
from __future__ import annotations

from typing import List, Tuple

D = 768          # embed_dim, network.py:1073
H = 12           # nhead,     network.py:1076
DH = 64
FF = 1024        # dim_feedforward, network.py:1077
NLAYER = 12      # network.py:1078
NCLASS = 11      # Embedder(11, 768), network.py:1102

# kind -> (ordered embed-MLP names with input widths, output width)
NET_KINDS = {
    "surfpos": ([("p_embed", 6)], 6),
    "surfz": ([("z_embed", 48), ("p_embed", 6)], 48),
    "edgepos": ([("surfz_embed", 48), ("surfp_embed", 6), ("edgep_embed", 6)], 6),
    "edgez": ([("surfz_embed", 48), ("edgez_embed", 12), ("surfp_embed", 6),
               ("edgep_embed", 6), ("vertp_fc", 6)], 18),
}

Spec = List[Tuple[str, Tuple[int, ...]]]


def _mlp(name: str, d_in: int, d_out: int) -> Spec:
    # nn.Sequential(Linear(d_in,768), LayerNorm(768), SiLU, Linear(768,d_out)) -> indices 0,1,3
    return [
        (f"{name}.0.weight", (D, d_in)), (f"{name}.0.bias", (D,)),
        (f"{name}.1.weight", (D,)), (f"{name}.1.bias", (D,)),
        (f"{name}.3.weight", (d_out, D)), (f"{name}.3.bias", (d_out,)),
    ]


def encoder_spec(prefix: str = "net") -> Spec:
    out: Spec = []
    for i in range(NLAYER):
        p = f"{prefix}.layers.{i}"
        out += [
            (f"{p}.self_attn.in_proj_weight", (3 * D, D)), (f"{p}.self_attn.in_proj_bias", (3 * D,)),
            (f"{p}.self_attn.out_proj.weight", (D, D)), (f"{p}.self_attn.out_proj.bias", (D,)),
            (f"{p}.linear1.weight", (FF, D)), (f"{p}.linear1.bias", (FF,)),
            (f"{p}.linear2.weight", (D, FF)), (f"{p}.linear2.bias", (D,)),
            (f"{p}.norm1.weight", (D,)), (f"{p}.norm1.bias", (D,)),
            (f"{p}.norm2.weight", (D,)), (f"{p}.norm2.bias", (D,)),
        ]
    out += [(f"{prefix}.norm.weight", (D,)), (f"{prefix}.norm.bias", (D,))]
    return out


def denoiser_spec(kind: str, use_cf: bool) -> Spec:
    embeds, d_out = NET_KINDS[kind]
    out = encoder_spec("net")
    for name, d_in in embeds:
        out += _mlp(name, d_in, D)
    out += _mlp("time_embed", D, D)
    out += _mlp("fc_out", D, d_out)
    if use_cf:
        out += [("class_embed.embed.weight", (NCLASS, D))]
    return out


# ------------------------------------------------------------------------------------------------ VAE decoders
# Checkpoints hold the full auto-encoders; sample.py:83,98 load them with strict=False into decoder-only modules, so
# only `decoder.*` and `post_quant_conv.*` keys matter (SURVEY.md Appendix A.1 / A.2 key lists).
def _conv(name: str, cout: int, cin: int, *k: int, bias: bool = True) -> Spec:
    out: Spec = [(f"{name}.weight", (cout, cin) + tuple(k))]
    if bias:
        out.append((f"{name}.bias", (cout,)))
    return out


def _norm(name: str, c: int) -> Spec:
    return [(f"{name}.weight", (c,)), (f"{name}.bias", (c,))]


def _resnet2d(name: str, cin: int, cout: int) -> Spec:
    out = _norm(f"{name}.norm1", cin) + _conv(f"{name}.conv1", cout, cin, 3, 3)
    out += _norm(f"{name}.norm2", cout) + _conv(f"{name}.conv2", cout, cout, 3, 3)
    if cin != cout:
        out += _conv(f"{name}.conv_shortcut", cout, cin, 1, 1)
    return out


def surf_decoder_spec() -> Spec:
    """AutoencoderKLFastDecode (network.py:948-1040) = diffusers 0.27 `Decoder`, cfg sample.py:72-82:
    block_out_channels [128,256,512,512], layers_per_block 2 (-> 3 resnets per up block), latent 3, groups 32."""
    d = "decoder"
    out = _conv("post_quant_conv", 3, 3, 1, 1)
    out += _conv(f"{d}.conv_in", 512, 3, 3, 3)
    out += _resnet2d(f"{d}.mid_block.resnets.0", 512, 512)
    a = f"{d}.mid_block.attentions.0"
    out += _norm(f"{a}.group_norm", 512)
    for n in ("to_q", "to_k", "to_v"):
        out += [(f"{a}.{n}.weight", (512, 512)), (f"{a}.{n}.bias", (512,))]
    out += [(f"{a}.to_out.0.weight", (512, 512)), (f"{a}.to_out.0.bias", (512,))]
    out += _resnet2d(f"{d}.mid_block.resnets.1", 512, 512)
    chans = [(512, 512), (512, 512), (512, 256), (256, 128)]
    for i, (cin, cout) in enumerate(chans):
        for j in range(3):
            out += _resnet2d(f"{d}.up_blocks.{i}.resnets.{j}", cin if j == 0 else cout, cout)
        if i < 3:
            out += _conv(f"{d}.up_blocks.{i}.upsamplers.0.conv", cout, cout, 3, 3)
    out += _norm(f"{d}.conv_norm_out", 128) + _conv(f"{d}.conv_out", 3, 128, 3, 3)
    return out


def _resconv1d(name: str, cin: int, cmid: int, cout: int) -> Spec:
    out: Spec = []
    if cin != cout:
        out += _conv(f"{name}.conv_skip", cout, cin, 1, bias=False)
    out += _conv(f"{name}.conv_1", cmid, cin, 5) + _norm(f"{name}.group_norm_1", cmid)
    out += _conv(f"{name}.conv_2", cout, cmid, 5) + _norm(f"{name}.group_norm_2", cout)
    return out


def edge_decoder_spec() -> Spec:
    """AutoencoderKL1DFastDecode (network.py:786-858) -> Decoder1D (:188-299), cfg sample.py:86-97:
    block_out_channels [128,256,512]; mid = 6 x (ResConvBlock + SelfAttention1d(512, 16 heads)) (network.py:51-83);
    3 UpBlock1D (network.py:30-48) each 3 ResConvBlocks + cubic Upsample1d (buffer `up.kernel`, 8 taps)."""
    d = "decoder"
    out = _conv("post_quant_conv", 3, 3, 1)
    out += _conv(f"{d}.conv_in", 512, 3, 3)
    for i in range(6):
        out += _resconv1d(f"{d}.mid_block.resnets.{i}", 512, 512, 512)
    for i in range(6):
        a = f"{d}.mid_block.attentions.{i}"
        out += _norm(f"{a}.group_norm", 512)
        for n in ("query", "key", "value", "proj_attn"):
            out += [(f"{a}.{n}.weight", (512, 512)), (f"{a}.{n}.bias", (512,))]
    for i, (cin, cout) in enumerate([(512, 512), (512, 256), (256, 128)]):
        b = f"{d}.up_blocks.{i}"
        out += _resconv1d(f"{b}.resnets.0", cin, cin, cin)
        out += _resconv1d(f"{b}.resnets.1", cin, cin, cin)
        out += _resconv1d(f"{b}.resnets.2", cin, cin, cout)
        out += [(f"{b}.up.kernel", (8,))]
    out += _norm(f"{d}.conv_norm_out", 128) + _conv(f"{d}.conv_out", 3, 128, 3)
    return out


CUBIC_UP_KERNEL = [2 * v for v in (-0.01171875, -0.03515625, 0.11328125, 0.43359375, 0.43359375, 0.11328125,
                                   -0.03515625, -0.01171875)]   # diffusers Upsample1d("cubic") buffer (kernel * 2)


# ------------------------------------------------------------------------------------------------ VAE encoders
CUBIC_DOWN_KERNEL = [v / 2 for v in CUBIC_UP_KERNEL]      # diffusers Downsample1d("cubic") buffer (un-doubled taps)


def surf_encoder_spec() -> Spec:
    """AutoencoderKLFastEncode (network.py:861-945) = diffusers 0.27 `Encoder` + quant_conv; block_out_channels
    [128,256,512,512], layers_per_block 2, double_z (6 output channels), trainer.py:20-30 / SURVEY Appendix A.1."""
    e = "encoder"
    out = _conv(f"{e}.conv_in", 128, 3, 3, 3)
    chans = [(128, 128), (128, 256), (256, 512), (512, 512)]
    for i, (cin, cout) in enumerate(chans):
        for j in range(2):
            out += _resnet2d(f"{e}.down_blocks.{i}.resnets.{j}", cin if j == 0 else cout, cout)
        if i < 3:
            out += _conv(f"{e}.down_blocks.{i}.downsamplers.0.conv", cout, cout, 3, 3)
    out += _resnet2d(f"{e}.mid_block.resnets.0", 512, 512)
    a = f"{e}.mid_block.attentions.0"
    out += _norm(f"{a}.group_norm", 512)
    for n in ("to_q", "to_k", "to_v"):
        out += [(f"{a}.{n}.weight", (512, 512)), (f"{a}.{n}.bias", (512,))]
    out += [(f"{a}.to_out.0.weight", (512, 512)), (f"{a}.to_out.0.bias", (512,))]
    out += _resnet2d(f"{e}.mid_block.resnets.1", 512, 512)
    out += _norm(f"{e}.conv_norm_out", 512) + _conv(f"{e}.conv_out", 6, 512, 3, 3)
    out += _conv("quant_conv", 6, 6, 1, 1)
    return out


def edge_encoder_spec() -> Spec:
    """AutoencoderKL1DFastEncode (network.py:690-783) -> Encoder1D (:86-185): conv_in k3 3->128, three diffusers
    DownBlock1D (cubic Downsample1d first, then ResConvBlock(in,out,out), (out,out,out), (out,out,out)), the 1-D mid block
    (6 x ResConvBlock + SelfAttention1d), GroupNorm32 + SiLU + conv_out 512->6, quant_conv."""
    e = "encoder"
    out = _conv(f"{e}.conv_in", 128, 3, 3)
    for i, (cin, cout) in enumerate([(128, 128), (128, 256), (256, 512)]):
        b = f"{e}.down_blocks.{i}"
        out += [(f"{b}.down.kernel", (8,))]
        out += _resconv1d(f"{b}.resnets.0", cin, cout, cout)
        out += _resconv1d(f"{b}.resnets.1", cout, cout, cout)
        out += _resconv1d(f"{b}.resnets.2", cout, cout, cout)
    for i in range(6):
        out += _resconv1d(f"{e}.mid_block.resnets.{i}", 512, 512, 512)
    for i in range(6):
        a = f"{e}.mid_block.attentions.{i}"
        out += _norm(f"{a}.group_norm", 512)
        for n in ("query", "key", "value", "proj_attn"):
            out += [(f"{a}.{n}.weight", (512, 512)), (f"{a}.{n}.bias", (512,))]
    out += _norm(f"{e}.conv_norm_out", 512) + _conv(f"{e}.conv_out", 6, 512, 3)
    out += _conv("quant_conv", 6, 6, 1)
    return out
