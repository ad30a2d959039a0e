"""Weight packing rejects an incomplete or mis-shaped checkpoint: bg_denoiser_create / bg_vae_create return
BG_STATUS_MISSING_WEIGHT for a missing key and BG_STATUS_BAD_ARG for a tensor of the wrong size, and bg_last_error
names the weight (include/brepgen_b200.h)."""
import ctypes as C

import pytest
import torch

from brepgen_b200 import _ffi
from brepgen_b200.spec import denoiser_spec, edge_encoder_spec, surf_decoder_spec

pytestmark = pytest.mark.gpu

MISSING_WEIGHT, BAD_ARG = -5, -1


def _create(kind, sd):
    arr = _ffi.named_tensors(sd, torch.device("cuda", torch.cuda.current_device()))
    out = C.c_void_p()
    if kind.startswith("vae"):
        status = _ffi.lib().bg_vae_create(int(kind[-1]), arr, len(arr), _ffi.current_stream(), C.byref(out))
    else:
        status = _ffi.lib().bg_denoiser_create(3, 0, 1, arr, len(arr), None, _ffi.current_stream(), C.byref(out))
    torch.cuda.synchronize()
    assert status != 0 and not out.value, "create accepted a broken checkpoint"
    return status, _ffi.lib().bg_last_error().decode()


@pytest.mark.parametrize("kind,spec,key", [
    ("denoiser", denoiser_spec("edgez", False), "net.layers.5.self_attn.in_proj_weight"),
    ("vae0", surf_decoder_spec(), "decoder.mid_block.attentions.0.to_k.weight"),
    ("vae3", edge_encoder_spec(), "encoder.down_blocks.1.resnets.0.conv_skip.weight"),
])
def test_missing_or_misshaped_weight_is_named(kind, spec, key):
    sd = {k: torch.zeros(shape, device="cuda") for k, shape in spec}
    assert key in sd
    status, msg = _create(kind, {k: v for k, v in sd.items() if k != key})
    assert status == MISSING_WEIGHT and key in msg, (status, msg)
    status, msg = _create(kind, {**sd, key: torch.zeros(sd[key].numel() + 1, device="cuda")})
    assert status == BAD_ARG and key in msg, (status, msg)
