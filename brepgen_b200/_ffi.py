"""ctypes binding of libbrepgen_b200.so (the C ABI in include/brepgen_b200.h).

The product path has NO fallback: if the shared library is missing or the device is not sm_90 (H100), calls raise.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("BG_LIB", os.path.join(_HERE, "libbrepgen_b200.so"))   # BG_LIB: debug builds only

vp, i32, i64, u64, f32, sz = C.c_void_p, C.c_int, C.c_int64, C.c_uint64, C.c_float, C.c_size_t


class BgNamedTensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", vp), ("numel", i64)]


class BgDenoiserArgs(C.Structure):
    _fields_ = [("B", i32), ("S", i32), ("E", i32), ("x", vp), ("timesteps", vp), ("n_timesteps", i32),
                ("surfPos", vp), ("surfZ", vp), ("edgePos", vp), ("mask", vp), ("class_label", vp), ("out", vp), ("compact", i32)]


# name -> (restype, argtypes); every symbol include/brepgen_b200.h declares (tests check the export list against this)
SIGNATURES = {
    "bg_version": (i32, []),
    "bg_last_error": (C.c_char_p, []),
    "bg_check_device": (i32, []),
    "bg_launch_count": (u64, []),
    "bg_denoiser_create": (i32, [i32, i32, i32, C.POINTER(BgNamedTensor), i32, vp, vp, C.POINTER(vp)]),
    "bg_denoiser_destroy": (None, [vp]),
    "bg_denoiser_workspace_bytes": (sz, [vp, i32, i32, i32]),
    "bg_denoiser_forward": (i32, [vp, C.POINTER(BgDenoiserArgs), vp, sz, vp]),
    "bg_vae_create": (i32, [i32, C.POINTER(BgNamedTensor), i32, vp, C.POINTER(vp)]),
    "bg_vae_create_ex": (i32, [i32, i32, C.POINTER(BgNamedTensor), i32, vp, C.POINTER(vp)]),
    "bg_vae_destroy": (None, [vp]),
    "bg_vae_workspace_bytes": (sz, [vp, i32]),
    "bg_vae_decode": (i32, [vp, vp, i32, vp, vp, sz, vp]),
    "bg_vae_decode_hw": (i32, [vp, vp, i32, i32, vp, vp, sz, vp]),
    "bg_vae_encode": (i32, [vp, vp, i32, i32, vp, vp, sz, vp]),
    "bg_vae_encode_moments": (i32, [vp, vp, i32, i32, vp, vp, sz, vp]),
    "bg_vae_posterior": (i32, [vp, vp, i32, i32, i32, vp, vp, vp]),
    "bg_vae_reconstruct_workspace_bytes": (sz, [vp, vp, i32]),
    "bg_vae_reconstruct": (i32, [vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, sz, vp]),
    "bg_ddpm_step": (i32, [vp, vp, f32, vp, vp, vp, u64, u64, vp, i64, i64, i64, f32, f32, f32, f32, f32, f32, vp]),
    "bg_ddpm_step_tab": (i32, [vp, vp, f32, vp, vp, u64, u64, u64, vp, i64, vp, i64, vp, vp, f32, vp]),
    "bg_step_advance": (i32, [vp, i32, vp, vp, vp]),
    "bg_randn_keyed": (i32, [vp, i64, i64, i32, i64, vp, vp]),
    "bg_ddim_step": (i32, [vp, vp, f32, vp, vp, vp, u64, u64, vp, i64, i64, i64, f32, f32, f32, f32, f32, f32, i32, vp]),
    "bg_ddim_step_tab": (i32, [vp, vp, f32, vp, vp, u64, u64, u64, vp, i64, vp, i64, vp, vp, f32, i32, vp]),
    "bg_dpm_step": (i32, [vp, vp, f32, vp, vp, vp, vp, u64, u64, vp, i64, i64, i64, f32, f32, f32, f32, f32, f32, f32, f32,
                          vp]),
    "bg_dpm_step_tab": (i32, [vp, vp, f32, vp, vp, vp, u64, u64, u64, vp, i64, vp, i64, vp, vp, f32, vp]),
    "bg_replace_known": (i32, [vp, vp, vp, i64, i64, vp, u64, vp, i64, i64, f32, f32, vp]),
    "bg_replace_known_tab": (i32, [vp, vp, vp, i64, i64, u64, vp, i64, vp, vp, vp, vp]),
    "bg_add_noise_gather": (i32, [vp, i64, vp, i64, i32, f32, f32, f32, vp, vp, i64, i32, i64, vp, vp]),
    "bg_repaint_step": (i32, [vp, vp, f32, vp, vp, vp, vp, i64, vp, u64, vp, i64, i64, i64, f32, f32, f32, f32, f32, f32,
                              f32, vp]),
    "bg_repaint_step_tab": (i32, [vp, vp, f32, vp, vp, vp, vp, i64, u64, vp, i64, i64, vp, vp, f32, vp]),
    "bg_repaint_undo": (i32, [vp, i64, i32, vp, vp, u64, vp, i64, i64, vp]),
    "bg_repaint_undo_tab": (i32, [vp, i64, i32, u64, vp, i64, vp, vp, vp]),
    "bg_pndm_step":(i32, [vp, vp, i64, f32, f32, vp, f32, vp, f32, vp, f32, vp, f32, vp]),
    "bg_axpby": (i32, [vp, f32, vp, f32, vp, i64, vp]),
    "bg_dedup_surfaces": (i32, [vp, i32, i32, f32, vp, vp, vp]),
    "bg_dedup_edges": (i32, [vp, vp, i32, i32, i32, f32, vp, vp]),
    "bg_dedup_surfaces_index": (i32, [vp, i32, i32, f32, vp, vp, vp, vp]),
    "bg_fill_index": (i32, [vp, vp, i64, i64, i32, i32, vp, vp]),
    "bg_edge_endpoints": (i32, [vp, vp, f32, i64, vp, vp]),
    "bg_nn_exclude": (i32, [vp, vp, vp, i32, vp, vp]),
    "bg_pairs_within": (i32, [vp, i32, f32, vp, vp]),
    "bg_edge_pair_match": (i32, [vp, vp, i32, i32, f32, vp, vp]),
    "bg_edge_fit": (i32, [vp, vp, i32, vp, vp]),
    "bg_surf_init": (i32, [vp, vp, vp, vp, vp, i32, vp, vp]),
    "bg_surf_offset_opt": (i32, [vp, vp, vp, vp, vp, i32, i32, i32, f32, f32, f32, f32, f32, vp, vp, vp]),
    "bg_op_gemm_f16": (i32, [vp, i32, vp, i32, i32, i32, i32, vp, i32, i32, i32, vp, vp, i32, vp, i32, i32, vp]),
    "bg_op_gemm_f16_ex": (i32, [vp, i32, vp, i32, i32, i32, i32, vp, i32, i32, i32, vp, vp, i32, vp, i32, i32,
                                i32, i32, i32, vp, vp, vp]),
    "bg_op_conv_f16": (i32, [vp, i32, vp, i32, i32, i32, i32, i32, i32, i32, i32, i32, vp, i32, vp, vp, i32, vp]),
    "bg_op_attention": (i32, [vp, vp, i32, i32, vp, i32, vp, vp]),
    "bg_op_attention_varlen": (i32, [vp, vp, i32, i32, vp, vp, vp]),
    "bg_op_layernorm_f16": (i32, [vp, i32, vp, vp, vp, i32, i32, i32, vp]),
    "bg_op_layernorm_f16_ex": (i32, [vp, i32, vp, vp, vp, i32, i32, i32, i32, vp, vp]),
    "bg_op_cast_f16": (i32, [vp, vp, i64, vp]),
    "bg_op_embed_in": (i32, [vp, i32, i32, vp, vp, vp, vp, vp, i32, i32, vp, vp, vp]),
    "bg_op_ln_silu_head": (i32, [vp, i32, vp, vp, vp, vp, vp, i32, i32, vp, vp, vp]),
    "bg_op_compact": (i32, [vp, i32, i32, vp, vp, vp, vp, vp]),
    "bg_op_groupnorm": (i32, [vp, i32, i32, i32, i32, f32, vp, vp, i32, vp, vp, vp, vp]),
    "bg_op_vae_attention": (i32, [vp, vp, i32, i32, i32, f32, vp]),
    "bg_op_cubic1d": (i32, [vp, vp, i32, i32, i32, vp, i32, vp]),
    "bg_op_cast_split": (i32, [vp, vp, i64, i32, vp]),
    "bg_op_upsample2x_split": (i32, [vp, vp, i32, i32, i32, i32, vp]),
    "bg_op_postquant": (i32, [vp, vp, vp, vp, i32, i32, vp]),
    "bg_op_im2col": (i32, [vp, i32, vp, i32, i32, i32, i32, i32, i32, i32, i32, i32, vp]),
}

_lib: Optional[C.CDLL] = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(brepgen_b200 has no CPU / PyTorch fallback)")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype, fn.argtypes = res, args
        _lib = l
    return _lib


def check(status: int, what: str = "") -> None:
    if status != 0:
        msg = lib().bg_last_error().decode(errors="replace")
        raise RuntimeError(f"brepgen_b200 {what} failed (status {status}): {msg}")


def ptr(t) -> Optional[int]:
    """device pointer of a torch tensor (or None)"""
    return None if t is None else t.data_ptr()


def named_tensors(state_dict, device):
    """a state dict as the BgNamedTensor array bg_denoiser_create / bg_vae_create read (the array refers to the tensors'
    memory: keep them alive until the call's stream has been synchronised)"""
    import torch
    arr = (BgNamedTensor * len(state_dict))()
    for i, (k, v) in enumerate(state_dict.items()):
        if v.device != device or v.dtype != torch.float32 or not v.is_contiguous():
            raise RuntimeError(f"parameter {k} must be contiguous fp32 on {device} (call .to(device) first)")
        arr[i].name, arr[i].data, arr[i].numel = k.encode(), v.data_ptr(), v.numel()
    return arr


def current_stream() -> int:
    import torch
    return torch.cuda.current_stream().cuda_stream


# Kernels launched through CUDA-graph replays do not pass through the library's host-side launch counter (bg_launch_count
# counts a captured launch once, at capture time).  Code that replays a captured sequence adds `launches per replay` here,
# so that bench.py's `gpu_launches` = bg_launch_count() + replayed_launches is the number of kernels that really ran.
replayed_launches = 0


def note_replay(launches_per_replay: int, times: int = 1) -> None:
    global replayed_launches
    replayed_launches += int(launches_per_replay) * int(times)
