"""ctypes binding of libmeshanything_b200.so (include/meshanything_b200.h).

The library is built in-tree by `meshanything_b200.build` (nvcc, sm_90a).  There is no CPU or
PyTorch fallback: if the shared object cannot be loaded every call raises.
"""
from __future__ import annotations

import ctypes as C
import math
import numbers
import operator
import os
from typing import Optional

import torch

from . import build as _build

MA_MAX_LAYERS = 32
EPI_NONE, EPI_RELU, EPI_GELU = 0, 1, 2
GEN_NO_GRAPH, GEN_NO_FAST, GEN_NO_PDL, GEN_NO_EARLY_EXIT, GEN_NO_MEGA, GEN_TC = 1, 2, 4, 8, 16, 64

_vp = C.c_void_p


class DecoderWeights(C.Structure):
    _fields_ = (
        [("n_layers", C.c_int), ("vocab", C.c_int), ("codebook", C.c_int), ("npos", C.c_int)]
        + [(n, _vp * MA_MAX_LAYERS) for n in ("wqkv", "bqkv", "wo", "bo", "w1", "b1", "w2", "b2",
                                              "ln1g", "ln1b", "ln2g", "ln2b")]
        + [(n, _vp) for n in ("lm_head", "tok_table", "extra", "tok_pos", "cond", "pos")]
    )


class Sampling(C.Structure):
    _fields_ = [("do_sample", C.c_int), ("top_k", C.c_int), ("top_p", C.c_float), ("seed", C.c_uint64)]


_lib = None

EXPORTS = [
    "ma_abi_version", "ma_last_error", "ma_launch_count", "ma_linear_f16", "ma_layernorm",
    "ma_attention_scratch_bytes", "ma_attention_f16", "ma_attention_decode_f16", "ma_kv_cache_bytes", "ma_decoder_workspace_bytes",
    "ma_decode_generate", "ma_encoder_workspace_bytes", "ma_encoder_forward",
    "ma_detokenize_workspace_bytes", "ma_detokenize", "ma_linear_tc_f16", "ma_set_tensor_cores", "ma_sample_tokens",
    "ma_attention_tc_f16", "ma_transpose_heads_f16",
    "ma_decode_slots_init", "ma_decode_slot_prefill", "ma_decode_slots_step", "ma_decode_slots_poll",
    "ma_linear_ws_set_mode", "ma_decode_slots_seek", "ma_decode_slot_stream", "ma_linear_ws_scratch_bytes", "ma_linear_ws_f16",
    "ma_sample_surface_workspace_bytes", "ma_sample_surface", "ma_tensor_core_linear_counts", "ma_decode_persistent_supported",
    "ma_udf_grid", "ma_marching_cubes_workspace_bytes", "ma_marching_cubes_count", "ma_marching_cubes_emit",
    "ma_mesh_score_workspace_bytes", "ma_mesh_score",
    "ma_estimate_normals_workspace_bytes", "ma_estimate_normals", "ma_estimate_normals_set_events",
    "ma_estimate_normals_last_rounds",
    "ma_remove_outliers_workspace_bytes", "ma_remove_outliers", "ma_remove_outliers_set_events",
    "ma_farthest_point_sample_workspace_bytes", "ma_farthest_point_sample", "ma_farthest_point_sample_set_path",
    "ma_farthest_point_sample_last_path",
    "ma_remove_plane_workspace_bytes", "ma_remove_plane", "ma_remove_plane_set_events",
    "ma_split_objects_workspace_bytes", "ma_split_objects", "ma_split_objects_set_events",
    "ma_smooth_points_workspace_bytes", "ma_smooth_points", "ma_smooth_points_set_events", "ma_smooth_points_set_order",
    "ma_transfer_colors_workspace_bytes", "ma_transfer_colors", "ma_transfer_colors_set_events",
    "ma_fourier_embed_f16", "ma_scatter_heads_f16", "ma_residual_add", "ma_convert_rows", "ma_add_table",
    "ma_gather_codes", "ma_coords",
]
FPS_AUTO, FPS_ONE_CTA, FPS_GRID_SHARED, FPS_GRID_GLOBAL = 0, 1, 2, 3   # ma_farthest_point_sample_set_path


def lib_path() -> str:
    return _build.LIB


def lib():
    """Load (building if stale and nvcc is available) the shared library."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB
    # rebuild when the library is older than its sources -- in a development checkout only (.git present, nvcc
    # available): the GPU box gets the prebuilt file with a snapshot whose mtimes are those of the copy
    dev_tree = os.path.isdir(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), ".git"))
    stale = (os.path.exists(path) and dev_tree and _build.have_nvcc()
             and os.environ.get("MA_B200_NO_AUTOBUILD") != "1" and _build._stale())
    if not os.path.exists(path) or stale or (os.environ.get("MA_B200_REBUILD") == "1"):
        path = _build.build(force=True)
    L = C.CDLL(path)
    L.ma_abi_version.restype = C.c_int
    L.ma_last_error.restype = C.c_char_p
    L.ma_launch_count.restype = C.c_ulonglong
    L.ma_linear_f16.argtypes = [_vp, _vp, _vp, C.c_int, _vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _vp]
    L.ma_layernorm.argtypes = [_vp, _vp, _vp, _vp, C.c_float, C.c_int, C.c_int, _vp, _vp, _vp]
    L.ma_attention_scratch_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
    L.ma_attention_scratch_bytes.restype = C.c_size_t
    L.ma_attention_f16.argtypes = [_vp, C.c_int, _vp, _vp, C.c_long, C.c_int, _vp, _vp, C.c_int, C.c_int,
                                   C.c_float, _vp, C.c_int, _vp, _vp]
    L.ma_kv_cache_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
    L.ma_kv_cache_bytes.restype = C.c_size_t
    L.ma_decoder_workspace_bytes.argtypes = [C.c_int, C.c_int]
    L.ma_decoder_workspace_bytes.restype = C.c_size_t
    L.ma_decode_generate.argtypes = [C.POINTER(DecoderWeights), _vp, C.c_int, C.c_int, C.c_int, C.POINTER(Sampling),
                                     C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, C.c_int, _vp]
    L.ma_sample_tokens.argtypes = [_vp, C.c_int, C.c_int, C.POINTER(Sampling), _vp, _vp, _vp]
    L.ma_attention_decode_f16.argtypes = [_vp, C.c_int, _vp, _vp, C.c_long, _vp, C.c_int, C.c_int, C.c_float, _vp, C.c_int,
                                          _vp, _vp]
    L.ma_attention_tc_f16.argtypes = [_vp, C.c_int, _vp, _vp, C.c_long, C.c_long, C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.c_float, _vp, C.c_int, _vp]
    L.ma_transpose_heads_f16.argtypes = [_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_long, C.c_int, _vp, _vp]
    L.ma_decode_slots_init.argtypes = [C.c_int, C.c_int, C.c_int, _vp, _vp]
    L.ma_linear_ws_set_mode.argtypes = [C.c_int]
    L.ma_linear_ws_set_mode.restype = None
    L.ma_decode_slot_stream.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, _vp, _vp]
    L.ma_decode_slots_seek.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _vp, _vp]
    L.ma_decode_slot_prefill.argtypes = [C.POINTER(DecoderWeights), _vp, C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.POINTER(Sampling), C.c_int, C.c_int, _vp, _vp, _vp, _vp]
    L.ma_decode_slots_step.argtypes = [C.POINTER(DecoderWeights), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                       C.POINTER(Sampling), C.c_int, C.c_int, _vp, _vp, _vp, C.c_int, _vp]
    L.ma_decode_slots_poll.argtypes = [C.c_int, C.c_int, _vp, _vp, _vp, _vp]
    L.ma_decode_persistent_supported.argtypes = []
    L.ma_decode_persistent_supported.restype = C.c_int
    L.ma_encoder_workspace_bytes.argtypes = [C.c_int]
    L.ma_encoder_workspace_bytes.restype = C.c_size_t
    L.ma_encoder_forward.argtypes = [_vp, _vp, C.c_int, _vp, _vp, _vp, _vp]
    L.ma_detokenize_workspace_bytes.argtypes = [C.c_int, C.c_int]
    L.ma_detokenize_workspace_bytes.restype = C.c_size_t
    L.ma_detokenize.argtypes = [_vp, _vp, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp]
    L.ma_linear_ws_scratch_bytes.restype = C.c_size_t
    L.ma_linear_ws_f16.argtypes = [_vp, _vp, _vp, C.c_int, _vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _vp, _vp]
    L.ma_sample_surface_workspace_bytes.argtypes = [C.c_int]
    L.ma_sample_surface_workspace_bytes.restype = C.c_size_t
    L.ma_sample_surface.argtypes = [_vp, _vp, C.c_int, C.c_int, C.c_ulonglong, _vp, _vp, _vp, _vp]
    L.ma_udf_grid.argtypes = [_vp, _vp, C.c_int, C.c_int, C.c_float, _vp, _vp]
    L.ma_marching_cubes_workspace_bytes.argtypes = [C.c_int]
    L.ma_marching_cubes_workspace_bytes.restype = C.c_size_t
    L.ma_marching_cubes_count.argtypes = [_vp, C.c_int, C.c_float, _vp, C.POINTER(C.c_int64), _vp]
    L.ma_marching_cubes_emit.argtypes = [_vp, C.c_int, C.c_float, _vp, _vp, _vp, _vp]
    L.ma_mesh_score_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int]
    L.ma_mesh_score_workspace_bytes.restype = C.c_size_t
    L.ma_mesh_score.argtypes = [_vp, _vp, C.c_int, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]
    L.ma_estimate_normals_workspace_bytes.argtypes = [C.c_int, C.c_int]
    L.ma_estimate_normals_workspace_bytes.restype = C.c_size_t
    L.ma_estimate_normals.argtypes = [_vp, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp]
    L.ma_estimate_normals_set_events.argtypes = [_vp]
    L.ma_estimate_normals_set_events.restype = None
    L.ma_estimate_normals_last_rounds.argtypes = []
    L.ma_estimate_normals_last_rounds.restype = C.c_int
    L.ma_remove_outliers_workspace_bytes.argtypes = [C.c_int, C.c_int]
    L.ma_remove_outliers_workspace_bytes.restype = C.c_size_t
    L.ma_remove_outliers.argtypes = [_vp, C.c_int, C.c_int, C.c_double, C.c_double, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                     _vp]
    L.ma_remove_outliers_set_events.argtypes = [_vp]
    L.ma_remove_outliers_set_events.restype = None
    L.ma_farthest_point_sample_workspace_bytes.argtypes = [C.c_int, C.c_int]
    L.ma_farthest_point_sample_workspace_bytes.restype = C.c_size_t
    L.ma_farthest_point_sample.argtypes = [_vp, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp, _vp]
    L.ma_farthest_point_sample_set_path.argtypes = [C.c_int]
    L.ma_farthest_point_sample_set_path.restype = C.c_int
    L.ma_farthest_point_sample_last_path.argtypes = []
    L.ma_farthest_point_sample_last_path.restype = C.c_int
    L.ma_remove_plane_workspace_bytes.argtypes = [C.c_int, C.c_int]
    L.ma_remove_plane_workspace_bytes.restype = C.c_size_t
    L.ma_remove_plane.argtypes = [_vp, C.c_int, C.c_int, C.c_float, C.c_ulonglong, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                  _vp]
    L.ma_remove_plane_set_events.argtypes = [_vp]
    L.ma_remove_plane_set_events.restype = None
    L.ma_split_objects_workspace_bytes.argtypes = [C.c_int, C.c_int]
    L.ma_split_objects_workspace_bytes.restype = C.c_size_t
    L.ma_split_objects.argtypes = [_vp, C.c_int, C.c_float, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp]
    L.ma_split_objects_set_events.argtypes = [_vp]
    L.ma_split_objects_set_events.restype = None
    L.ma_smooth_points_workspace_bytes.argtypes = [C.c_int, C.c_int]
    L.ma_smooth_points_workspace_bytes.restype = C.c_size_t
    L.ma_smooth_points.argtypes = [_vp, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp]
    L.ma_smooth_points_set_events.argtypes = [_vp]
    L.ma_smooth_points_set_events.restype = None
    L.ma_smooth_points_set_order.argtypes = [C.c_int]
    L.ma_smooth_points_set_order.restype = None
    L.ma_transfer_colors_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
    L.ma_transfer_colors_workspace_bytes.restype = C.c_size_t
    L.ma_transfer_colors.argtypes = [_vp, C.c_int, _vp, C.c_int, _vp, _vp, C.c_int, C.c_float, _vp, _vp, _vp, _vp, _vp,
                                     _vp, _vp, _vp, _vp]
    L.ma_transfer_colors_set_events.argtypes = [_vp]
    L.ma_transfer_colors_set_events.restype = None
    L.ma_fourier_embed_f16.argtypes = [_vp, C.c_long, _vp, _vp]
    L.ma_scatter_heads_f16.argtypes = [_vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_long, _vp, C.c_long, _vp]
    L.ma_residual_add.argtypes = [_vp, _vp, _vp, C.c_long, _vp]
    L.ma_convert_rows.argtypes = [_vp, C.c_int, C.c_long, _vp, C.c_int, C.c_long, C.c_long, C.c_int, C.c_long, _vp]
    L.ma_add_table.argtypes = [_vp, _vp, _vp, C.c_int, _vp, C.c_long, _vp]
    L.ma_gather_codes.argtypes = [_vp, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp, _vp, _vp]
    L.ma_coords.argtypes = [_vp, _vp, _vp, C.c_long, _vp]
    L.ma_linear_tc_f16.argtypes = [_vp, _vp, _vp, C.c_int, _vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _vp]
    L.ma_set_tensor_cores.argtypes = [C.c_int]
    L.ma_tensor_core_linear_counts.argtypes = [C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong)]
    L.ma_tensor_core_linear_counts.restype = None
    if L.ma_abi_version() != 1:
        raise RuntimeError("libmeshanything_b200.so: ABI version mismatch")
    _lib = L
    return L


def check(rc: int, what: str):
    if rc != 0:
        raise RuntimeError(f"{what} failed: {lib().ma_last_error().decode()}")


def ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("meshanything_b200: tensors must live on a CUDA device (no CPU fallback)")


def _check_points(what: str, points, n_min: int) -> int:
    """N of a cloud handed to a point-cloud entry point: ValueError unless `points` is a contiguous fp32 [N, 3] CUDA
    tensor of finite coordinates with n_min <= N <= 2^24."""
    if not isinstance(points, torch.Tensor):
        raise ValueError(f"{what}: points must be a torch tensor, got {type(points).__name__}")
    if points.dim() != 2 or points.shape[1] != 3:
        raise ValueError(f"{what}: points [N, 3], got {tuple(points.shape)}")
    if points.dtype != torch.float32:
        raise ValueError(f"{what}: points must be float32, got {points.dtype}")
    if not points.is_contiguous():
        raise ValueError(f"{what}: points must be contiguous")
    if not points.is_cuda:
        raise ValueError(f"{what}: points must live on a CUDA device (no CPU fallback)")
    n = points.shape[0]
    if not n_min <= n <= 1 << 24:
        raise ValueError(f"{what}: {n_min} <= N <= 2^24, got N = {n}")
    if not bool(torch.isfinite(points).all()):
        raise ValueError(f"{what}: non-finite coordinates")
    return n


def _check_int(what: str, name: str, value, lo: int, hi: int) -> int:
    """`value` as an int in [lo, hi]; ValueError otherwise, and for bool, which operator.index would accept."""
    if isinstance(value, bool):
        raise ValueError(f"{what}: {name} must be an integer, got {value!r}")
    try:
        value = operator.index(value)
    except TypeError:
        raise ValueError(f"{what}: {name} must be an integer, got {value!r}") from None
    if not lo <= value <= hi:
        raise ValueError(f"{what}: {lo} <= {name} <= {hi}, got {value}")
    return value


def _check_share(what: str, name: str, value, square: bool = False) -> float:
    """`value`, a share of the frame's side, rounded to fp32: ValueError unless it is a finite real number in (0, 1]
    that stays above 0 in fp32 and, with `square`, whose fp32 square stays above 0 too."""
    if isinstance(value, bool):
        raise ValueError(f"{what}: {name} must be a real number")
    try:
        value = float(value)
    except (TypeError, ValueError):
        raise ValueError(f"{what}: {name} must be a real number, got {value!r}") from None
    v32 = C.c_float(value).value
    if not (math.isfinite(value) and 0 < value <= 1 and 0 < v32 <= 1 and (not square or C.c_float(v32 * v32).value > 0)):
        rule = "its fp32 square > 0" if square else "> 0 in fp32"
        raise ValueError(f"{what}: 0 < {name} <= 1 (and {rule}), got {value}")
    return v32


# ---------------------------------------------------------------- canonical building blocks

def linear_f16(w: torch.Tensor, bias: Optional[torch.Tensor], x: torch.Tensor, epilogue: int = EPI_NONE,
               out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp16(x @ w.T + bias) with the canonical accumulation order.  w [N,K] fp16, x [M,K] fp16."""
    _need_cuda(w, bias, x)
    assert w.dtype == torch.float16 and x.dtype == torch.float16 and w.is_contiguous()
    assert x.dim() == 2 and x.stride(1) == 1
    M, K = x.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=torch.float16, device=x.device)
    check(lib().ma_linear_f16(ptr(w), ptr(bias), ptr(x), x.stride(0), ptr(out), out.stride(0), M, N, K, epilogue,
                              stream_ptr()), "ma_linear_f16")
    return out


def sample_surface(vertices: torch.Tensor, faces: torch.Tensor, n_samples: int, seed: int = 0,
                   want_index: bool = False):
    """Area-weighted surface samples + face normals on the GPU: fp16 [n_samples, 6] (and the face of every sample).

    vertices [V, 3] finite, faces [F, 3] with indices in [0, V), F >= 1, n_samples >= 1, 0 <= seed < 2^64.  Every bad
    input raises ValueError before anything is launched.  A mesh whose faces all have zero area gets the last face and a
    zero normal for every sample (DESIGN.md section 1.5)."""
    _need_cuda(vertices, faces)
    if vertices.dim() != 2 or vertices.shape[1] != 3 or faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError(f"sample_surface: vertices [V, 3] and faces [F, 3], got {tuple(vertices.shape)} and "
                         f"{tuple(faces.shape)}")
    if faces.shape[0] < 1:
        raise ValueError("sample_surface: a mesh without faces has no surface to sample")
    try:
        n_samples, seed = operator.index(n_samples), operator.index(seed)
    except TypeError:
        raise ValueError(f"sample_surface: n_samples and seed must be integers, got {n_samples!r}, {seed!r}") from None
    if not 1 <= n_samples < 1 << 31:
        raise ValueError(f"sample_surface: 1 <= n_samples < 2^31, got {n_samples}")
    if not 0 <= seed < 1 << 64:
        raise ValueError(f"sample_surface: 0 <= seed < 2^64, got {seed}")
    if faces.dtype.is_floating_point or faces.dtype.is_complex or faces.dtype == torch.bool:
        raise ValueError(f"sample_surface: integer face indices, got {faces.dtype}")
    V = vertices.shape[0]
    if int(faces.min()) < 0 or int(faces.max()) >= V:
        raise ValueError(f"sample_surface: face indices outside [0, {V})")
    v = vertices.to(torch.float32).contiguous()
    if not bool(torch.isfinite(v).all()):
        raise ValueError("sample_surface: non-finite vertex coordinates")
    f = faces.to(torch.int32).contiguous()
    F = f.shape[0]
    ws = torch.empty(lib().ma_sample_surface_workspace_bytes(F), dtype=torch.uint8, device=v.device)
    out = torch.empty((n_samples, 6), dtype=torch.float16, device=v.device)
    idx = torch.empty((n_samples,), dtype=torch.int32, device=v.device) if want_index else None
    check(lib().ma_sample_surface(ptr(v), ptr(f), F, n_samples, int(seed), ptr(out), ptr(idx), ptr(ws), stream_ptr()),
          "ma_sample_surface")
    return (out, idx) if want_index else out


# ---------------------------------------------------------------- glue kernels of the encoder / detokenizer (test hooks)

def fourier_embed_f16(pc: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """pc fp16 [rows, 6] -> fp16 [rows, 256] = [xyz | sin 24 | cos 24 | normal | zeros] (a1 of the encoder)."""
    _need_cuda(pc, out)
    assert pc.dtype == torch.float16 and pc.is_contiguous() and pc.dim() == 2 and pc.shape[1] == 6
    rows = pc.shape[0]
    if out is None:
        out = torch.empty((rows, 256), dtype=torch.float16, device=pc.device)
    assert out.dtype == torch.float16 and out.is_contiguous() and out.numel() >= rows * 256
    check(lib().ma_fourier_embed_f16(ptr(pc), rows, ptr(out), stream_ptr()), "ma_fourier_embed_f16")
    return out


def scatter_heads_f16(src: torch.Tensor, col0: int, head_stride: int, H: int, rows_per_slot: int, T: int,
                      dst: torch.Tensor, rows: Optional[int] = None) -> torch.Tensor:
    """Head slices of src fp16 [rows, ld] into dst (flat fp16, >= (rows / rows_per_slot) * H * T * 64 elements):
    dst[((slot H + h) T + t) 64 + d] = src[m, col0 + h head_stride + d], slot = m // rows_per_slot,
    t = m % rows_per_slot."""
    _need_cuda(src, dst)
    assert src.dtype == torch.float16 and dst.dtype == torch.float16 and src.stride(1) == 1 and dst.is_contiguous()
    rows = src.shape[0] if rows is None else rows
    check(lib().ma_scatter_heads_f16(ptr(src), src.stride(0), col0, head_stride, H, rows_per_slot, T, ptr(dst), rows,
                                     stream_ptr()), "ma_scatter_heads_f16")
    return dst


def residual_add(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """In place: x fp32 += float(y), or x fp16 = fp16(float(x) + float(y)); y fp16, numel % 4 == 0."""
    _need_cuda(x, y)
    assert x.is_contiguous() and y.is_contiguous() and y.dtype == torch.float16 and x.numel() == y.numel()
    x32, x16 = (x, None) if x.dtype == torch.float32 else (None, x)
    check(lib().ma_residual_add(ptr(x32), ptr(x16), ptr(y), x.numel(), stream_ptr()), "ma_residual_add")
    return x


def convert_rows(src: torch.Tensor, dst: torch.Tensor, rows: int, cols: int, src_rows_mod: int = 0) -> torch.Tensor:
    """dst[r, :cols] = src[r % src_rows_mod (or r), :cols] converted to dst's dtype (fp16 / fp32); src and dst may be
    row-strided views: their stride(0) is passed as lds / ldd."""
    _need_cuda(src, dst)
    assert src.dtype in (torch.float16, torch.float32) and dst.dtype in (torch.float16, torch.float32)
    assert src.stride(1) == 1 and dst.stride(1) == 1
    check(lib().ma_convert_rows(ptr(src), int(src.dtype == torch.float16), src.stride(0), ptr(dst),
                                int(dst.dtype == torch.float16), dst.stride(0), rows, cols, src_rows_mod, stream_ptr()),
          "ma_convert_rows")
    return dst


def add_table(y16: torch.Tensor, table: torch.Tensor, mask: Optional[torch.Tensor] = None,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp32 [rows, 768] = (mask[r] ? float(y16[r]) : 0) + table[r % table_rows]."""
    _need_cuda(y16, table, mask, out)
    assert y16.dtype == torch.float16 and table.dtype == torch.float32 and y16.is_contiguous() and table.is_contiguous()
    assert y16.shape[1] == 768 and table.shape[1] == 768 and (mask is None or mask.dtype == torch.int32)
    if out is None:
        out = torch.empty((y16.shape[0], 768), dtype=torch.float32, device=y16.device)
    assert out.dtype == torch.float32 and out.is_contiguous() and out.shape == (y16.shape[0], 768)
    check(lib().ma_add_table(ptr(y16), ptr(mask), ptr(table), table.shape[0], ptr(out), y16.shape[0], stream_ptr()),
          "ma_add_table")
    return out


def gather_codes(gen_ids: torch.Tensor, F: int, codebook: torch.Tensor, out=None):
    """gen_ids int32 [B, max_new] -> (code16 fp16 [B*F, 3072], mask int32 [B*F], ids int32 [B*F, 9]); `out` may give
    the three destination tensors."""
    _need_cuda(gen_ids, codebook)
    assert gen_ids.dtype == torch.int32 and gen_ids.is_contiguous() and codebook.dtype == torch.float32
    assert codebook.is_contiguous() and codebook.shape[1] == 1024
    B, max_new = gen_ids.shape
    dev = gen_ids.device
    code16, mask, ids = out if out is not None else (
        torch.empty((B * F, 3072), dtype=torch.float16, device=dev), torch.empty((B * F,), dtype=torch.int32, device=dev),
        torch.empty((B * F, 9), dtype=torch.int32, device=dev))
    check(lib().ma_gather_codes(ptr(gen_ids), max_new, B, F, ptr(codebook), ptr(code16), ptr(mask), ptr(ids),
                                stream_ptr()), "ma_gather_codes")
    return code16, mask, ids


def coords(logits: torch.Tensor, mask: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """logits fp16 [faces, 1152] -> fp32 [faces, 9] = argmax bin / 128 - 0.5 (lowest index on ties), NaN where mask is 0."""
    _need_cuda(logits, mask, out)
    assert logits.dtype == torch.float16 and logits.is_contiguous() and logits.shape[1] == 1152
    assert mask.dtype == torch.int32 and mask.is_contiguous()
    faces = logits.shape[0]
    if out is None:
        out = torch.empty((faces, 9), dtype=torch.float32, device=logits.device)
    check(lib().ma_coords(ptr(logits), ptr(mask), ptr(out), faces, stream_ptr()), "ma_coords")
    return out


def udf_grid(vertices: torch.Tensor, faces: torch.Tensor, n: int, band: Optional[float] = None) -> torch.Tensor:
    """Narrow-band unsigned distance field fp32 [n, n, n]: field[i, j, k] = min(band, distance from the grid point
    (-1 + i dx, -1 + j dx, -1 + k dx), dx = 2/n, to the nearest face); band defaults to 3 dx."""
    _need_cuda(vertices, faces)
    v = vertices.to(torch.float32).contiguous()
    f = faces.to(torch.int32).contiguous()
    if v.dim() != 2 or v.shape[1] != 3 or f.dim() != 2 or f.shape[1] != 3:
        raise ValueError("udf_grid: vertices [V, 3] and faces [F, 3]")
    if not bool(torch.isfinite(v).all()):
        raise ValueError("udf_grid: non-finite vertex coordinates")
    if f.numel() and (int(f.min()) < 0 or int(f.max()) >= v.shape[0]):
        raise ValueError(f"udf_grid: face indices outside [0, {v.shape[0]})")
    if not 2 <= n <= 1024:
        raise ValueError("udf_grid: 2 <= n <= 1024")
    band = 3.0 * 2.0 / n if band is None else float(band)
    out = torch.empty((n, n, n), dtype=torch.float32, device=v.device)
    check(lib().ma_udf_grid(ptr(v), ptr(f), f.shape[0], n, C.c_float(band), ptr(out), stream_ptr()), "ma_udf_grid")
    return out


def marching_cubes(field: torch.Tensor, level: float):
    """Marching cubes of fp32 [n, n, n] at `level` -> (vertices fp32 [V, 3] in index space, faces int32 [T, 3]); the
    faces' right-hand normals point toward increasing field.  Reads the two counts back once (synchronises)."""
    _need_cuda(field)
    fld = field.to(torch.float32).contiguous()
    n = fld.shape[0]
    if fld.dim() != 3 or fld.shape != (n, n, n) or not 2 <= n <= 1024:
        raise ValueError("marching_cubes: field [n, n, n], 2 <= n <= 1024")
    ws = torch.empty(lib().ma_marching_cubes_workspace_bytes(n), dtype=torch.uint8, device=fld.device)
    counts = (C.c_int64 * 2)()
    check(lib().ma_marching_cubes_count(ptr(fld), n, C.c_float(level), ptr(ws), counts, stream_ptr()),
          "ma_marching_cubes_count")
    verts = torch.empty((counts[0], 3), dtype=torch.float32, device=fld.device)
    tris = torch.empty((counts[1], 3), dtype=torch.int32, device=fld.device)
    check(lib().ma_marching_cubes_emit(ptr(fld), n, C.c_float(level), ptr(ws), ptr(verts), ptr(tris), stream_ptr()),
          "ma_marching_cubes_emit")
    return verts, tris


def mesh_score(meshes: torch.Tensor, clouds: torch.Tensor, want_terms: bool = False):
    """Chamfer terms of S x N candidate meshes against their clouds (ma_mesh_score; metrics.score adds the frame map).

    meshes fp32 [S, N, F, 3, 3] (NaN rows = absent faces), clouds fp32 [S, P, 6] already in the output frame.
    Returns (terms fp64 [S, N, 4] = p2m, m2p, nc_p, nc_m; valid faces int32 [S, N]); with want_terms also the
    per-point (distance fp32 [S, N, P], face int32) and per-quadrature-point (distance fp32 [S, N, F, 16], cloud index
    int32) results."""
    _need_cuda(meshes, clouds)
    m = meshes.to(torch.float32).contiguous()
    c = clouds.to(torch.float32).contiguous()
    if m.dim() != 5 or tuple(m.shape[3:]) != (3, 3) or c.dim() != 3 or c.shape[2] != 6 or c.shape[0] != m.shape[0]:
        raise ValueError("mesh_score: meshes [S, N, F, 3, 3] and clouds [S, P, 6]")
    S, N, F = m.shape[:3]
    P = c.shape[1]
    if min(S, N, F, P) < 1 or S * N > 65535:
        raise ValueError("mesh_score: S, N, F, P >= 1 and S * N <= 65535")
    if m.device != c.device:
        raise ValueError("mesh_score: meshes and clouds on different devices")
    if not bool(torch.isfinite(c).all()):
        raise ValueError("mesh_score: non-finite cloud")
    if not bool(torch.isfinite(m[~torch.isnan(m[..., 0, 0])]).all()):
        raise ValueError("mesh_score: non-finite coordinates in a valid face (only a NaN first coordinate marks a face "
                         "absent)")
    dev = m.device
    ws = torch.empty(lib().ma_mesh_score_workspace_bytes(S, N, F, P), dtype=torch.uint8, device=dev)
    out = torch.empty((S, N, 4), dtype=torch.float64, device=dev)
    faces = torch.empty((S, N), dtype=torch.int32, device=dev)
    extra = (torch.empty((S, N, P), dtype=torch.float32, device=dev), torch.empty((S, N, P), dtype=torch.int32, device=dev),
             torch.empty((S, N, F, 16), dtype=torch.float32, device=dev),
             torch.empty((S, N, F, 16), dtype=torch.int32, device=dev)) if want_terms else (None,) * 4
    check(lib().ma_mesh_score(ptr(m), ptr(c), S, N, F, P, ptr(out), ptr(faces), *[ptr(t) for t in extra], ptr(ws),
                              stream_ptr()), "ma_mesh_score")
    return (out, faces, *extra) if want_terms else (out, faces)


def estimate_normals(points: torch.Tensor, k: int = 16, want_terms: bool = False):
    """Oriented unit normals of a bare cloud (ma_estimate_normals; normals.estimate_normals adds the frame map).

    points fp32 [N, 3], contiguous, on a CUDA device, finite, already in the output frame; 1 <= k <= 64,
    k < N <= 2^24.  Returns normals fp32 [N, 3]; with want_terms (normals, kNN int32 [N, k] in rank order, unoriented
    normals fp32 [N, 3]).  Every bad input raises ValueError before anything is launched."""
    k = _check_int("estimate_normals", "k", k, 1, 64)
    n = _check_points("estimate_normals", points, k + 1)
    dev = points.device
    ws = torch.empty(lib().ma_estimate_normals_workspace_bytes(n, k), dtype=torch.uint8, device=dev)
    out = torch.empty((n, 3), dtype=torch.float32, device=dev)
    knn = torch.empty((n, k), dtype=torch.int32, device=dev) if want_terms else None
    uno = torch.empty((n, 3), dtype=torch.float32, device=dev) if want_terms else None
    with torch.cuda.device(dev):
        check(lib().ma_estimate_normals(ptr(points), n, k, ptr(out), ptr(knn), ptr(uno), ptr(ws), stream_ptr()),
              "ma_estimate_normals")
    return (out, knn, uno) if want_terms else out


def remove_outliers(points: torch.Tensor, k: int = 16, std_ratio: float = 2.0, min_component: float = 0.01,
                    want_terms: bool = False):
    """Outlier removal of a cloud (ma_remove_outliers; outliers.remove_outliers adds the frame map).

    points fp32 [N, 3], contiguous, on a CUDA device, finite, already in the output frame; 1 <= k <= 64,
    k < N <= 2^24.  Returns (kept indices int64 [n_kept] ascending, keep mask bool [N], stats fp64 [8] on the host: mu,
    sigma, threshold, statistical inliers, components, components dropped, kept points, connectivity rounds); with
    want_terms also (mean neighbour distance fp64 [N], kNN int32 [N, k] in rank order).  Every bad input raises
    ValueError before anything is launched.  Reads the stats back (synchronises)."""
    k = _check_int("remove_outliers", "k", k, 1, 64)
    n = _check_points("remove_outliers", points, k + 1)
    if not math.isfinite(std_ratio):
        raise ValueError(f"remove_outliers: std_ratio must be finite, got {std_ratio}")
    if not (math.isfinite(min_component) and min_component >= 0):
        raise ValueError(f"remove_outliers: min_component must be finite and >= 0, got {min_component}")
    dev = points.device
    ws = torch.empty(lib().ma_remove_outliers_workspace_bytes(n, k), dtype=torch.uint8, device=dev)
    keep = torch.empty((n,), dtype=torch.uint8, device=dev)
    idx = torch.empty((n,), dtype=torch.int64, device=dev)
    n_kept = torch.empty((1,), dtype=torch.int64, device=dev)
    stats = torch.empty((8,), dtype=torch.float64, device=dev)
    mean = torch.empty((n,), dtype=torch.float64, device=dev) if want_terms else None
    knn = torch.empty((n, k), dtype=torch.int32, device=dev) if want_terms else None
    with torch.cuda.device(dev):
        check(lib().ma_remove_outliers(ptr(points), n, k, C.c_double(std_ratio), C.c_double(min_component), ptr(keep),
                                       ptr(idx), ptr(n_kept), ptr(mean), ptr(knn), ptr(stats), ptr(ws), stream_ptr()),
              "ma_remove_outliers")
        st = stats.cpu().numpy()
    out = (idx[:int(st[6])], keep.bool(), st)
    return (*out, mean, knn) if want_terms else out


def farthest_point_sample(points: torch.Tensor, m: int, start: int = 0):
    """Farthest-point subsampling of a cloud (ma_farthest_point_sample; subsample.farthest_point_sample adds the frame
    map).

    points fp32 [N, 3], contiguous, on a CUDA device, finite, already in the output frame; 1 <= m <= N <= 2^24,
    0 <= start < N.  Returns (picks int64 [m] in pick order, r2 fp32 [m]: r2[t] the squared covering radius of the first
    t + 1 picks), both on the device.  Every bad input raises ValueError before anything is launched."""
    n = _check_points("farthest_point_sample", points, 1)
    m = _check_int("farthest_point_sample", "m", m, 1, n)
    start = _check_int("farthest_point_sample", "start", start, 0, n - 1)
    dev = points.device
    ws = torch.empty(lib().ma_farthest_point_sample_workspace_bytes(n, m), dtype=torch.uint8, device=dev)
    idx = torch.empty((m,), dtype=torch.int64, device=dev)
    r2 = torch.empty((m,), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        check(lib().ma_farthest_point_sample(ptr(points), n, m, start, ptr(idx), ptr(r2), ptr(ws), stream_ptr()),
              "ma_farthest_point_sample")
    return idx, r2


PLANE_MAX_H = 65536


def remove_plane(points: torch.Tensor, distance: float = 0.01, iterations: int = 1000, seed: int = 0,
                 want_terms: bool = False):
    """Removal of the dominant plane of a cloud (ma_remove_plane; plane.remove_plane adds the frame map).

    points fp32 [N, 3], contiguous, on a CUDA device, finite, already in the output frame; 3 <= N <= 2^24; distance the
    on-plane threshold t in the frame, 0 < t <= 1 (rounded to fp32, which must stay > 0); 1 <= iterations <= 65536
    hypotheses; an integer seed in [0, 2^64).  Returns (kept indices int64 [n_kept] ascending, keep mask bool [N],
    stats fp64 [12] on the host: found, nx, ny, nz, d, winning hypothesis, its count, valid hypotheses, on, above,
    below, kept); with want_terms also (on-plane count int32 [H] and plane fp32 [H, 4] of every hypothesis).  Every bad
    input raises ValueError before anything is launched.  Reads the stats back (synchronises)."""
    n = _check_points("remove_plane", points, 3)
    iterations = _check_int("remove_plane", "iterations", iterations, 1, PLANE_MAX_H)
    seed = _check_int("remove_plane", "seed", seed, 0, (1 << 64) - 1)
    t32 = _check_share("remove_plane", "distance", distance)
    dev = points.device
    ws = torch.empty(lib().ma_remove_plane_workspace_bytes(n, iterations), dtype=torch.uint8, device=dev)
    keep = torch.empty((n,), dtype=torch.uint8, device=dev)
    idx = torch.empty((n,), dtype=torch.int64, device=dev)
    n_kept = torch.empty((1,), dtype=torch.int64, device=dev)
    stats = torch.empty((12,), dtype=torch.float64, device=dev)
    counts = torch.empty((iterations,), dtype=torch.int32, device=dev) if want_terms else None
    planes = torch.empty((iterations, 4), dtype=torch.float32, device=dev) if want_terms else None
    with torch.cuda.device(dev):
        check(lib().ma_remove_plane(ptr(points), n, iterations, C.c_float(t32), seed, ptr(keep), ptr(idx), ptr(n_kept),
                                    ptr(counts), ptr(planes), ptr(stats), ptr(ws), stream_ptr()), "ma_remove_plane")
        st = stats.cpu().numpy()
    out = (idx[:int(st[11])], keep.bool(), st)
    return (*out, counts, planes) if want_terms else out


def split_objects(points: torch.Tensor, distance: float = 0.02, min_points: int = 4096):
    """Splitting a cloud into objects (ma_split_objects; objects.split_objects adds the frame map).

    points fp32 [N, 3], contiguous, on a CUDA device, finite, already in the output frame; 1 <= N <= 2^24; distance
    the neighbour distance e in the frame, 0 < e <= 1 (rounded to fp32; fp32(e e) must stay > 0); 1 <= min_points <= N.
    Returns (labels int32 [N], object indices int64 [points in objects], offsets int64 [objects + 1], stats int64 [6]
    on the host: clusters, objects, points in objects, dropped clusters, points in dropped clusters, largest dropped
    cluster).  Every bad input raises ValueError before anything is launched.  Reads the stats back (synchronises)."""
    n = _check_points("split_objects", points, 1)
    min_points = _check_int("split_objects", "min_points", min_points, 1, n)
    e32 = _check_share("split_objects", "distance", distance, square=True)
    dev = points.device
    ws = torch.empty(lib().ma_split_objects_workspace_bytes(n, min_points), dtype=torch.uint8, device=dev)
    labels = torch.empty((n,), dtype=torch.int32, device=dev)
    idx = torch.empty((n,), dtype=torch.int64, device=dev)
    offsets = torch.empty((n // min_points + 1,), dtype=torch.int64, device=dev)
    stats = torch.empty((6,), dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        check(lib().ma_split_objects(ptr(points), n, C.c_float(e32), min_points, ptr(labels), ptr(idx), ptr(offsets),
                                     ptr(stats), ptr(ws), stream_ptr()), "ma_split_objects")
        st = stats.cpu().numpy()
    return labels, idx[:int(st[2])], offsets[:int(st[1]) + 1], st


SMOOTH_MIN_K = 5


def smooth_points(points: torch.Tensor, k: int = 24, want_terms: bool = False):
    """Moving-least-squares smoothing of a cloud (ma_smooth_points; smooth.smooth_points adds the frame map and the way
    back to the input's units).

    points fp32 [N, 3], contiguous, on a CUDA device, finite, already in the output frame; 5 <= k <= 64,
    k < N <= 2^24.  Returns (smoothed points fp32 [N, 3] in the frame, stats int64 [3] on the host: quadratic fits,
    singular fallbacks, far fallbacks); with want_terms also (unit normal of every local frame fp32 [N, 3], outcome
    uint8 [N]: 0 quadratic, 1 singular, 2 far, kNN int32 [N, k] in rank order).  Every bad input raises ValueError
    before anything is launched.  Reads the stats back (synchronises)."""
    k = _check_int("smooth_points", "k", k, SMOOTH_MIN_K, 64)
    n = _check_points("smooth_points", points, k + 1)
    dev = points.device
    ws = torch.empty(lib().ma_smooth_points_workspace_bytes(n, k), dtype=torch.uint8, device=dev)
    out = torch.empty((n, 3), dtype=torch.float32, device=dev)
    stats = torch.empty((3,), dtype=torch.int64, device=dev)
    normals = torch.empty((n, 3), dtype=torch.float32, device=dev) if want_terms else None
    flags = torch.empty((n,), dtype=torch.uint8, device=dev) if want_terms else None
    knn = torch.empty((n, k), dtype=torch.int32, device=dev) if want_terms else None
    with torch.cuda.device(dev):
        check(lib().ma_smooth_points(ptr(points), n, k, ptr(out), ptr(normals), ptr(flags), ptr(knn), ptr(stats),
                                     ptr(ws), stream_ptr()), "ma_smooth_points")
        st = stats.cpu().numpy()
    return (out, st, normals, flags, knn) if want_terms else (out, st)


COLORS_MAX_F = 1 << 16
COLORS_MAX_V = 3 * COLORS_MAX_F


def transfer_colors(vertices: torch.Tensor, faces: torch.Tensor, points: torch.Tensor, colors: torch.Tensor,
                    r: float, want_terms: bool = False):
    """The colours of a scan carried onto a mesh (ma_transfer_colors; colors.transfer_colors adds the frame map).

    vertices fp32 [V, 3] and points fp32 [N, 3], finite and already in the points' frame; faces int32 [F, 3] with
    indices in [0, V); colors fp32 [N, 3] in [0, 1]; all contiguous on one CUDA device; 1 <= V <= 196608,
    1 <= F <= 65536, 1 <= N <= 2^24; r > 0 finite (rounded to fp32, which must stay > 0).  Returns (vertex colours fp32
    [V, 3], stats int64 [3] on the host: points used, points beyond r, fallback vertices); with want_terms also (nearest
    face int32 [N], its distance fp32 [N], weights fp32 [N, 3], sums uint64 as int64 [V, 4] = W, C_r, C_g, C_b, fallback
    flags uint8 [V]).  Every bad input raises ValueError before anything is launched.  Reads the stats back
    (synchronises)."""
    what = "transfer_colors"
    n = _check_points(what, points, 1)
    dev = points.device
    for name, t, rows in (("vertices", vertices, None), ("colors", colors, n)):
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"{what}: {name} must be a torch tensor, got {type(t).__name__}")
        if t.dim() != 2 or t.shape[1] != 3 or (rows is not None and t.shape[0] != rows):
            raise ValueError(f"{what}: {name} [{'N' if rows else 'V'}, 3], got {tuple(t.shape)}")
        if t.dtype != torch.float32 or not t.is_contiguous() or t.device != dev:
            raise ValueError(f"{what}: {name} must be contiguous float32 on {dev}, got {t.dtype} on {t.device}")
        if not bool(torch.isfinite(t).all()):
            raise ValueError(f"{what}: non-finite {name}")
    if not bool(((colors >= 0) & (colors <= 1)).all()):
        raise ValueError(f"{what}: colors outside [0, 1]")
    V = vertices.shape[0]
    if not 1 <= V <= COLORS_MAX_V:
        raise ValueError(f"{what}: 1 <= V <= {COLORS_MAX_V}, got V = {V}")
    if not isinstance(faces, torch.Tensor):
        raise ValueError(f"{what}: faces must be a torch tensor, got {type(faces).__name__}")
    if faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError(f"{what}: faces [F, 3], got {tuple(faces.shape)}")
    if faces.dtype != torch.int32 or not faces.is_contiguous() or faces.device != dev:
        raise ValueError(f"{what}: faces must be contiguous int32 on {dev}, got {faces.dtype} on {faces.device}")
    F = faces.shape[0]
    if not 1 <= F <= COLORS_MAX_F:
        raise ValueError(f"{what}: 1 <= F <= {COLORS_MAX_F}, got F = {F}")
    if int(faces.min()) < 0 or int(faces.max()) >= V:
        raise ValueError(f"{what}: face indices outside [0, {V})")
    if isinstance(r, bool) or not isinstance(r, numbers.Real):
        raise ValueError(f"{what}: r must be a real number, got {r!r}")
    r = float(r)
    r32 = C.c_float(r).value
    if not (math.isfinite(r) and math.isfinite(r32) and r32 > 0):
        raise ValueError(f"{what}: r > 0 and finite (also in fp32), got {r}")
    ws = torch.empty(lib().ma_transfer_colors_workspace_bytes(V, F, n), dtype=torch.uint8, device=dev)
    out = torch.empty((V, 3), dtype=torch.float32, device=dev)
    stats = torch.empty((3,), dtype=torch.int64, device=dev)
    extra = (torch.empty((n,), dtype=torch.int32, device=dev), torch.empty((n,), dtype=torch.float32, device=dev),
             torch.empty((n, 3), dtype=torch.float32, device=dev), torch.empty((V, 4), dtype=torch.int64, device=dev),
             torch.empty((V,), dtype=torch.uint8, device=dev)) if want_terms else (None,) * 5
    with torch.cuda.device(dev):
        check(lib().ma_transfer_colors(ptr(vertices), V, ptr(faces), F, ptr(points), ptr(colors), n, C.c_float(r32),
                                       ptr(out), ptr(stats), *[ptr(t) for t in extra], ptr(ws), stream_ptr()),
              "ma_transfer_colors")
        st = stats.cpu().numpy()
    return (out, st, *extra) if want_terms else (out, st)


def tensor_core_linear_counts():
    """(Linear calls of the encoder / detokenizer that ran on the tensor cores, calls that fell back to the canonical kernel)."""
    a, b = C.c_ulonglong(0), C.c_ulonglong(0)
    lib().ma_tensor_core_linear_counts(C.byref(a), C.byref(b))
    return a.value, b.value


_ws_scratch = {}


def _linear_out(out: Optional[torch.Tensor], M: int, N: int, device) -> torch.Tensor:
    if out is None:
        return torch.empty((M, N), dtype=torch.float16, device=device)
    _need_cuda(out)
    assert out.dtype == torch.float16 and out.shape == (M, N) and out.stride(1) == 1
    return out


def linear_ws_f16(w: torch.Tensor, bias: Optional[torch.Tensor], x: torch.Tensor, epilogue: int = EPI_NONE,
                  out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp16(x @ w.T + bias) for M <= 128 rows on the weight-streaming wgmma GEMM (hardware accumulation order).
    x and out may be row-strided views (a column slice of a wider buffer): their stride(0) is passed as ldx / ldy."""
    _need_cuda(w, bias, x)
    assert x.dim() == 2 and x.stride(1) == 1
    M, K = x.shape
    N = w.shape[0]
    scr = _ws_scratch.get(x.device)
    if scr is None:
        scr = _ws_scratch[x.device] = torch.zeros(lib().ma_linear_ws_scratch_bytes(), dtype=torch.uint8, device=x.device)
    out = _linear_out(out, M, N, x.device)
    check(lib().ma_linear_ws_f16(ptr(w), ptr(bias), ptr(x), x.stride(0), ptr(out), out.stride(0), M, N, K, epilogue,
                                 ptr(scr), stream_ptr()), "ma_linear_ws_f16")
    return out


def linear_tc_f16(w: torch.Tensor, bias: Optional[torch.Tensor], x: torch.Tensor, epilogue: int = EPI_NONE,
                  out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp16(x @ w.T + bias) on the wgmma tensor cores (hardware accumulation order).
    x and out may be row-strided views (a column slice of a wider buffer): their stride(0) is passed as ldx / ldy."""
    _need_cuda(w, bias, x)
    assert x.dim() == 2 and x.stride(1) == 1
    M, K = x.shape
    N = w.shape[0]
    out = _linear_out(out, M, N, x.device)
    check(lib().ma_linear_tc_f16(ptr(w), ptr(bias), ptr(x), x.stride(0), ptr(out), out.stride(0), M, N, K, epilogue,
                                 stream_ptr()), "ma_linear_tc_f16")
    return out


def transpose_heads_f16(src: torch.Tensor, col0: int, head_stride: int, H: int, n: int, n_slots: int) -> torch.Tensor:
    """src fp16 [n_slots*n, ld] -> V^T fp16 [n_slots, H, 64, Tpad] (Tpad = n rounded up to 128, zero padded)."""
    _need_cuda(src)
    Tpad = (n + 127) // 128 * 128
    dst = torch.empty((n_slots, H, 64, Tpad), dtype=torch.float16, device=src.device)
    check(lib().ma_transpose_heads_f16(ptr(src), src.stride(0), col0, head_stride, H, n, Tpad, n_slots, ptr(dst),
                                       stream_ptr()), "ma_transpose_heads_f16")
    return dst


def attention_tc_f16(q: torch.Tensor, k: torch.Tensor, vt: torch.Tensor, nkeys: int, rows_per_slot: int,
                     scale: float = 0.125) -> torch.Tensor:
    """q [n_slots*rows_per_slot, H*64]; k [n_slots, H, T, 64]; vt [n_slots, H, 64, Tpad] (V transposed, zero beyond
    nkeys) -> [rows, H*64], on the wgmma tensor cores."""
    _need_cuda(q, k, vt)
    S, H, T, _ = k.shape
    Tpad = vt.shape[3]
    assert q.is_contiguous() and k.is_contiguous() and vt.is_contiguous() and q.shape[0] == S * rows_per_slot
    out = torch.empty_like(q)
    check(lib().ma_attention_tc_f16(ptr(q), q.stride(0), ptr(k), ptr(vt), T, Tpad, H, rows_per_slot, S, nkeys,
                                    C.c_float(scale), ptr(out), out.stride(0), stream_ptr()), "ma_attention_tc_f16")
    return out


def sample_tokens(logits: torch.Tensor, do_sample: bool = True, top_k: int = 50, top_p: float = 0.95, seed: int = 0,
                  want_support: bool = False):
    """One pick of the sampling chain (TopK -> TopP -> multinomial) over fp16 logits [B, vocab]."""
    _need_cuda(logits)
    assert logits.dtype == torch.float16 and logits.is_contiguous()
    B, vocab = logits.shape
    tok = torch.empty((B,), dtype=torch.int32, device=logits.device)
    sup = torch.empty((B, 256), dtype=torch.int32, device=logits.device) if want_support else None
    s = Sampling(int(do_sample), int(top_k), float(top_p), int(seed))
    check(lib().ma_sample_tokens(ptr(logits), B, vocab, C.byref(s), ptr(tok), ptr(sup), stream_ptr()),
          "ma_sample_tokens")
    return (tok, sup) if want_support else tok


def layernorm(x: Optional[torch.Tensor], res16: Optional[torch.Tensor], gamma: torch.Tensor, beta: torch.Tensor,
              eps: float = 1e-5, want32: bool = True, want16: bool = True):
    _need_cuda(x, res16, gamma, beta)
    src = x if x is not None else res16
    M, W = src.shape
    o32 = torch.empty((M, W), dtype=torch.float32, device=src.device) if want32 else None
    o16 = torch.empty((M, W), dtype=torch.float16, device=src.device) if want16 else None
    check(lib().ma_layernorm(ptr(x), ptr(res16), ptr(gamma), ptr(beta), eps, M, W, ptr(o32), ptr(o16), stream_ptr()),
          "ma_layernorm")
    return o32, o16


def attention_decode_f16(qkv: torch.Tensor, k: torch.Tensor, v: torch.Tensor, nkeys: torch.Tensor,
                         scale: float = 0.125) -> torch.Tensor:
    """qkv [M,3072] fp16 (q | k | v of the current token); k,v [M,16,T,64] fp16 caches (updated in place at nkeys-1);
    nkeys int32 [M] counts the current token.  Returns the attention output [M,1024] fp16."""
    _need_cuda(qkv, k, v, nkeys)
    M = qkv.shape[0]
    assert qkv.shape[1] == 3072 and qkv.is_contiguous() and k.is_contiguous() and v.is_contiguous()
    assert k.shape[0] == M and k.shape[1] == 16 and k.shape[3] == 64
    T = k.shape[2]
    max_keys = int(nkeys.max().item())
    scratch = torch.zeros(lib().ma_attention_scratch_bytes(M, 16, max_keys), dtype=torch.uint8, device=qkv.device)
    out = torch.empty((M, 1024), dtype=torch.float16, device=qkv.device)
    check(lib().ma_attention_decode_f16(ptr(qkv), 3072, ptr(k), ptr(v), T, ptr(nkeys), max_keys, M, scale, ptr(out),
                                        1024, ptr(scratch), stream_ptr()), "ma_attention_decode_f16")
    return out


def attention_f16(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, nkeys: torch.Tensor,
                  slots: Optional[torch.Tensor] = None, scale: float = 0.125) -> torch.Tensor:
    """q [M,H,64] fp16; k,v [S,H,T,64] fp16 (S cache slots); nkeys int32 [M]; slots int32 [M] or None (slot m)."""
    _need_cuda(q, k, v, nkeys, slots)
    M, H, D = q.shape
    assert D == 64 and k.is_contiguous() and v.is_contiguous() and q.is_contiguous()
    T = k.shape[2]
    max_keys = int(nkeys.max().item())
    scratch = torch.zeros(lib().ma_attention_scratch_bytes(M, H, max_keys), dtype=torch.uint8, device=q.device)
    out = torch.empty((M, H, D), dtype=torch.float16, device=q.device)
    check(lib().ma_attention_f16(ptr(q), H * D, ptr(k), ptr(v), T, H, ptr(slots), ptr(nkeys), max_keys, M, scale,
                                 ptr(out), H * D, ptr(scratch), stream_ptr()), "ma_attention_f16")
    return out
