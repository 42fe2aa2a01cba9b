"""ctypes binding of libmeshanything_b200.so (include/meshanything_b200.h).

The library is built in-tree by `meshanything_b200.build` (nvcc, sm_90a).  There is no CPU or
PyTorch fallback: if the shared object cannot be loaded every call raises.
"""
from __future__ import annotations

import ctypes as C
import math
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
    """Area-weighted surface samples + face normals on the GPU: fp16 [n_samples, 6] (and the face of every sample)."""
    _need_cuda(vertices, faces)
    v = vertices.to(torch.float32).contiguous()
    f = faces.to(torch.int32).contiguous()
    F = f.shape[0]
    ws = torch.empty(lib().ma_sample_surface_workspace_bytes(F), dtype=torch.uint8, device=v.device)
    out = torch.empty((n_samples, 6), dtype=torch.float16, device=v.device)
    idx = torch.empty((n_samples,), dtype=torch.int32, device=v.device) if want_index else None
    check(lib().ma_sample_surface(ptr(v), ptr(f), F, n_samples, int(seed), ptr(out), ptr(idx), ptr(ws), stream_ptr()),
          "ma_sample_surface")
    return (out, idx) if want_index else out


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

    points fp32 [N, 3], finite, already in the output frame; 1 <= k <= 64, k < N <= 2^24.  Returns normals fp32 [N, 3];
    with want_terms (normals, kNN int32 [N, k] in rank order, unoriented normals fp32 [N, 3])."""
    _need_cuda(points)
    p = points.to(torch.float32).contiguous()
    if p.dim() != 2 or p.shape[1] != 3:
        raise ValueError("estimate_normals: points [N, 3]")
    n = p.shape[0]
    if not 1 <= k <= 64:
        raise ValueError(f"estimate_normals: 1 <= k <= 64, got k = {k}")
    if not k < n <= 1 << 24:
        raise ValueError(f"estimate_normals: k < N <= 2^24, got N = {n}, k = {k}")
    if not bool(torch.isfinite(p).all()):
        raise ValueError("estimate_normals: non-finite coordinates")
    ws = torch.empty(lib().ma_estimate_normals_workspace_bytes(n, k), dtype=torch.uint8, device=p.device)
    out = torch.empty((n, 3), dtype=torch.float32, device=p.device)
    knn = torch.empty((n, k), dtype=torch.int32, device=p.device) if want_terms else None
    uno = torch.empty((n, 3), dtype=torch.float32, device=p.device) if want_terms else None
    check(lib().ma_estimate_normals(ptr(p), n, k, ptr(out), ptr(knn), ptr(uno), ptr(ws), stream_ptr()),
          "ma_estimate_normals")
    return (out, knn, uno) if want_terms else out


def remove_outliers(points: torch.Tensor, k: int = 16, std_ratio: float = 2.0, min_component: float = 0.01,
                    want_terms: bool = False):
    """Outlier removal of a cloud (ma_remove_outliers; outliers.remove_outliers adds the frame map).

    points fp32 [N, 3], finite, already in the output frame; 1 <= k <= 64, k < N <= 2^24.  Returns (kept indices int64
    [n_kept] ascending, keep mask bool [N], stats fp64 [8] on the host: mu, sigma, threshold, statistical inliers,
    components, components dropped, kept points, connectivity rounds); with want_terms also (mean neighbour distance
    fp64 [N], kNN int32 [N, k] in rank order).  Reads the stats back (synchronises)."""
    _need_cuda(points)
    p = points.to(torch.float32).contiguous()
    if p.dim() != 2 or p.shape[1] != 3:
        raise ValueError("remove_outliers: points [N, 3]")
    n = p.shape[0]
    if not 1 <= k <= 64:
        raise ValueError(f"remove_outliers: 1 <= k <= 64, got k = {k}")
    if not k < n <= 1 << 24:
        raise ValueError(f"remove_outliers: k < N <= 2^24, got N = {n}, k = {k}")
    if not math.isfinite(std_ratio):
        raise ValueError(f"remove_outliers: std_ratio must be finite, got {std_ratio}")
    if not (math.isfinite(min_component) and min_component >= 0):
        raise ValueError(f"remove_outliers: min_component must be finite and >= 0, got {min_component}")
    if not bool(torch.isfinite(p).all()):
        raise ValueError("remove_outliers: non-finite coordinates")
    dev = p.device
    ws = torch.empty(lib().ma_remove_outliers_workspace_bytes(n, k), dtype=torch.uint8, device=dev)
    keep = torch.empty((n,), dtype=torch.uint8, device=dev)
    idx = torch.empty((n,), dtype=torch.int64, device=dev)
    n_kept = torch.empty((1,), dtype=torch.int64, device=dev)
    stats = torch.empty((8,), dtype=torch.float64, device=dev)
    mean = torch.empty((n,), dtype=torch.float64, device=dev) if want_terms else None
    knn = torch.empty((n, k), dtype=torch.int32, device=dev) if want_terms else None
    check(lib().ma_remove_outliers(ptr(p), n, k, C.c_double(std_ratio), C.c_double(min_component), ptr(keep), ptr(idx),
                                   ptr(n_kept), ptr(mean), ptr(knn), ptr(stats), ptr(ws), stream_ptr()),
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
    if not isinstance(points, torch.Tensor):
        raise ValueError(f"farthest_point_sample: points must be a torch tensor, got {type(points).__name__}")
    if points.dim() != 2 or points.shape[1] != 3:
        raise ValueError(f"farthest_point_sample: points [N, 3], got {tuple(points.shape)}")
    if points.dtype != torch.float32:
        raise ValueError(f"farthest_point_sample: points must be float32, got {points.dtype}")
    if not points.is_contiguous():
        raise ValueError("farthest_point_sample: points must be contiguous")
    if not points.is_cuda:
        raise ValueError("farthest_point_sample: points must live on a CUDA device (no CPU fallback)")
    if isinstance(m, bool) or isinstance(start, bool):
        raise ValueError("farthest_point_sample: m and start must be integers")
    try:
        m, start = operator.index(m), operator.index(start)
    except TypeError:
        raise ValueError(f"farthest_point_sample: m and start must be integers, got {m!r}, {start!r}") from None
    n = points.shape[0]
    if not 1 <= m <= n <= 1 << 24:
        raise ValueError(f"farthest_point_sample: 1 <= m <= N <= 2^24, got N = {n}, m = {m}")
    if not 0 <= start < n:
        raise ValueError(f"farthest_point_sample: 0 <= start < N, got start = {start}, N = {n}")
    if not bool(torch.isfinite(points).all()):
        raise ValueError("farthest_point_sample: non-finite coordinates")
    dev = points.device
    ws = torch.empty(lib().ma_farthest_point_sample_workspace_bytes(n, m), dtype=torch.uint8, device=dev)
    idx = torch.empty((m,), dtype=torch.int64, device=dev)
    r2 = torch.empty((m,), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        check(lib().ma_farthest_point_sample(ptr(points), n, m, start, ptr(idx), ptr(r2), ptr(ws), stream_ptr()),
              "ma_farthest_point_sample")
    return idx, r2


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
