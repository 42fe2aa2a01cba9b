"""numpy restatement of csrc/subsample.cu (test infrastructure only): farthest-point subsampling as DESIGN.md section 1.4
defines it.

fp32 arrays and separate numpy operations (numpy never fuses a multiply-add), the d^2 formula of the kNN of section 1.2
(tests/normals_oracle._d2); the next pick is np.argmax over D with the picked points set to -1, which gives the lowest
index on ties.  idx and r2 agree with the GPU bit for bit.
"""
import numpy as np

from tests import outliers_oracle as OO

F32 = np.float32

frame_map = OO.frame_map     # float64 input: shifted by its float64 bounding-box centre, then metrics.to_output_frame


def farthest_point_sample(points_frame, m, start=0):
    """Points already in the frame (fp32 [N, 3]) -> (idx int64 [m] in pick order, r2 fp32 [m])."""
    p = np.ascontiguousarray(points_frame, F32)
    n = len(p)
    assert 1 <= m <= n and 0 <= start < n
    x, y, z = p[:, 0].copy(), p[:, 1].copy(), p[:, 2].copy()
    d = np.full(n, np.inf, F32)
    key = np.empty(n, F32)
    picked = np.zeros(n, bool)
    idx = np.empty(m, np.int64)
    r2 = np.empty(m, F32)
    w = start
    for t in range(m):
        idx[t] = w
        picked[w] = True
        dx, dy, dz = x - x[w], y - y[w], z - z[w]
        np.minimum(d, (dx * dx + dy * dy) + dz * dz, out=d)
        r2[t] = d.max()                       # picked points hold d = 0 (their own d^2)
        np.copyto(key, d)
        key[picked] = F32(-1)
        w = int(np.argmax(key))
    return idx, r2


def torch_bruteforce(p, m, start=0):
    """The same definition as a loop of torch operations on p's device (fp32 [N, 3] in the frame): the same fp32 formula
    in separate kernels (no fused multiply-add), the next pick from torch.max over the packed int64 keys
    D_bits << 32 | ~i (0 for picked points), so ties resolve exactly.  -> (idx int64 [m], r2 fp32 [m]) on the device."""
    import torch
    n = p.shape[0]
    x, y, z = (p[:, a].contiguous() for a in range(3))
    d = torch.full((n,), float("inf"), dtype=torch.float32, device=p.device)
    picked = torch.zeros(n, dtype=torch.bool, device=p.device)
    low = (~torch.arange(n, dtype=torch.int64, device=p.device)) & 0xFFFFFFFF
    zero = torch.zeros((), dtype=torch.int64, device=p.device)
    w = torch.tensor(start, dtype=torch.int64, device=p.device)
    idx = torch.empty(m, dtype=torch.int64, device=p.device)
    r2 = torch.empty(m, dtype=torch.float32, device=p.device)
    for t in range(m):
        idx[t] = w
        picked[w] = True
        dx, dy, dz = x - x[w], y - y[w], z - z[w]
        d = torch.minimum(d, (dx * dx + dy * dy) + dz * dz)
        r2[t] = d.max()
        key = torch.where(picked, zero, (d.view(torch.int32).to(torch.int64) << 32) | low)
        w = (~torch.max(key)) & 0xFFFFFFFF
    return idx, r2
