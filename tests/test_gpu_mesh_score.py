"""-m gpu: the best-of-N mesh score (csrc/mesh_score.cu) against its numpy restatement (tests/mesh_score_oracle.py) --
per-point and per-quadrature-point distances and argmins bit for bit, fp64 terms to 1e-12 -- plus
MeshAnything.forward_candidates and `main.py --num_samples`.  The two argument checks of the command line need no
device and run everywhere."""
import argparse
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from meshanything_b200 import capi, metrics
from meshanything_b200.inputs import synthetic_pc_normal
from tests import mesh_score_oracle as M

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32


def _dev():
    return torch.device("cuda", 0)


def _meshes(S, N, F, seed):
    """Random soups in the detokenizer frame with absent rows at random positions, a duplicated face, a segment, a
    point and a zero-area sliver."""
    rng = np.random.RandomState(seed)
    m = rng.uniform(-0.5, 0.5, (S, N, F, 3, 3)).astype(F32)
    if F >= 5:
        m[:, :, 1] = m[:, :, 0]                                      # duplicated face
        m[:, :, 2, 1] = m[:, :, 2, 0]                                # segment
        m[:, :, 3] = m[:, :, 3, :1]                                  # point
        m[:, :, 4, 2] = 0.5 * (m[:, :, 4, 0] + m[:, :, 4, 1])        # collinear: (near) zero area
    absent = rng.rand(S, N, F) < 0.15
    m[absent] = np.nan
    return m


def _close(a, b, rtol=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    same_inf = np.isinf(a) == np.isinf(b)
    fin = np.isfinite(b)
    return bool(same_inf.all() and (np.abs(a[fin] - b[fin]) <= rtol * np.abs(b[fin])).all())


def _bits(x):
    return np.asarray(x).view(np.uint32)


@gpu
@pytest.mark.parametrize("S,N,F,P", [(3, 5, 1, 4096), (3, 5, 37, 1000), (2, 2, 800, 4096), (2, 2, 1600, 1000),
                                     (1, 3, 2000, 1000)])
def test_kernel_matches_the_oracle_bit_for_bit(S, N, F, P):
    meshes = _meshes(S, N, F, seed=F + P)
    pc = synthetic_pc_normal(S, first=F, n_points=P)
    cloud = metrics.to_output_frame(pc.to(_dev()))
    assert np.array_equal(_bits(cloud.cpu().numpy()), _bits(M.frame_map(pc.numpy())))
    mg = torch.from_numpy(meshes).to(_dev())
    out = capi.mesh_score(mg, cloud, want_terms=True)
    terms, faces, pdist, pface, qdist, qpoint = [t.cpu().numpy() for t in out]
    again = [t.cpu().numpy() for t in capi.mesh_score(mg, cloud, want_terms=True)]
    for x, y in zip((terms, faces, pdist, pface, qdist, qpoint), again):   # two calls: identical bits
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))
    _, _, res = M.score(meshes, pc.numpy())
    for s in range(S):
        for n in range(N):
            r = res[s][n]
            assert faces[s, n] == r["faces"]
            assert np.array_equal(_bits(pdist[s, n]), _bits(r["point_dist"])), (s, n, "point distance")
            assert np.array_equal(pface[s, n], r["point_face"]), (s, n, "point face")
            assert np.array_equal(_bits(qdist[s, n]), _bits(r["quad_dist"])), (s, n, "quadrature distance")
            assert np.array_equal(qpoint[s, n], r["quad_point"]), (s, n, "quadrature point")
            assert _close(terms[s, n], [r["p2m"], r["m2p"], r["nc_p"], r["nc_m"]]), (s, n, terms[s, n])
    # the public score: the frame map, chamfer = p2m + m2p, the selection
    sc = metrics.score(mg, pc)
    chamfer, nc, _ = M.score(meshes, pc.numpy())
    assert _close(sc["chamfer"].cpu().numpy(), chamfer) and _close(sc["normal_consistency"].cpu().numpy(), nc)
    assert np.array_equal(metrics.select(sc["chamfer"]).cpu().numpy(), M.select(sc["chamfer"].cpu().numpy()))
    one = metrics.score(mg[:, 0], pc)                              # [S, F, 3, 3]: one candidate per shape
    assert one["chamfer"].shape == (S,) and torch.equal(one["chamfer"], sc["chamfer"][:, 0])


@gpu
def test_empty_and_degenerate_candidates_score_inf():
    good = _meshes(1, 1, 20, seed=1)[0, 0]
    empty = np.full_like(good, np.nan)
    flat = good.copy()
    flat[:, 1] = flat[:, 0]                                          # every face a segment: zero area
    meshes = torch.from_numpy(np.stack([empty, flat, good])[None]).to(_dev())
    pc = synthetic_pc_normal(1, first=2, n_points=500)
    sc = metrics.score(meshes, pc)
    ch = sc["chamfer"].cpu().numpy()[0]
    assert np.isinf(ch[0]) and np.isinf(ch[1]) and np.isfinite(ch[2])
    assert sc["normal_consistency"][0, :2].tolist() == [0.0, 0.0]
    present = int((~np.isnan(good[:, 0, 0])).sum())
    assert sc["faces"][0].tolist() == [0, present, present]
    assert int(metrics.select(sc["chamfer"])[0]) == 2
    assert int(metrics.select(sc["chamfer"][:, :2])[0]) == 0          # every candidate +inf: candidate 0
    with pytest.raises(ValueError, match="non-finite"):
        bad = meshes.clone()
        bad[0, 2, 0, 1, 1] = float("nan")                            # NaN inside a valid face
        metrics.score(bad, pc)


def _model(F):
    from MeshAnything.models.meshanything import MeshAnything
    from meshanything_b200 import checkpoint as ck
    args = argparse.Namespace(llm="facebook/opt-350m", codebook_size=8192, codebook_dim=1024, n_max_triangles=F, seed=0)
    model = MeshAnything(args)
    model.load_state_dict(ck.synthetic_state_dict(0), strict=True, device=_dev())
    return model


@gpu
def test_forward_candidates_is_one_sampled_forward_plus_the_score():
    F, N = 16, 3
    pc = synthetic_pc_normal(2, first=30)
    model = _model(F)
    with pytest.raises(ValueError):
        model.forward_candidates(pc, 0)
    res = model.forward_candidates(pc, N)
    assert model._calls == 1
    assert res.meshes.shape == (2, N, F, 3, 3) and res.best.shape == (2, F, 3, 3)
    assert res.chamfer.shape == (2, N) and res.normal_consistency.shape == (2, N) and res.index.shape == (2,)
    ref = _model(F)(pc.to(_dev()).repeat_interleave(N, 0), sampling=True)   # a fresh model: the same _calls
    got = res.meshes.reshape(2 * N, F, 3, 3)
    assert torch.equal(torch.isnan(got), torch.isnan(ref))
    assert torch.equal(torch.nan_to_num(got), torch.nan_to_num(ref))
    for b in range(2):
        assert torch.equal(torch.nan_to_num(res.best[b]), torch.nan_to_num(res.meshes[b, res.index[b]]))
    chamfer, nc, _ = M.score(res.meshes.cpu().numpy(), pc.numpy())
    assert _close(res.chamfer.cpu().numpy(), chamfer) and _close(res.normal_consistency.cpu().numpy(), nc)
    assert np.array_equal(res.index.cpu().numpy(), M.select(chamfer))
    print("forward_candidates: chamfer", np.round(chamfer, 4).tolist(), "kept", res.index.tolist())


def _main(args, tmp_path, timeout=900):
    return subprocess.run([sys.executable, os.path.join(ROOT, "main.py"), "--out_dir", str(tmp_path / "out"),
                           "--pretrained_weights", "synthetic"] + args, cwd=ROOT, capture_output=True, text=True,
                          timeout=timeout)


@gpu
def test_main_cli_num_samples_keeps_the_best(tmp_path):
    in_dir = tmp_path / "in"
    in_dir.mkdir()
    for i in range(2):
        np.save(in_dir / f"s{i}.npy", synthetic_pc_normal(1, first=40 + i)[0].numpy().astype(np.float16))
    r = _main(["--input_type", "pc_normal", "--input_dir", str(in_dir), "--n_max_triangles", "6", "--sampling",
               "--num_samples", "3", "--batchsize_per_gpu", "2"], tmp_path)
    assert r.returncode == 0, r.stderr[-2000:]
    objs = sorted(f for _, _, fs in os.walk(tmp_path / "out") for f in fs if f.endswith(".obj"))
    assert objs == ["s0_gen.obj", "s1_gen.obj"]
    for uid in ("s0", "s1"):
        lines = [ln for ln in r.stdout.splitlines() if ln.startswith(f"{uid} sample ")]
        assert len(lines) == 3 and all("chamfer" in ln and "normal consistency" in ln for ln in lines), r.stdout
        assert sum("kept" in ln for ln in lines) == 1


def test_main_cli_num_samples_needs_sampling(tmp_path):
    r = _main(["--input_type", "pc_normal", "--input_path", "x.npy", "--num_samples", "3"], tmp_path, timeout=300)
    assert r.returncode != 0 and "ValueError" in r.stderr and "needs --sampling" in r.stderr


def test_main_cli_num_samples_rejects_continuous_batching(tmp_path):
    r = _main(["--input_type", "pc_normal", "--input_path", "x.npy", "--num_samples", "3", "--sampling",
               "--continuous_batching"], tmp_path, timeout=300)
    assert r.returncode != 0 and "ValueError" in r.stderr and "--continuous_batching" in r.stderr
