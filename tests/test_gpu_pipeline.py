"""-m gpu: encoder (a1-a8), detokenizer (a17-a18) and the MeshAnything.forward drop-in on the GPU.

Floating-point stages are compared with the fp32 torch restatement (oracle/torch_ref.py, itself pinned to the
reference's own modules) under a stated tolerance: the GPU path rounds every Linear input/output to fp16 as CUDA
autocast does in the reference, the restatement does not round.  Integer results (token ids) are bit-exact
against the CPU oracle given the same prefix.
"""
import argparse

import pytest
import torch

from meshanything_b200 import checkpoint as ck
from meshanything_b200.inputs import synthetic_pc_normal

gpu = pytest.mark.gpu

# stated tolerances (DESIGN.md section 6)
TOL_PF_MAX, TOL_PF_MEAN = 1.5e-2, 2.5e-3      # measured 3.5e-3 / 5.9e-4 (unit-variance LayerNorm output after 9 blocks)
TOL_PREFIX_MAX, TOL_PREFIX_MEAN = 4e-2, 6e-3  # measured 1.0e-2 / 1.6e-3 (std 1.4, 16 more fp16-stream blocks + cond_proj)
F_SMALL = 8


def _dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def full():
    sd = ck.make_state_dict(ck.all_specs(24), 0)
    return sd


@gpu
def test_encoder_vs_fp32_reference(full):
    from meshanything_b200.encoder import EncoderArena
    from oracle import torch_ref
    pc = synthetic_pc_normal(3, first=0)
    enc = EncoderArena(full, _dev())
    pf, prefix = enc.forward(pc.to(_dev()))
    with torch.no_grad():
        rpf, rprefix = torch_ref.encoder_forward(full, pc)
    d1, d2 = (pf.cpu() - rpf).abs(), (prefix.cpu() - rprefix).abs()
    print("point_feature err max %.4g mean %.4g ; prefix err max %.4g mean %.4g" % (d1.max(), d1.mean(), d2.max(), d2.mean()))
    assert d1.max() < TOL_PF_MAX and d1.mean() < TOL_PF_MEAN
    assert d2.max() < TOL_PREFIX_MAX and d2.mean() < TOL_PREFIX_MEAN
    # batch invariance of the canonical kernels: shape 1 alone gives the same bits
    pf1, prefix1 = enc.forward(pc[1:2].to(_dev()))
    assert torch.equal(pf1[0], pf[1]) and torch.equal(prefix1[0], prefix[1])


@gpu
def test_encoder_and_detokenizer_with_tensor_core_attention(full):
    """ma_set_tensor_cores(2): attention of the encoder / detokenizer on the tensor cores too -- same stated tolerances against
    the fp32 restatement, and close to the default (canonical attention) path."""
    from meshanything_b200 import capi
    from meshanything_b200.encoder import EncoderArena, TokenizerArena
    from oracle import torch_ref
    pc = synthetic_pc_normal(2, first=0)
    enc = EncoderArena(full, _dev())
    pf1, prefix1 = enc.forward(pc.to(_dev()))
    old = capi.lib().ma_set_tensor_cores(2)
    try:
        pf, prefix = enc.forward(pc.to(_dev()))
        with torch.no_grad():
            rpf, rprefix = torch_ref.encoder_forward(full, pc)
        d1, d2 = (pf.cpu() - rpf).abs(), (prefix.cpu() - rprefix).abs()
        print("tc-attention: point_feature err max %.4g mean %.4g ; prefix err max %.4g mean %.4g ; vs default path %.4g"
              % (d1.max(), d1.mean(), d2.max(), d2.mean(), (pf - pf1).abs().max()))
        assert d1.max() < TOL_PF_MAX and d1.mean() < TOL_PF_MEAN
        assert d2.max() < TOL_PREFIX_MAX and d2.mean() < TOL_PREFIX_MEAN
        F = 12
        g = torch.Generator().manual_seed(5)
        gen_ids = torch.randint(3, 8195, (2, 9 * F + 2), generator=g, dtype=torch.int64)
        gen_ids[0, 1 + 9 * 10:] = 2
        tok = TokenizerArena(full, _dev())
        coords = tok.detokenize(gen_ids.to(torch.int32).to(_dev()), pf1, F).cpu()
        with torch.no_grad():
            rcoords = torch_ref.detokenize(full, torch_ref.postprocess_ids(gen_ids, F), pf1.cpu())
        assert torch.equal(torch.isnan(coords), torch.isnan(rcoords))
        valid = ~torch.isnan(rcoords)
        assert (coords[valid] == rcoords[valid]).float().mean() > 0.97
    finally:
        capi.lib().ma_set_tensor_cores(old)


@gpu
def test_detokenizer_vs_fp32_reference(full):
    from meshanything_b200.encoder import EncoderArena, TokenizerArena
    from oracle import torch_ref
    F = 12
    g = torch.Generator().manual_seed(5)
    gen_ids = torch.randint(3, 8195, (2, 9 * F + 2), generator=g, dtype=torch.int64)
    gen_ids[0, 1 + 9 * 7 + 4] = 1          # eos inside face 7 -> face 7 absent
    gen_ids[0, 1 + 9 * 10:] = 2            # padding after face 9
    gen_ids[1, 1 + 9 * 11 + 8] = 0
    pc = synthetic_pc_normal(2, first=0)
    pf, _ = EncoderArena(full, _dev()).forward(pc.to(_dev()))
    tok = TokenizerArena(full, _dev())
    coords, ids = tok.detokenize(gen_ids.to(torch.int32).to(_dev()), pf, F, want_ids=True)
    ref_ids = torch_ref.postprocess_ids(gen_ids, F)
    assert torch.equal(ids.cpu().long(), ref_ids)
    with torch.no_grad():
        rcoords, rlogits = torch_ref.detokenize(full, ref_ids, pf.cpu(), return_logits=True)
    c = coords.cpu()
    assert torch.equal(torch.isnan(c), torch.isnan(rcoords))
    valid = ~torch.isnan(rcoords)
    same = (c[valid] == rcoords[valid])
    # a bin may differ only where the reference's top-2 logit margin is within the fp16 noise of the logits
    top2 = torch.topk(rlogits, 2, dim=-1).values
    margin = (top2[..., 0] - top2[..., 1]).view(2, F, 3, 3)[valid]
    print("detok bins equal: %d / %d ; max margin at a mismatch %.4g" % (same.sum(), same.numel(),
                                                                         margin[~same].max() if (~same).any() else 0.0))
    assert same.float().mean() > 0.97
    assert (margin[~same] < 0.08).all()
    # (no adjacency requirement on a flipped bin: with a random-weight tokenizer the two leading logits of a
    # near-tie belong to unrelated bins; the margin criterion above is the meaningful one)


@gpu
def test_forward_drop_in(full):
    """MeshAnything(args).load_state_dict(strict=True); model(pc_normal) -> [B,F,3,3]; ids bit-exact vs the oracle."""
    from MeshAnything.models.meshanything import MeshAnything
    from oracle.decoder import OracleDecoder
    from oracle import torch_ref
    args = argparse.Namespace(llm="facebook/opt-350m", codebook_size=8192, codebook_dim=1024, n_max_triangles=F_SMALL,
                              seed=0)
    model = MeshAnything(args)
    with pytest.raises(RuntimeError):
        model.load_state_dict({k: v for k, v in full.items() if k != "cond_proj.bias"}, strict=True, device=_dev())
    # weights arrive as views into ONE packed fp32 device buffer (what the NCCL broadcast at init produces):
    # arbitrary 4-byte offsets must not break the 16-byte loads of the kernels
    from meshanything_b200 import parallel
    packed = parallel.broadcast_state_dict(full, ck.all_specs(24), _dev())
    model.load_state_dict(packed, strict=True, device=_dev())
    del packed
    pc = synthetic_pc_normal(2, first=3)                       # host tensor: forward copies it
    out = model(pc)
    assert out.shape == (2, F_SMALL, 3, 3) and out.dtype == torch.float32 and out.is_cuda
    v = out[~torch.isnan(out)]
    assert (v >= -0.5).all() and (v < 0.5).all()
    ids = model.last_ids.cpu()
    # decoder leg: same prefix -> the oracle's ids
    pf, prefix = model.point_encoder._last
    oracle = OracleDecoder(full, 24, 257 + 9 * F_SMALL + 2)
    for b in range(2):
        ref, _ = oracle.generate(prefix[b].cpu(), 9 * F_SMALL + 2)
        assert ids[b].tolist()[:len(ref)] == ref
    # detokenizer leg on the same ids
    with torch.no_grad():
        rc, rlog = torch_ref.detokenize(full, torch_ref.postprocess_ids(ids.long(), F_SMALL), pf.cpu(), return_logits=True)
    assert torch.equal(torch.isnan(out.cpu()), torch.isnan(rc))
    valid = ~torch.isnan(rc)
    same = out.cpu()[valid] == rc[valid]
    top2 = torch.topk(rlog, 2, dim=-1).values
    margin = (top2[..., 0] - top2[..., 1]).view(2, F_SMALL, 3, 3)[valid]
    assert same.float().mean() > 0.97 and (margin[~same] < 0.08).all()      # the rule of the dedicated detokenizer test
    # END TO END with the encoder in the loop: greedy ids from the GPU encoder's prefix (within 1e-2 of the fp32
    # reference, test_encoder_vs_fp32_reference) against the oracle's ids from the fp32 REFERENCE prefix.  A free-running
    # greedy decode amplifies any logit difference at a near-tie, so what is asserted is the teacher-forced view: along
    # the reference path the GPU logits stay close and the argmax agrees wherever the margin is clear.  The first
    # divergence step and the agreement rate of the free-running ids are reported.
    from meshanything_b200.decoder import Generator
    n64 = 9 * 64 + 2
    with torch.no_grad():
        _, ref_prefix = torch_ref.encoder_forward(full, pc[:1])
    oracle64 = OracleDecoder(full, 24, 257 + n64)
    ref_ids, ref_logits = oracle64.generate(ref_prefix[0], n64, keep_logits=True)
    g64 = Generator(model._dec, 1, 257 + n64)
    got_ids, _ = g64.generate(prefix[:1], n64)
    got_ids = got_ids[0].cpu().tolist()
    first_div = next((i for i, (a, b) in enumerate(zip(got_ids, ref_ids)) if a != b), len(ref_ids))
    agree = sum(a == b for a, b in zip(got_ids, ref_ids)) / len(ref_ids)
    forced = torch.tensor([ref_ids + [2] * (n64 - len(ref_ids))], dtype=torch.int32)
    _, _, tf = g64.generate(prefix[:1], n64, forced_ids=forced, want_logits=True, eos_id=-1)
    rl = torch.stack(ref_logits).float()
    gl = tf[:len(ref_logits), 0].cpu().float()
    d = (gl - rl).abs()
    t2 = torch.topk(rl, 2, dim=1).values
    clear = (t2[:, 0] - t2[:, 1]) > 0.25
    print("end to end (GPU encoder prefix vs fp32 reference prefix, F=64): first divergence at step %d of %d, free-running "
          "agreement %.3f; teacher-forced logits max |diff| %.4f mean %.5f, argmax agreement %.4f (%d positions with margin > 0.25)"
          % (first_div, len(ref_ids), agree, float(d.max()), float(d.mean()),
             float((gl.argmax(1) == rl.argmax(1)).float().mean()), int(clear.sum())))
    assert first_div >= 1
    assert d.max() < 5e-2 and d.mean() < 5e-3
    assert torch.equal(gl.argmax(1)[clear], rl.argmax(1)[clear])
    # one shape alone, and sampling mode
    out1 = model(pc[:1].to(_dev()))
    assert torch.equal(torch.nan_to_num(out1[0]), torch.nan_to_num(out[0]))
    outs = model(pc, sampling=True)
    assert outs.shape == out.shape
    # continuous batching over 2 cache slots: every shape equals its padded-batch result
    q = model.forward_queue([pc[0], pc[1], pc[0]], slots=2, poll_every=16)
    assert len(q) == 3
    for got, want in zip(q, (out[0], out[1], out[0])):
        assert torch.equal(torch.nan_to_num(got), torch.nan_to_num(want))
    assert model.last_queue_stats.prefills == 3


@gpu
def test_main_cli_writes_obj(tmp_path):
    """`python main.py --input_type pc_normal --input_path x.npy ...` (reference flags, main.py:60-89) writes <uid>_gen.obj."""
    import os
    import subprocess
    import sys
    import numpy as np
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pc = synthetic_pc_normal(1, first=7)[0].numpy().astype(np.float16)
    extra = np.concatenate([pc, pc[:100]], axis=0)            # > 4096 points: exercises the np.random.choice subsample
    npy = tmp_path / "shape7.npy"
    np.save(npy, extra)
    out_dir = tmp_path / "out"
    r = subprocess.run([sys.executable, os.path.join(root, "main.py"), "--input_type", "pc_normal", "--input_path", str(npy),
                        "--out_dir", str(out_dir), "--pretrained_weights", "synthetic", "--n_max_triangles", "6",
                        "--seed", "0"], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    objs = [os.path.join(dp, f) for dp, _, fs in os.walk(out_dir) for f in fs if f.endswith("_gen.obj")]
    assert len(objs) == 1 and os.path.basename(objs[0]) == "shape7_gen.obj"
    txt = open(objs[0]).read()
    assert txt.count("\nf ") + txt.startswith("f ") >= 1 and "v " in txt
    # the reference's input assertions (main.py:24,54)
    bad = tmp_path / "bad.npy"
    np.save(bad, pc[:1000])
    r2 = subprocess.run([sys.executable, os.path.join(root, "main.py"), "--input_type", "pc_normal", "--input_path", str(bad),
                         "--out_dir", str(out_dir), "--pretrained_weights", "synthetic", "--n_max_triangles", "6"],
                        cwd=root, capture_output=True, text=True, timeout=600)
    assert r2.returncode != 0 and "at least 4096 points" in r2.stderr


@gpu
def test_main_cli_continuous_batching(tmp_path):
    """`--input_dir` with three shapes through two cache slots (`--continuous_batching --batchsize_per_gpu 2`) writes the
    same OBJ files as the padded-batch loop."""
    import os
    import subprocess
    import sys
    import numpy as np
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    in_dir = tmp_path / "in"
    in_dir.mkdir()
    for i in range(3):
        np.save(in_dir / f"s{i}.npy", synthetic_pc_normal(1, first=20 + i)[0].numpy().astype(np.float16))
    texts = []
    for extra in ([], ["--continuous_batching"]):
        out_dir = tmp_path / ("out" + str(len(extra)))
        r = subprocess.run([sys.executable, os.path.join(root, "main.py"), "--input_type", "pc_normal", "--input_dir",
                            str(in_dir), "--out_dir", str(out_dir), "--pretrained_weights", "synthetic",
                            "--n_max_triangles", "6", "--batchsize_per_gpu", "2", "--seed", "0"] + extra,
                           cwd=root, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        objs = sorted(os.path.join(dp, f) for dp, _, fs in os.walk(out_dir) for f in fs if f.endswith("_gen.obj"))
        assert [os.path.basename(o) for o in objs] == ["s0_gen.obj", "s1_gen.obj", "s2_gen.obj"]
        texts.append([open(o).read() for o in objs])
    assert texts[0] == texts[1]


@gpu
def test_kernel_selections_all_meet_the_tolerance(full):
    """ma_set_tensor_cores 0 (canonical CUDA-core kernels), 1 (wgmma GEMMs, canonical attention) and 2 (default):
    every selection stays inside the stated encoder tolerance, and they agree with each other to fp16 noise."""
    from meshanything_b200 import capi
    from meshanything_b200.encoder import EncoderArena
    from oracle import torch_ref
    pc = synthetic_pc_normal(1, first=4)
    enc = EncoderArena(full, _dev())
    with torch.no_grad():
        rpf, rprefix = torch_ref.encoder_forward(full, pc)
    outs = {}
    old = capi.lib().ma_set_tensor_cores(2)
    try:
        for mode in (0, 1, 2):
            capi.lib().ma_set_tensor_cores(mode)
            pf, prefix = enc.forward(pc.to(_dev()))
            outs[mode] = pf.cpu()
            d1, d2 = (pf.cpu() - rpf).abs(), (prefix.cpu() - rprefix).abs()
            print("mode %d: point_feature err max %.4g ; prefix err max %.4g" % (mode, d1.max(), d2.max()))
            assert d1.max() < TOL_PF_MAX and d1.mean() < TOL_PF_MEAN, mode
            assert d2.max() < TOL_PREFIX_MAX and d2.mean() < TOL_PREFIX_MEAN, mode
    finally:
        capi.lib().ma_set_tensor_cores(old)
    assert (outs[0] - outs[2]).abs().max() < 2 * TOL_PF_MAX and (outs[1] - outs[2]).abs().max() < 2 * TOL_PF_MAX


@gpu
def test_gpu_surface_sampler_matches_the_numpy_sampler_distribution():
    """SURVEY 8(f)3: ma_sample_surface (area-weighted face pick by inverse CDF, uniform barycentric point, face normal)
    against the numpy restatement of trimesh's sampler in mesh_to_pc.SimpleMesh: the per-face hit counts of 200 000
    samples follow the face areas (the numpy sampler's own counts are checked with the same bound), every point lies in
    its face's plane inside the triangle, the normal is the face normal, and process_mesh_to_pc uses it on a GPU box."""
    import numpy as np
    import mesh_to_pc
    from meshanything_b200 import capi
    rng = np.random.RandomState(3)
    V, F, n = 300, 500, 200_000
    verts = rng.randn(V, 3).astype(np.float32)
    faces = np.stack([rng.choice(V, 3, replace=False) for _ in range(F)]).astype(np.int32)
    # a few degenerate and tiny faces: they must (almost) never be hit
    faces[7] = [5, 5, 9]
    verts[faces[11, 1]] = verts[faces[11, 0]] + 1e-4
    mesh = mesh_to_pc.SimpleMesh(verts, faces)
    tri = verts[faces].astype(np.float64)
    area = 0.5 * np.linalg.norm(np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]), axis=1)
    p = area / area.sum()
    out, idx = capi.sample_surface(torch.from_numpy(verts).to(_dev()), torch.from_numpy(faces).to(_dev()), n, seed=5,
                                   want_index=True)
    out, idx = out.cpu().float().numpy(), idx.cpu().numpy()
    counts = np.bincount(idx, minlength=F)
    sigma = np.sqrt(n * p * (1 - p)) + 1.0
    assert (np.abs(counts - n * p) < 5 * sigma).all()
    assert counts[7] == 0
    np.random.seed(0)
    _, idx_np = mesh.sample(n, return_index=True)
    assert (np.abs(np.bincount(idx_np, minlength=F) - n * p) < 5 * sigma).all()      # same law for the host sampler
    # geometry: barycentric coordinates of every point w.r.t. its face are in [0, 1] (fp16 rounding of the output)
    a, b, c = tri[idx, 0], tri[idx, 1], tri[idx, 2]
    nrm = np.cross(b - a, c - a)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    pts = out[:, :3].astype(np.float64)
    scale = np.abs(tri).max()
    assert np.abs(((pts - a) * nrm).sum(1)).max() < 4e-3 * scale                     # in the plane
    m = np.stack([b - a, c - a], axis=2)                                             # [n, 3, 2]
    sol = np.einsum("nij,nj->ni", np.linalg.pinv(m), pts - a)
    assert sol.min() > -2e-2 and (sol.sum(1)).max() < 1 + 2e-2
    assert np.abs(out[:, 3:] - nrm).max() < 2e-3
    # uniform inside a triangle: the mean barycentric coordinates of the samples of the largest face are 1/3
    big = int(np.argmax(area))
    sb = sol[idx == big]
    assert len(sb) > 1000 and np.abs(sb.mean(0) - 1.0 / 3.0).max() < 0.03
    # the drop-in entry point uses the GPU sampler here and returns what the reference returns
    np.random.seed(1)
    clouds, used = mesh_to_pc.process_mesh_to_pc([mesh])
    assert clouds[0].shape == (4096, 6) and clouds[0].dtype == np.float16 and used[0] is mesh
    assert np.abs(np.linalg.norm(clouds[0][:, 3:].astype(np.float32), axis=1) - 1).max() < 2e-3


@gpu
def test_safetensors_checkpoint_round_trip(tmp_path):
    """SURVEY 8(f)4 / main.py:95-104: a safetensors file with the published key list (fp32 tensors, BERT layers in the
    optimum-BetterTransformer spelling) goes through `main.load_model` into the fp16 / fp32 arenas and gives exactly the
    mesh of a model loaded from the in-memory tensors; the same checkpoint re-saved with plain HF BertLayer names
    (what `BetterTransformer.reverse` or a non-optimum save would produce) loads to the same result; a missing or an
    unexpected key is an error under strict=True, as in the reference."""
    import main as cli
    from safetensors.torch import save_file
    from MeshAnything.models.meshanything import MeshAnything
    NL = 2                                                    # decoder layers (keeps the file at ~1.3 GB)
    specs = ck.all_specs(NL)
    sd = ck.make_state_dict(specs, 0)
    args = argparse.Namespace(llm="facebook/opt-350m", codebook_size=8192, codebook_dim=1024, n_max_triangles=6, seed=0,
                              pretrained_weights=str(tmp_path / "MeshAnything_350m.pth"))
    save_file({k: v.contiguous() for k, v in sd.items()}, args.pretrained_weights)
    orig_expected = MeshAnything.expected_keys
    MeshAnything.expected_keys = lambda self: list(specs.keys())
    try:
        model = cli.load_model(args, device=_dev())
        ref = MeshAnything(args)
        ref.load_state_dict(sd, strict=True, device=_dev())
        pc = synthetic_pc_normal(1, first=3).to(_dev())
        a, b = model(pc), ref(pc)
        assert torch.equal(torch.nan_to_num(a, nan=7.0), torch.nan_to_num(b, nan=7.0))
        assert torch.equal(model.last_ids, ref.last_ids)
        # plain HF spelling of the BERT layers
        hf = {k: v for k, v in sd.items() if not k.startswith("tokenizer.decoder.layer.")}
        w = 768
        for i in range(6):
            q, o = f"tokenizer.decoder.layer.{i}", f"tokenizer.decoder.layer.{i}"
            iw, ib = sd[f"{q}.in_proj_weight"], sd[f"{q}.in_proj_bias"]
            for j, nm in enumerate(("query", "key", "value")):
                hf[f"{o}.attention.self.{nm}.weight"] = iw[j * w:(j + 1) * w].clone()
                hf[f"{o}.attention.self.{nm}.bias"] = ib[j * w:(j + 1) * w].clone()
            for src, dst in (("out_proj", "attention.output.dense"), ("linear1", "intermediate.dense"),
                             ("linear2", "output.dense")):
                hf[f"{o}.{dst}.weight"], hf[f"{o}.{dst}.bias"] = sd[f"{q}.{src}_weight"], sd[f"{q}.{src}_bias"]
            for src, dst in (("norm1", "attention.output.LayerNorm"), ("norm2", "output.LayerNorm")):
                hf[f"{o}.{dst}.weight"], hf[f"{o}.{dst}.bias"] = sd[f"{q}.{src}_weight"], sd[f"{q}.{src}_bias"]
        args2 = argparse.Namespace(**{**vars(args), "pretrained_weights": str(tmp_path / "hf_names.safetensors")})
        save_file({k: v.contiguous() for k, v in hf.items()}, args2.pretrained_weights)
        model2 = cli.load_model(args2, device=_dev())
        assert torch.equal(torch.nan_to_num(model2(pc), nan=7.0), torch.nan_to_num(b, nan=7.0))
        # strictness
        broken = dict(sd)
        broken.pop("cond_proj.weight")
        with pytest.raises(RuntimeError, match="cond_proj.weight"):
            MeshAnything(args).load_state_dict(broken, strict=True, device=_dev())
        extra = dict(sd)
        extra["not.a.key"] = torch.zeros(1)
        with pytest.raises(RuntimeError, match="not.a.key"):
            MeshAnything(args).load_state_dict(extra, strict=True, device=_dev())
    finally:
        MeshAnything.expected_keys = orig_expected


@gpu
def test_config1_mouse_example():
    """BASELINE configs[0] plumbing on the GPU: the pc_normal the reference's own Dataset makes of pc_examples/mouse.npy
    (committed fixture tests/golden/config1_mouse.npz; tests/test_host_io.py checks that our Dataset reproduces it bit for
    bit) through MeshAnything.forward at a 64-face cap; the token ids behind the mesh must be the CPU oracle's for the
    encoder prefix this GPU produced."""
    import os
    import numpy as np
    from MeshAnything.models.meshanything import MeshAnything
    from oracle.decoder import OracleDecoder
    fx = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "config1_mouse.npz"))
    pc = torch.from_numpy(fx["pc_normal"][None])
    args = argparse.Namespace(llm="facebook/opt-350m", codebook_size=8192, codebook_dim=1024, n_max_triangles=64, seed=0)
    sd = ck.synthetic_state_dict(0)
    model = MeshAnything(args)
    model.load_state_dict(sd, strict=True, device=_dev())
    out = model(pc.to(_dev()))
    assert out.shape == (1, 64, 3, 3)
    ok = ~torch.isnan(out)
    assert ok.any() and float(out[ok].min()) >= -0.5 and float(out[ok].max()) < 0.5
    # the decoder leg against the CPU oracle on the prefix this GPU's encoder produced: bit-exact ids
    ids = model.last_ids.cpu()
    _, prefix = model.point_encoder._last
    ref, _ = OracleDecoder(sd, 24, 257 + 9 * 64 + 2).generate(prefix[0].cpu(), 9 * 64 + 2)
    assert ids[0].tolist()[:len(ref)] == ref


@gpu
def test_config1_chain_against_reference_modules():
    """BASELINE configs[0] on the GPU against tests/golden/config1_chain.npz (reference Dataset -> reference
    AlignedShapeLatentPerceiver -> decoder oracle -> HF BertEncoder detokenizer, see make_golden_config1.py):
      * decoder: greedy ids from the REFERENCE encoder's prefix are the committed ids, bit for bit (578 tokens);
      * encoder: ma_encoder_forward on the mouse point cloud within the encoder tolerances of DESIGN.md section 6 of the
        reference modules' output (fixture stored as fp16);
      * detokenizer: ma_detokenize on the committed ids / point_feature gives the HF BertEncoder's bins (>= 97 %)."""
    import os
    import numpy as np
    from meshanything_b200.decoder import DecoderArena, Generator
    from meshanything_b200.encoder import EncoderArena, TokenizerArena
    g = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    pc = torch.from_numpy(np.load(os.path.join(g, "config1_mouse.npz"))["pc_normal"][None])
    fx = np.load(os.path.join(g, "config1_chain.npz"))
    sd = ck.synthetic_state_dict(0)
    n = 9 * 64 + 2
    ref_prefix = torch.from_numpy(fx["prefix"]).float()
    ids, lens = Generator(DecoderArena(sd, _dev()), 1, 257 + n).generate(ref_prefix[None].to(_dev()), n)
    assert int(lens[0]) == n and ids[0].cpu().tolist() == fx["ids"].astype(np.int64).tolist()
    pf, prefix = EncoderArena(sd, _dev()).forward(pc.to(_dev()))
    ref_pf = torch.from_numpy(fx["point_feature"]).float()
    e_pf, e_pre = (pf[0].cpu() - ref_pf).abs(), (prefix[0].cpu() - ref_prefix).abs()
    print(f"config 1 encoder vs the reference modules: point_feature max {float(e_pf.max()):.4f} mean {float(e_pf.mean()):.5f}, "
          f"prefix max {float(e_pre.max()):.4f} mean {float(e_pre.mean()):.5f}")
    assert e_pf.max() < 1.5e-2 + 2e-3 and e_pf.mean() < 2.5e-3 and e_pre.max() < 4e-2 + 4e-3 and e_pre.mean() < 6e-3
    coords = TokenizerArena(sd, _dev()).detokenize(torch.from_numpy(fx["ids"].astype(np.int32))[None].to(_dev()),
                                                   ref_pf[None].to(_dev()), 64)
    ref_coords = torch.from_numpy(fx["bins"].astype(np.float32)).view(64, 3, 3) / 128 - 0.5
    assert not torch.isnan(coords).any()
    assert float((coords[0].cpu() == ref_coords).float().mean()) >= 0.97
