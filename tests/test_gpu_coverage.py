"""Inputs the golden-vector tests never reach: batch composition and partial tiles of the shading kernels, multi-chunk renders
and queries, and the per-sample error of every engine against the fp64 oracle.

Shading a sample must not depend on which other samples share its tile or its launch: the geometry front kernel takes 20
samples per tile, the density tail 64 and the colour kernel 40, ghost rows of a partial tile are clamped onto the last valid
sample and never written.  A stale shared-memory column, a ghost row that leaks into a written row or a wrong bias / padding
word changes some sample's result with the batch it is shaded in, which the checks here see bit for bit.  Renders and
queries are split into chunks (renders at 32 Mi samples, or ``KPN_CHUNK_SAMPLES``; queries at 4 Mi points), and every chunk
writes its part of the outputs and of the statistics at its own offsets: a frame must be bit-identical however it is split.

Per-sample accuracy is measured on a pool of points the oracle finds valid in the bench scene, labelled by the regime it
exercises (interior, clamped border taps, near a keypoint, far from every keypoint, small boundary weight), against the oracle
run in fp64.  Each gate below is 2-3x the largest error measured on an H100 80GB HBM3 (700 W power limit) over all families,
or the gate the other tests hold the engine to where that is tighter (numbers per family are printed).
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from keypointnerf_b200 import distributed as D
from keypointnerf_b200 import synthetic as syn
from keypointnerf_b200.testing import build_model, scene_tensors
from oracle import kpnerf_oracle as O  # checker only
from tests import chunk_worker
from tests.util import COLOUR_WGS, TAIL_WGS, front_wgs, tile_samples

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# samples per tile and warpgroups per CTA (one CTA per SM) of the geometry front kernel at 18 keypoints, the density tail and
# the colour kernel
TILE_ROWS = tile_samples(3)
WGS = (front_wgs(18), TAIL_WGS, COLOUR_WGS)

# Per-sample gates against the fp64 oracle, per engine and output.  Largest errors measured on an H100 (all families):
#   engine 0 (wgmma, two-term density tail): sdf 9.13e-4, rad 2.62e-2, rgb 5.60e-5.  The rad gate stays at the 5e-2 the other
#     tensor-core tests use (1.9x); sdf and rgb are tightened from 5e-3 / 5e-4.
#   engine 1 (fp32 CUDA cores): sdf 2.02e-5, rad 6.20e-4, rgb 2.89e-5.  These are the fp32 oracle's own distances from the fp64
#     one on the same pool (fp32 round-off of the projection, amplified by the x30 density gain on rad), so rad is gated at
#     1.5e-3, not at the 1e-4 of the other outputs.
#   engine 2 (wgmma, density tail without W_lo): sdf 8.56e-4, rad 3.01e-2, rgb 6.80e-5.
GATE = {
    0: dict(sdf=2.5e-3, rad=5e-2, rgb=1.5e-4),
    1: dict(sdf=5e-5, rad=1.5e-3, rgb=7e-5),
    2: dict(sdf=2.5e-3, rad=7e-2, rgb=1.5e-4),
}


def _unproject(KRT, W, H, view, u, v, zc):
    """World points that view ``view`` sees at normalised image coordinates (u, v) and camera depth zc."""
    x, y = (u + 1.0) * 0.5 * (W - 1.0), (v + 1.0) * 0.5 * (H - 1.0)
    h = np.stack([x * zc, y * zc, zc], -1) - KRT[view, :3, 3]
    return h @ np.linalg.inv(KRT[view, :3, :3]).T


def build_pool(scene, n=40000, seed=7):
    """About ``n`` points (and view directions) that the oracle finds valid in ``scene``, shuffled, with their families.
    Candidates: a box around the keypoints, gaussian clouds around the keypoints, a wide box, and points just inside / just
    outside the image edges of each source view (normalised |u| or |v| in (0.8, 1.01])."""
    rng = np.random.default_rng(seed)
    KRT = scene["KRT"].astype(np.float64)
    W, H = float(scene["width"]), float(scene["height"])
    kpt = scene["kpt3d"][0].astype(np.float64)

    def edge(count, lo, hi):
        view, side = rng.integers(0, 3, count), rng.integers(0, 4, count)
        mag = rng.uniform(lo, hi, count) * np.where(side % 2 == 0, 1.0, -1.0)
        other = rng.uniform(-0.6, 0.6, count)
        u, v = np.where(side < 2, mag, other), np.where(side < 2, other, mag)
        zc = rng.uniform(2.2, 3.8, count)
        return np.concatenate([_unproject(KRT, W, H, i, u[view == i], v[view == i], zc[view == i]) for i in range(3)])

    cand = np.concatenate([
        rng.uniform([-0.5, -1.0, -0.5], [0.5, 1.0, 0.5], (12000, 3)),
        kpt[rng.integers(0, len(kpt), 5000)] + rng.normal(0.0, 0.015, (5000, 3)),
        rng.uniform(-1.5, 1.5, (12000, 3)),
        edge(32000, 1.0, 1.01),
        edge(16000, 0.8, 1.0),
    ]).astype(np.float32)
    view = rng.normal(size=cand.shape)
    view = (view / np.linalg.norm(view, axis=-1, keepdims=True)).astype(np.float32)
    xy, z = O.project(scene, torch.from_numpy(cand))
    valid = O.validity(scene, xy, z).numpy()
    idx = rng.permutation(np.flatnonzero(valid))[:n]
    pts, view = cand[idx], view[idx]
    # families, from the oracle's own projection (fp64)
    with O.precision(torch.float64):
        xy, z = O.project(scene, torch.from_numpy(pts))
    xy, z = xy.numpy(), z.numpy()
    a = np.abs(xy).max(-1)                                                   # (V, N): larger of |u|, |v| per view
    d2 = ((pts.astype(np.float64)[:, None] - kpt[None]) ** 2).sum(-1)
    wk = np.exp(-d2 / (2.0 * 0.1 ** 2)).max(1)                               # largest keypoint-encoding weight (sigma 0.1)
    xyz = 0.5 * np.concatenate([xy, z], -1) + 0.5
    db = np.minimum(xyz, 1.0 - xyz)
    bw = (1.0 / (1.0 + np.exp(-5.0 * (db / 0.1 - 1.0)))).prod(-1).min(0)     # smallest un-normalised boundary weight of a view
    fam = {
        "interior": (a < 0.9).all(0) & (wk >= 1e-2) & (wk <= 0.9) & (bw > 0.05),
        "border_taps": ((a > 1.0) & (a <= 1.01)).any(0),
        "near_kpt": wk > 0.9,
        "far_kpt": wk < 1e-2,
        "small_bw": bw < 0.05,
    }
    return pts, view, fam


@pytest.fixture(scope="module")
def bench():
    scene = syn.make_scene(src_size=512, n_kpt=18)
    weights = syn.make_weights(18)
    target = syn.make_target(size=512)
    net = build_model(weights, 18, "cuda:0")
    a = scene_tensors(scene, target, "cuda:0")
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    return scene, weights, m, a


@pytest.fixture(scope="module")
def pool(bench):
    scene, weights, m, a = bench
    pts, view, fam = build_pool(scene)
    with O.precision(torch.float64):
        ref, valid = O.query(scene, O.fold_weights(weights), torch.from_numpy(pts), torch.from_numpy(view))
    assert bool(valid.all())
    return torch.from_numpy(pts).cuda(), torch.from_numpy(view).cuda(), fam, ref.numpy()


def batch_sizes():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ns = {1, 2, 19, 20, 21, 39, 40, 41, 63, 64, 65, 127, 128, 129}
    for rows, wgs in zip(TILE_ROWS, WGS):
        wave = sms * wgs * rows   # one full persistent wave of the kernel
        ns |= {wave - 1, wave, wave + 1, 2 * wave + 1}
    return sorted(ns)


def test_pool_families_and_validity(bench, pool):
    """Every family of the pool is populated, and the kernels' validity test agrees with the oracle's on all of it."""
    scene, weights, m, a = bench
    pts, view, fam, ref = pool
    counts = {k: int(v.sum()) for k, v in fam.items()}
    print(f"pool of {pts.shape[0]} valid points; families {counts}")
    assert pts.shape[0] >= 30000 and min(counts.values()) >= 200, counts
    for engine in (0, 1):
        _, valid = m.query(pts, view, engine=engine)
        assert bool(valid.all()), engine


@pytest.mark.parametrize("engine", [0, 1, 2])
def test_query_result_does_not_depend_on_the_batch(bench, pool, engine):
    """query(pool[:n]) equals the first n rows of query(pool) bit for bit, for batch sizes around every tile height and around
    one and two full persistent waves of each kernel; a permuted pool gives the permuted result."""
    scene, weights, m, a = bench
    pts, view, fam, ref = pool
    full, _ = m.query(pts, view, engine=engine)
    bad = []
    for n in batch_sizes():
        assert n <= pts.shape[0]
        out, valid = m.query(pts[:n], view[:n], engine=engine)
        if not (torch.equal(out, full[:n]) and bool(valid.all())):
            bad.append(n)
    gen = torch.Generator(device="cuda").manual_seed(11)
    perm = torch.randperm(pts.shape[0], generator=gen, device="cuda")
    out_p, _ = m.query(pts[perm], view[perm], engine=engine)
    m.check_health()
    assert not bad, f"engine {engine}: batches of {bad} samples differ from the same samples shaded in the whole pool"
    assert torch.equal(out_p, full[perm])


def test_engine_aliases_are_bit_identical(bench, pool):
    """Engines 3 and 4 run the same kernels as engine 0."""
    scene, weights, m, a = bench
    pts, view, fam, ref = pool
    o0, v0 = m.query(pts, view, engine=0)
    for engine in (3, 4):
        o, v = m.query(pts, view, engine=engine)
        assert torch.equal(o, o0) and torch.equal(v, v0), engine
    kw = dict(K=a["cam_tar"]["K"], RT=a["cam_tar"]["RT"], znear=2.0, zfar=5.0, x0=1, y0=2, step=4, nx=128, ny=128, S_c=32, S_f=32,
              fine=True, debug=True)
    f0 = m.render(engine=0, **kw)
    for engine in (3, 4):
        f = m.render(engine=engine, **kw)
        for k in f0:
            assert torch.equal(f[k], f0[k]), (engine, k)


@pytest.mark.parametrize("engine", [0, 1, 2])
def test_query_error_per_family_against_fp64_oracle(bench, pool, engine):
    """Per-sample error of each engine against the fp64 oracle, per family and output (sdf_raw, rad, rgb)."""
    scene, weights, m, a = bench
    pts, view, fam, ref = pool
    out, _ = m.query(pts, view, engine=engine)
    err = np.abs(out.cpu().numpy().astype(np.float64) - ref)
    cols = {"sdf": err[:, 0], "rad": err[:, 1], "rgb": err[:, 2:].max(1)}
    worst = {k: 0.0 for k in cols}
    for f, mask in fam.items():
        row = {k: float(v[mask].max()) for k, v in cols.items()}
        print(f"engine {engine} {f:12s} " + " ".join(f"{k} {v:.2e}" for k, v in row.items()))
        worst = {k: max(worst[k], row[k]) for k in cols}
    print(f"engine {engine} all          " + " ".join(f"{k} {v:.2e}" for k, v in worst.items()))
    gate = GATE[engine]
    assert all(worst[k] <= gate[k] for k in cols), (worst, gate)


def _frame_phases(m, kw, sub=2):
    """The frame and its sub x sub lattice phases (one rank's share each, reference pixel_shuffle assembly)."""
    before = m.stats()["kernel_launches"]
    frame = m.render(x0=0, y0=0, step=1, nx=1024, ny=1024, **kw)
    st = m.stats()
    frame_launches = st["kernel_launches"] - before
    phases, valid = [], 0
    for r in range(sub * sub):
        py, px, sy, sx = D.lattice_phase(r, sub * sub)
        before = m.stats()["kernel_launches"]
        phases.append(((py, px), m.render(x0=px, y0=py, step=sx, step_y=sy, nx=1024 // sx, ny=1024 // sy, **kw)))
        s = m.stats()
        valid += s["samples_valid"]
        phase_launches = s["kernel_launches"] - before
    return frame, st, frame_launches, phases, valid, phase_launches


@pytest.mark.parametrize("mode", ["coarse128", "fine64_ert"])
def test_multi_chunk_frame_equals_single_chunk_phases(bench, mode):
    """A 1024 x 1024 frame (4 chunks of 262144 rays) equals its 2 x 2 lattice phases (one chunk each) bit for bit on every output,
    including the per-sample compositing weights and resampled depths, and the valid-sample counts add up; the fine pass on the
    frame's own depths passed back as z_fine_override reproduces the fine outputs."""
    scene, weights, m, a = bench
    t = syn.make_target(size=1024)
    kw = dict(K=torch.from_numpy(t["K"]).cuda(), RT=torch.from_numpy(t["RT"]).cuda(), znear=2.0, zfar=5.0, debug=True)
    kw.update(dict(S_c=128) if mode == "coarse128" else dict(S_c=64, S_f=64, fine=True, ert_eps=1e-4))
    frame, st, frame_launches, phases, valid, phase_launches = _frame_phases(m, kw)
    assert frame_launches >= phase_launches + 3 * 3, (frame_launches, phase_launches)   # the frame really took 4 chunks
    assert st["samples_valid"] == valid and st["samples_total"] == 1024 * 1024 * (128 if mode == "coarse128" else 64 + 128)
    S = {"contrib": kw["S_c"], "z_fine": kw["S_c"] + kw.get("S_f", 0)}
    for (py, px), ph in phases:
        for k, v in ph.items():
            if k in S:   # per-ray rows (rays, S), row-major over the lattice
                f = frame[k].reshape(1024, 1024, S[k])[py::2, px::2].reshape(-1, S[k])
            else:
                f = frame[k][..., py::2, px::2]
            assert torch.equal(f, v), (mode, k, py, px)
    if mode == "fine64_ert":
        kw2 = dict(kw, debug=False)
        again = m.render(x0=0, y0=0, step=1, nx=1024, ny=1024, z_fine_override=frame["z_fine"].clone(), **kw2)
        for k in ("tex_fg_fine", "depth_fine", "alpha_fine", "sdf", "tex_fg", "alpha"):
            assert torch.equal(again[k], frame[k]), k
    m.check_health()


def _run_child(cfg, chunk_samples, out_dir):
    env = dict(os.environ, KPN_CHUNK_SAMPLES=str(chunk_samples))
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "chunk_worker.py"), cfg, str(out_dir)], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=600)
    print(p.stdout[-2000:], p.stderr[-4000:])
    assert p.returncode == 0 and "CHUNK_WORKER_OK" in p.stdout
    return dict(np.load(os.path.join(out_dir, cfg + ".npz")))


def _n_chunks(rays, smax, chunk_samples):
    rc = max(128, (chunk_samples // smax) // 128 * 128)   # rays per chunk, as the library computes it
    return -(-rays // rc)


@pytest.mark.parametrize("cfg,chunk_samples", [("partial", 65536), ("bench", 1 << 20)])
def test_small_chunks_in_a_child_process_equal_one_chunk(cfg, chunk_samples, tmp_path):
    """The same renders with KPN_CHUNK_SAMPLES set (many chunks; the last one partial for "partial", 32 chunks of one geometry
    slice each for the bench frame) and with the default (one chunk) are bit-identical, outputs and valid-sample counts."""
    assert "KPN_CHUNK_SAMPLES" not in os.environ, "the in-process side must use the default chunk size"
    child = _run_child(cfg, chunk_samples, tmp_path)
    here = chunk_worker.render_config(cfg)
    rays, smax = chunk_worker.SHAPES[cfg]
    n = _n_chunks(rays, smax, chunk_samples)
    assert n >= 13 and _n_chunks(rays, smax, 32 << 20) == 1
    assert set(child) == set(here)
    for k in sorted(here):
        if k.endswith(".launches"):   # the child's renders really ran chunk by chunk (>= 3 launches per extra chunk)
            assert child[k] >= here[k] + 3 * (n - 1), (k, int(child[k]), int(here[k]), n)
        else:
            assert np.array_equal(child[k], here[k]), k


@pytest.mark.parametrize("engine", [0, 1])
def test_multi_chunk_query_equals_split_calls(bench, engine):
    """4 Mi + 4099 points (two query chunks, the second partial) equal the same points in two calls, bit for bit."""
    scene, weights, m, a = bench
    n0 = 4 << 20
    n = n0 + 4099
    gen = torch.Generator(device="cuda").manual_seed(3)
    pts = (torch.rand(n, 3, generator=gen, device="cuda") - 0.5) * 3.0
    view = torch.nn.functional.normalize(torch.randn(n, 3, generator=gen, device="cuda"), dim=-1)
    before = m.stats()["kernel_launches"]
    full, vf = m.query(pts, view, engine=engine)
    st = m.stats()
    full_launches = st["kernel_launches"] - before
    o1, v1 = m.query(pts[:n0], view[:n0], engine=engine)
    c1 = m.stats()["samples_valid"]
    before = m.stats()["kernel_launches"]
    o2, v2 = m.query(pts[n0:], view[n0:], engine=engine)
    s2 = m.stats()
    m.check_health()
    assert 0.1 < float(vf.float().mean()) < 0.9
    assert torch.equal(vf, torch.cat([v1, v2])) and torch.equal(full, torch.cat([o1, o2]))
    assert st["samples_valid"] == c1 + s2["samples_valid"]
    assert full_launches >= 2 * (s2["kernel_launches"] - before)
