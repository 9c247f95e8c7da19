"""Tile scheduling of the three-warpgroup CTAs of the tensor-core engine (engine 0).

With 15-20 keypoints the geometry front kernel runs three warpgroups per CTA (20 samples per tile with 3 views, 16 with 4), and
the colour kernel always does (40 / 32 samples per tile).  Warpgroup w of CTA b shades tiles 3b + w, 3b + w + 3 * grid, ...  A
sample's result must not depend on the batch it is shaded in: the checks here shade the first n points of a pool for batch
sizes that leave warpgroups of the last CTA without a tile, end in a partial tile, and sit one below, at and one above one and
two full persistent waves (3 tiles per SM), and compare them bit for bit with the same points shaded in the whole pool.  Before
each call the output buffer's memory is filled with NaN, so a tile that no warpgroup shades shows up as NaN rows.  The whole
pool is also held to the fp32 engine (engine 1), so that a tile skipped or shaded twice in every batch is caught too.
"""
import numpy as np
import pytest
import torch

from keypointnerf_b200 import synthetic as syn
from keypointnerf_b200.testing import build_model, scene_tensors
from oracle import kpnerf_oracle as O  # checker only

pytestmark = pytest.mark.gpu

WGS = 3   # warpgroups per CTA of both kernels at these keypoint counts
# largest |engine 0 - engine 1| allowed per output on the whole pool: a coarse bound, about 10x the largest errors of either
# engine against the fp64 oracle at 18 keypoints (test_gpu_coverage); a tile shaded with another tile's samples is off by far more
GATE = dict(sdf=1e-2, rad=0.25, rgb=1e-3)


def _tile_rows(nv):
    """Samples per tile of the front kernel and of the colour kernel."""
    return 2 * (32 // nv), 4 * (32 // nv)


def _batch_sizes(nv, sms):
    ns = set()
    for rows in _tile_rows(nv):
        wave = WGS * sms * rows
        # 1..5 tiles and a wave plus one or two tiles: the last CTA has idle warpgroups; each also ends in a partial tile
        for tiles in (1, 2, 3, 4, 5, WGS * sms + 1, WGS * sms + 2):
            ns |= {tiles * rows, tiles * rows - rows // 2}
        ns |= {wave - 1, wave, wave + 1, 2 * wave - 1, 2 * wave, 2 * wave + 1}
    return sorted(ns)


def _pool(scene, n, seed=5):
    rng = np.random.default_rng(seed)
    kpt = scene["kpt3d"][0]
    cand = np.concatenate([rng.uniform([-0.5, -1.0, -0.5], [0.5, 1.0, 0.5], (3 * n, 3)),
                           kpt[rng.integers(0, len(kpt), n // 2)] + rng.normal(0.0, 0.015, (n // 2, 3))]).astype(np.float32)
    view = rng.normal(size=cand.shape)
    view = (view / np.linalg.norm(view, axis=-1, keepdims=True)).astype(np.float32)
    xy, z = O.project(scene, torch.from_numpy(cand))
    idx = rng.permutation(np.flatnonzero(O.validity(scene, xy, z).numpy()))[:n]
    assert idx.size == n, idx.size
    return torch.from_numpy(cand[idx]).cuda(), torch.from_numpy(view[idx]).cuda()


def _query(m, pts, view, engine=0):
    """query() with the memory its output is likely to reuse filled with NaN first."""
    junk = torch.full((pts.shape[0], 5), float("nan"), device=pts.device)
    del junk
    return m.query(pts, view, engine=engine)


@pytest.mark.parametrize("n_kpt,n_views", [(18, 3), (20, 3), (18, 4)])
def test_result_does_not_depend_on_the_batch_with_three_warpgroups(n_kpt, n_views):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sizes = _batch_sizes(n_views, sms)
    scene = syn.make_scene(src_size=512, n_views=n_views, n_kpt=n_kpt)
    weights = syn.make_weights(n_kpt)
    net = build_model(weights, n_kpt, "cuda:0")
    a = scene_tensors(scene, syn.make_target(size=512), "cuda:0")
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    pts, view = _pool(scene, max(sizes))

    full, valid = _query(m, pts, view)
    assert bool(valid.all()) and bool(torch.isfinite(full).all())
    ref, _ = m.query(pts, view, engine=1)
    err = {k: float((full[:, c] - ref[:, c]).abs().max()) for k, c in (("sdf", slice(0, 1)), ("rad", slice(1, 2)),
                                                                     ("rgb", slice(2, 5)))}
    assert all(err[k] <= GATE[k] for k in err), (err, GATE)

    bad = []
    for n in sizes:
        out, valid = _query(m, pts[:n], view[:n])
        if not (torch.equal(out, full[:n]) and bool(valid.all())):
            bad.append(n)
    m.check_health()
    assert not bad, f"{n_kpt} keypoints, {n_views} views: batches of {bad} samples differ from the whole pool"
