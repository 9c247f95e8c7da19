"""Every geometry-front instantiation of the tensor-core engine, run for several tiles per warpgroup, against the fp64 oracle.

geo_front_kernel<NV, NP, GRID> is instantiated per view count (3, 4), keypoint pair count NP = 1..16 and sample source (rays and
points, or kpn_query_grid's grid).  A warpgroup runs tiles tile0, tile0 + grid * FWG, ... of the work list, and two kinds of fault
only show from its second tile on: state carried from one tile to the next (the prefetched work-list entry and sample of
front_opts' FO_NEXT_ID / FO_NEXT_SAMPLE, and their clamp to the last entry), and the activation tile, which the L3 rows overwrite
as fp32, so that every layer-0 word of the next tile has to be written again.  The frame-sized sweeps of test_gpu_kpt and
test_gpu_views shade fewer samples than one persistent wave, so they run each instantiation for one tile per warpgroup at most.

Here every (n_views, n_kpt) with n_views in {3, 4} and n_kpt in 1..32 queries the nodes of a grid over the subject's box, a set
where valid and invalid points interleave (the work list is not the identity) and that holds at least three front waves of valid
points.  Each case checks (a) the valid rows against the fp64 oracle, (b) the grid query (the GRID = true instantiation) against
the point query bit for bit, and (c) that a prefix of the points, shaded after the reversed set has left other samples' data in
every scratch buffer and with the output's memory filled with NaN, gives the same rows bit for bit, for prefixes whose valid count
sits around one tile, one, two and three waves; the grid query's prefixes of whole z slices are held to the same rows.  The odd
and the even count of a pair reach the same instantiations, so every front function is checked twice.
"""
import time

import numpy as np
import pytest
import torch

from keypointnerf_b200 import synthetic as syn
from keypointnerf_b200.testing import build_model, scene_tensors
from oracle import kpnerf_oracle as O  # checker only
from tests import mesh_ref as M
from tests.test_gpu_coverage import GATE
from tests.test_gpu_mesh import _grid_over
from tests.test_gpu_occupancy import _query
from tests.util import front_wgs, tile_samples

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
DIMS = (61, 67, 71)   # 290 177 grid nodes; no extent divides another, so the grid's rows do not line up with the tiles


def _box(scene):
    """The keypoints' box (scene["bounds"]) joined with the cube |x|, |y|, |z| <= 0.2 m about the subject's centre.  From 8
    keypoints on the box already holds the cube; one keypoint's box is 0.2 m wide, at the top of the visual hull where the
    masks' top rows are cut, and finds only 1 % of its nodes valid."""
    b = np.asarray(scene["bounds"], np.float64).reshape(2, 3)
    return np.stack([np.minimum(b[0], -0.2), np.maximum(b[1], 0.2)])


def _oracle_fp64(scene, weights, pts, view, chunk=1 << 15):
    outs, valid = [], []
    with O.precision(torch.float64):
        fw = O.fold_weights(weights)
        for s in range(0, pts.shape[0], chunk):
            o, v = O.query(scene, fw, torch.from_numpy(pts[s:s + chunk]), torch.from_numpy(view[s:s + chunk]))
            outs.append(o.numpy())
            valid.append(v.numpy())
    return np.concatenate(outs), np.concatenate(valid)


# Per-count exceptions to the per-sample gates of test_gpu_coverage (engine 0), measured on an H100 80GB HBM3 (700 W):
#   3 views, 10 keypoints: rgb 2.74e-4 (at one point; ten points of 42 287 are above 1.5e-4).  Not a layout fault: 9 keypoints
#     run the same front function (NP = 5) at 1.07e-4; the fp32 engine is at 3.0e-6 and the fp32 oracle at 3.1e-6 (the point is
#     well conditioned in fp32); engine 2 (same front and colour kernels, density tail without W_lo) is at 1.82e-4 with its
#     worst error at another point.  It is the fp16 rounding of the tensor-core path with these weights.
GATE_EXCEPTIONS = {(3, 10): dict(rgb=4e-4)}


def _prefix_targets(n_valid, sms, fwg, fspt):
    """Valid counts of the prefixes: around one tile, one that leaves warpgroups of the last CTA without a tile, around one
    wave, half a tile into the third wave, one below three waves, and every valid point."""
    wave = sms * fwg * fspt
    ks = {1, fspt - 1, fspt, fspt + 1, (sms * fwg - 1) * fspt + fspt // 2, wave - 1, wave, wave + 1, 2 * wave + fspt // 2,
          3 * wave - 1, n_valid}
    return sorted(ks)


@pytest.mark.parametrize("n_kpt", range(1, 33))
@pytest.mark.parametrize("n_views", [3, 4])
def test_front_instantiation_over_many_tiles(n_views, n_kpt):
    """(a) valid mask equal to the oracle's, invalid rows zero, valid rows within GATE[0] of the fp64 oracle (GATE_EXCEPTIONS
    per count); (b) query_grid equal to columns 0-1 of query; (c) prefixes of the point set and of the grid equal to the same rows
    of the whole set.  Prints, per case, the valid points, the tiles each front warpgroup runs and the worst error per output."""
    t0 = time.perf_counter()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    fwg, fspt = front_wgs(n_kpt), tile_samples(n_views)[0]
    wave = sms * fwg * fspt
    scene = syn.make_scene(src_size=64, n_views=n_views, n_kpt=n_kpt, fg_mode="hull", fg_hole=True)
    weights = syn.make_weights(n_kpt)
    net = build_model(weights, n_kpt, DEV)
    a = scene_tensors(scene, syn.make_target(size=16), DEV)
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])

    origin, spacing = _grid_over(_box(scene), DIMS)
    pts_np = M.grid_points(origin, spacing, DIMS).reshape(-1, 3)
    rng = np.random.default_rng(100 * n_views + n_kpt)
    view_np = rng.normal(size=pts_np.shape)
    view_np = (view_np / np.linalg.norm(view_np, axis=-1, keepdims=True)).astype(np.float32)
    xy, z = O.project(scene, torch.from_numpy(pts_np))
    want_valid = O.validity(scene, xy, z).numpy()   # fp32, the arithmetic of the kernels' validity test
    vidx = np.flatnonzero(want_valid)
    n_valid = vidx.size
    # the premise: at least three waves of valid points (every front warpgroup runs three tiles or more), interleaved with
    # invalid ones
    assert n_valid >= 3 * wave, (n_valid, 3 * wave)
    assert 0.05 < n_valid / pts_np.shape[0] < 0.95, n_valid / pts_np.shape[0]
    ntiles = -(-n_valid // fspt)

    pts, view = torch.from_numpy(pts_np).to(DEV), torch.from_numpy(view_np).to(DEV)

    # (a) the valid rows against the fp64 oracle, invalid rows zero
    full, valid = _query(m, pts, view, engine=0)
    valid_np = valid.cpu().numpy()
    full_np = full.cpu().numpy()
    assert np.array_equal(valid_np, want_valid), f"{int((valid_np != want_valid).sum())} points differ in validity"
    assert np.all(full_np[~valid_np] == 0.0)
    ref, ref_valid = _oracle_fp64(scene, weights, pts_np[vidx], view_np[vidx])
    # a point on the edge of a mask's 0.1 threshold may fall on either side in fp32 and fp64; the fp64 oracle's outputs for
    # a point it finds invalid are not the shaded ones, so such points (at most one in ten thousand) are not compared
    assert (~ref_valid).sum() <= n_valid // 10000, int((~ref_valid).sum())
    err = np.abs(full_np[vidx][ref_valid].astype(np.float64) - ref[ref_valid])
    worst = {"sdf": float(err[:, 0].max()), "rad": float(err[:, 1].max()), "rgb": float(err[:, 2:].max())}
    gate = dict(GATE[0], **GATE_EXCEPTIONS.get((n_views, n_kpt), {}))

    # (b) the grid query equals the point query at the same points
    out2, valid2 = m.query_grid(origin, spacing, DIMS, engine=0)
    grid_ok = torch.equal(valid2.reshape(-1), valid) and torch.equal(out2.reshape(-1, 2), full[:, :2])

    # (c) prefixes of the point set, each after the reversed set has filled the work list and the scratch buffers
    rpts, rview = pts.flip(0).contiguous(), view.flip(0).contiguous()
    targets = _prefix_targets(n_valid, sms, fwg, fspt)
    bad = []
    for k in targets:
        assert 1 <= k <= n_valid
        n = int(vidx[k - 1]) + 1
        m.query(rpts, rview, engine=0)
        out, vp = _query(m, pts[:n], view[:n], engine=0)
        if not (torch.equal(out, full[:n]) and torch.equal(vp, valid[:n])):
            bad.append(k)
    # the grid's prefixes are its first nz z slices (x fastest): for each target, the fewest slices that hold that many valid
    # points
    slab = DIMS[0] * DIMS[1]
    valid_in_slices = want_valid.reshape(DIMS[2], slab).sum(1).cumsum()
    bad_grid = []
    for nz in sorted({int(np.searchsorted(valid_in_slices, k)) + 1 for k in targets}):
        n = nz * slab
        m.query(rpts, rview, engine=0)
        junk = torch.full((n, 2), float("nan"), device=DEV)
        del junk
        o2, v2 = m.query_grid(origin, spacing, (DIMS[0], DIMS[1], nz), engine=0)
        if not (torch.equal(o2.reshape(-1, 2), full[:n, :2]) and torch.equal(v2.reshape(-1), valid[:n])):
            bad_grid.append(nz)
    m.check_health()

    print(f"{n_views} views, {n_kpt:2d} keypoints: {n_valid} valid of {pts_np.shape[0]} ({n_valid / pts_np.shape[0]:.1%}), "
          f"{ntiles // (sms * fwg)}-{-(-ntiles // (sms * fwg))} tiles per warpgroup ({fwg} per CTA); "
          + " ".join(f"{k} {v:.2e}" for k, v in worst.items())
          + f"; grid {'==' if grid_ok else '!='} query; prefixes {'ok' if not bad else bad}; grid prefixes "
          + f"{'ok' if not bad_grid else bad_grid}; {time.perf_counter() - t0:.1f} s")
    assert all(worst[k] <= gate[k] for k in worst), (worst, gate)
    assert grid_ok, "kpn_query_grid differs from kpn_query at the same points"
    assert not bad, f"prefixes with {bad} valid points differ from the same rows of the whole set"
    assert not bad_grid, f"grid prefixes of {bad_grid} z slices differ from the same rows of the whole set"
