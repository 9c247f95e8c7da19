"""The colour kernel (shade_color_kernel<NV>) over several tiles per warpgroup, with 3 and 4 views, on both kinds of work list.

Each colour warpgroup runs tiles tile0, tile0 + grid * CWG, ... and fetches the next tile's inputs (work-list entry, sample,
projection, img / feat_tex taps, latent) while the current tile runs its stages; past the last tile that fetch is clamped to the
last entry.  A fault in that carry (a stale entry or latent, a missing clamp) only shows from a warpgroup's second tile on, or
at the end of the list.

Query mode: the colour work list is the first work list (the identity over an all-valid pool).  A shuffled pool of valid points
(consecutive tiles hold different rays and views) is shaded whole, then prefixes of it whose lengths sit around one tile and one,
two and three full persistent waves, each after the reversed pool has left other samples' data in the scratch buffers and with
the output's memory filled with NaN; every prefix must equal the same rows of the whole pool bit for bit.  The whole pool must
also equal the pool shaded in chunks of one wave, where no warpgroup runs a second tile, so that nothing is carried at all.

Render mode: colour_list_kernel's list is not the identity, and the latent is read through it.  A 4-view render_rays batch with
at least three colour waves must equal the same rays rendered in two calls bit for bit, and a small subset must agree with the
fp32 engine within the render gates of test_gpu_parity.
"""
import torch
import pytest

from keypointnerf_b200 import synthetic as syn
from keypointnerf_b200.testing import build_model, scene_tensors
from tests.test_gpu_occupancy import _pool, _query
from tests.test_gpu_parity import TOL
from tests.test_gpu_rays import _assert_bits, _flat
from tests.util import COLOUR_WGS, tile_samples

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _prefixes(sms, spt):
    wave = sms * COLOUR_WGS * spt
    ks = {1, spt - 1, spt, spt + 1}
    for w in (1, 2, 3):
        ks |= {w * wave - 1, w * wave, w * wave + 1}
    return sorted(ks)


@pytest.mark.parametrize("n_views", [3, 4])
def test_query_prefixes_equal_the_whole_pool(n_views):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    spt = tile_samples(n_views)[2]
    ks = _prefixes(sms, spt)
    n = ks[-1] + spt // 2 + 3   # the whole pool ends in a partial tile past the last prefix
    scene = syn.make_scene(src_size=128, n_views=n_views, n_kpt=18)
    net = build_model(syn.make_weights(18), 18, DEV)
    a = scene_tensors(scene, syn.make_target(size=16), DEV)
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    pts, view = _pool(scene, n, seed=11)

    full, valid = _query(m, pts, view)
    assert bool(valid.all()) and bool(torch.isfinite(full).all())
    rpts, rview = pts.flip(0).contiguous(), view.flip(0).contiguous()
    bad = []
    for k in ks:
        m.query(rpts, rview)
        out, vp = _query(m, pts[:k], view[:k])
        if not (torch.equal(out, full[:k]) and bool(vp.all())):
            bad.append(k)
    wave = sms * COLOUR_WGS * spt
    chunks = torch.cat([_query(m, pts[s:s + wave], view[s:s + wave])[0] for s in range(0, n, wave)])
    m.check_health()
    print(f"{n_views} views: pool {n}, {spt} samples per colour tile, prefixes {ks}: {'ok' if not bad else bad}; one-wave "
          f"chunks {'==' if torch.equal(chunks, full) else '!='} whole pool")
    assert not bad, f"prefixes {bad} differ from the same rows of the whole pool"
    assert torch.equal(chunks, full), "the pool shaded in one-wave chunks differs from the whole pool"


def test_render_rays_in_two_calls_equal_one_call():
    scene = syn.make_scene(src_size=128, n_views=4, n_kpt=18, fg_mode="hull")
    target = syn.make_target(size=256, azimuth=1.0)
    net = build_model(syn.make_weights(18), 18, DEV)
    a = scene_tensors(scene, target, DEV)
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    o, d, nf = m.camera_rays(K=a["cam_tar"]["K"], RT=a["cam_tar"]["RT"], znear=target["znear"], zfar=target["zfar"], x0=0, y0=0,
                             step=1, nx=256, ny=256)
    kw = dict(S_c=128)
    whole = _flat(m.render_rays(o, d, nf, **kw))
    coloured = m.stats()["samples_coloured"]
    wave = torch.cuda.get_device_properties(0).multi_processor_count * COLOUR_WGS * tile_samples(4)[2]
    assert coloured >= 3 * wave, (coloured, 3 * wave)

    R = o.shape[0]
    k = R // 3 + 7
    parts = [_flat(m.render_rays(o[s], d[s], nf[s], **kw)) for s in (slice(0, k), slice(k, R))]
    joined = {key: torch.cat([p[key] for p in parts], dim=-1 if key.startswith("tex_fg") else 0) for key in whole}
    _assert_bits(joined, whole)

    # a subset against the fp32 engine
    idx = torch.arange(R // 2 - 64, R // 2 + 64, device=DEV)
    r0 = _flat(m.render_rays(o[idx], d[idx], nf[idx], **kw))
    r1 = _flat(m.render_rays(o[idx], d[idx], nf[idx], **kw, engine=1))
    err = {key: float((r0[key] - r1[key]).abs().max()) for key in ("tex_fg", "alpha", "depth")}
    m.check_health()
    print(f"4 views: {R} rays, {coloured} coloured samples ({coloured / wave:.1f} waves); engine 0 vs 1: {err}")
    t = TOL[0]
    assert err["tex_fg"] <= t["rgb"] and err["alpha"] <= t["alpha"] and err["depth"] <= t["depth"], err
