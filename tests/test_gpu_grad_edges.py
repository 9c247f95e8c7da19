"""The backward of explicit ray batches at the edges tests/test_gpu_grad.py does not reach: the coarse-only pass, rays that miss,
start inside the box or come from several cameras, odd, minimal and maximal sample counts, losses on one output at a time, a
negative ani_al, clamped border taps of non-square sources, the tensor-core engines' fine depths, reproducibility, and batches of
several chunks.

Each case compares with fp64 oracle autograd as tests/test_gpu_grad.py does (tests/grad_oracle.py: the oracle renders at the fine
depths the GPU's forward resampled; every gradient within 1e-4 relative L2 and 1e-4 x max |ref|, with the documented exceptions
of the last colour bias and d ani_al), and asserts that it reaches the edge it is named for.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from keypointnerf_b200 import synthetic as syn
from keypointnerf_b200.model import param_grads
from oracle import kpnerf_oracle as O  # checker only
from tests import grad_chunk_worker as W
from tests import grad_oracle as GO
from tests.util import checksum, load_golden, scene_from_meta

pytestmark = pytest.mark.gpu

DEV = GO.DEV
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SP3 = {"sp_level": 3, "scale": 1.0, "sigma": 0.1}
# The visibility gate's biases sum d v2 (a scalar per sample and view) over every sample with both signs; on the orthographic
# rays and the long rays that sum cancels to a few 1e-3 of its terms, and its fp32 result (the fp32 oracle's as well as the
# GPU's) is further than 1e-4 from exact.  There they are gated against the scale of their layer's weight gradient.
VIS_BIASES = ("mlp_tex.vis_layer2.0.bias", "mlp_tex.vis_layer2.2.bias")


def _valid(scene, rays, z):
    """The oracle's validity of the samples o + z d, (R, S) bool, and their normalised projections (V, R, S, 2)."""
    o, d, _ = rays
    z = torch.as_tensor(z).double()
    pts = (o.double()[:, None] + d.double()[:, None] * z[..., None]).reshape(-1, 3)
    with O.precision(torch.float64):
        xy, zz = O.project(scene, pts)
        v = O.validity(scene, xy, zz)
    return v.reshape(z.shape), xy.reshape(xy.shape[0], *z.shape, 2)


def _marcher(net, a):
    return net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])


def _raw(g):
    """dW, db and d ani_al of a render_rays_backward result, as one list of CPU tensors."""
    return [t.cpu() for t in list(g["dW"]) + list(g["db"]) + [g["d_ani_al"]]]


def _bits_equal(x, y):
    return all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(x, y))


# ---- 1. the coarse-only backward -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_views", [1, 3, 4])
def test_coarse_only_against_oracle(n_views):
    """fine=False: the coarse pass without compositing weights or resampling, and a RayGrad without sdf; only the three coarse
    outputs come back."""
    scene, weights, sp, net, a, rays = GO.setup(n_views, 18, 3, 12)
    GO.check_against_oracle(net, a, scene, weights, sp, rays, 16, 16, fine=False, label="coarse only: ")


# ---- 2. mixed, missing and inside-the-box rays -----------------------------------------------------------------------------
def _fixture(name):
    """The rays, scene and weights of a ray golden, and at most 12 x 12 of its rays: every ray the oracle finds a valid coarse
    sample on (up to 72, alternating between origins) and as many of the others, among them every ray that starts inside the box."""
    g, meta, sha = load_golden(name)
    scene, weights, _ = scene_from_meta(dict(meta, tgt_size=meta.get("tgt_size", 8), azimuth=meta.get("azimuth", 1.0)))
    assert checksum(scene, weights) == sha
    o, d, nf = (torch.from_numpy(np.array(g[k])) for k in ("rays_o", "rays_d", "near_far"))
    cnt = _valid(scene, (o, d, nf), torch.from_numpy(np.array(g["z_coarse"])))[0].sum(1)
    b = torch.as_tensor(scene["bounds"]).reshape(2, 3)
    inside = ((o >= b[0]) & (o <= b[1])).all(-1)
    hit_idx = torch.nonzero(cnt > 0)[:, 0]
    _, cam = torch.unique(o[hit_idx], dim=0, return_inverse=True)
    n_cam = int(cam.max()) + 1
    if n_cam <= 4:   # a few cameras (one origin each): an equal share of each
        hit_idx = torch.cat([hit_idx[cam == c][: 72 // n_cam] for c in range(n_cam)])
    hit_idx = hit_idx[:72]
    rest = torch.nonzero((cnt == 0) & inside)[:, 0]
    rest = torch.cat([rest, torch.nonzero((cnt == 0) & ~inside)[:, 0]])[: 144 - hit_idx.numel()]
    sel = torch.sort(torch.cat([hit_idx, rest])).values
    rays = tuple(t[sel].contiguous() for t in (o, d, nf))
    return meta, scene, weights, rays, cnt[sel], inside[sel]


@pytest.mark.parametrize("name", ["rays_ortho", "rays_mixed"])
def test_fixture_rays_against_oracle(name):
    meta, scene, weights, rays, cnt, inside = _fixture(name)
    o, d, nf = rays
    assert o.shape[0] <= 144
    near, far, hit = O.ray_bbox(scene["bounds"], o, d)
    hit = hit.reshape(-1)
    if name == "rays_ortho":
        # rays without a valid sample (cnt = 0) next to rays that hit, some of them through the box; origins inside the box
        assert int((cnt == 0).sum()) > 0 and int(((cnt == 0) & hit).sum()) > 0 and int((cnt > 0).sum()) > 0
        assert int(inside.sum()) > 0 and int((inside & (cnt > 0)).sum()) > 0
    else:
        # two cameras (two ray origins), four source views with holed masks, per-ray near / far
        assert torch.unique(o, dim=0).shape[0] == 2 and meta["n_views"] == 4 and meta["fg_hole"]
        assert int((cnt > 0).sum()) > 0 and int((cnt == 0).sum()) > 0 and torch.unique(nf, dim=0).shape[0] > 1
    net, a = GO.bind(scene, weights, SP3, syn.make_target(8), meta["n_kpt"])
    GO.check_against_oracle(net, a, scene, weights, SP3, rays, meta["S_c"], meta["S_f"], label=f"{name}: ",
                            cancelling=VIS_BIASES if name == "rays_ortho" else ())


# ---- 3. sample counts ------------------------------------------------------------------------------------------------------
def _crosses_groups(scene, rays, ref_out, fwd, fine):
    """Per pass: the largest valid-sample count of a ray, and whether some ray has more than 32 valid samples and not a multiple
    of 32 (composite_backward_kernel's suffix scan carries across a partial group)."""
    res = []
    for z in [ref_out["z"]] + ([fwd["z_fine"].cpu()] if fine else []):
        c = _valid(scene, rays, z)[0].sum(1)
        res.append((int(c.max()), bool(((c > 32) & (c % 32 != 0)).any())))
    return res


@pytest.mark.parametrize("S_c,S_f,fine", [(3, 1, True), (33, 31, True), (48, 17, True), (37, 0, False)])
def test_sample_counts_against_oracle(S_c, S_f, fine):
    scene, weights, sp, net, a, rays = GO.setup(3, 18, 3, 12)
    *_, ref_out, fwd = GO.check_against_oracle(net, a, scene, weights, sp, rays, S_c, S_f, fine=fine, label=f"S {S_c}+{S_f}: ")
    passes = _crosses_groups(scene, rays, ref_out, fwd, fine)
    print("per pass (largest count, crosses a partial group):", passes)
    assert all(mx > 0 for mx, _ in passes)
    if fine and S_c + S_f > 32:
        assert passes[-1][1]   # the fine pass' longest rays span more than one 32-entry group


def test_long_rays_against_oracle():
    """S_c = 256, S_f = 1024, the longest rays check_render accepts, on 4 x 4 rays: tens of 32-entry groups per ray."""
    scene, weights, sp, net, a, rays = GO.setup(3, 18, 3, 4)
    *_, ref_out, fwd = GO.check_against_oracle(net, a, scene, weights, sp, rays, 256, 1024, label="long rays: ",
                                               cancelling=VIS_BIASES)
    passes = _crosses_groups(scene, rays, ref_out, fwd, True)
    print("per pass (largest count, crosses a partial group):", passes)
    assert all(x for _, x in passes) and passes[1][0] > 10 * 32


# ---- 4. one output at a time -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key,fine", [(k, True) for k in GO.OUT_KEYS] + [(k, False) for k in GO.COARSE_KEYS])
def test_one_output_at_a_time_against_oracle(key, fine):
    """A loss of one output; every other plane is null."""
    scene, weights, sp, net, a, rays = GO.setup(3, 18, 3, 12)
    G = {key: GO.loss_weights(rays[0].shape[0], keys=[key])[key]}
    GO.check_against_oracle(net, a, scene, weights, sp, rays, 16, 16, fine=fine, G=G, label=f"only {key}: ")


def test_power_of_two_scaling_and_sum_of_parts():
    """2 G gives twice G's dW, db and d ani_al: scaling by 2 is exact in fp32 and the summation order is fixed.  Only products
    that fall below the normal range (they round on an absolute grid) may differ, so every difference from 2 x (G's result) must
    be smaller than the smallest normal float; the tensors doubled bit for bit are counted.  The sum of the gradients of G's
    seven one-output parts equals G's within 1e-5 relative L2 (measured on an H100: up to 2.7e-6, in the geometry layers, whose
    gradients amplify fp32 round-off; the seven parts round differently from the whole)."""
    scene, weights, sp, net, a, rays = GO.setup(3, 18, 3, 12)
    m = _marcher(net, a)
    r = [t.to(DEV) for t in rays]
    G = {k: v.to(DEV) for k, v in GO.loss_weights(r[0].shape[0]).items()}
    kw = dict(S_c=16, S_f=16, fine=True)
    one = _raw(m.render_rays_backward(*r, G, **kw))
    two = _raw(m.render_rays_backward(*r, {k: 2.0 * v for k, v in G.items()}, **kw))
    exact = sum(torch.equal(y, 2.0 * x) for x, y in zip(one, two))
    d2 = max(float((y - 2.0 * x).abs().max()) for x, y in zip(one, two))
    print(f"2 G vs 2 x G: {exact} of {len(one)} tensors exactly doubled; largest difference {d2:.2e}")
    assert d2 < torch.finfo(torch.float32).tiny   # nothing but the residues of subnormal products
    parts = [_raw(m.render_rays_backward(*r, {k: G[k]}, **kw)) for k in GO.OUT_KEYS]
    names = [n for n, _, _, _ in syn.layer_table(18)]
    labels = [f"dW {n}" for n in names] + [f"db {n}" for n in names] + ["d ani_al"]
    worst, bad = 0.0, []
    for i, (lab, full) in enumerate(zip(labels, one)):
        s = sum(p[i].double() for p in parts)
        if lab == "db mlp_tex.out_layer.4":   # exact gradient 0: gated against the same layer's weight gradient
            e = float((s - full.double()).abs().max()) / float(one[labels.index("dW mlp_tex.out_layer.4")].abs().max())
        else:
            e = float((s - full.double()).norm()) / max(float(full.double().norm()), 1e-30)
        worst = max(worst, e)
        if e > 1e-5:
            bad.append(f"{lab}: {e:.2e}")
    print(f"sum of the seven parts vs the whole: largest relative distance {worst:.2e}")
    assert not bad, bad
    m.check_health()


# ---- 5. negative ani_al ----------------------------------------------------------------------------------------------------
def test_negative_ani_al():
    """The layers see |ani_al|: the forward at -0.2 is the forward at +0.2 bit for bit, dW / db are the same bits, d ani_al is
    exactly minus the +0.2 value and matches the oracle (whose .abs() supplies the sign), and param_grads passes it on unchanged."""
    scene, weights, sp, net, a, rays = GO.setup(3, 18, 3, 12)
    neg = dict(weights, **{"mlp_tex.ani_al": np.array(-0.2, dtype=np.float32)})
    net_n, a_n = GO.bind(scene, neg, sp, syn.make_target(size=12, zoom=2.0), 18)
    assert float(net_n.mlp_tex.ani_al) == -float(net.mlp_tex.ani_al) < 0
    r = [t.to(DEV) for t in rays]
    kw = dict(S_c=16, S_f=16, fine=True)
    m_p, m_n = _marcher(net, a), _marcher(net_n, a_n)
    for engine in (0, 1):
        fp = m_p.render_rays(*r, engine=engine, debug=True, **kw)
        fn = m_n.render_rays(*r, engine=engine, debug=True, **kw)
        for k in fp:
            assert torch.equal(fp[k].view(torch.int32), fn[k].view(torch.int32)), (engine, k)
    G = {k: v.to(DEV) for k, v in GO.loss_weights(r[0].shape[0]).items()}
    gp, gn = m_p.render_rays_backward(*r, G, **kw), m_n.render_rays_backward(*r, G, **kw)
    assert _bits_equal(_raw(gp)[:-1], _raw(gn)[:-1])
    assert float(gp["d_ani_al"]) != 0.0 and float(gn["d_ani_al"]) == -float(gp["d_ani_al"])
    pg = param_grads(net_n, gn, net_n.hot_parameters())
    assert torch.equal(pg[-1].cpu(), gn["d_ani_al"].reshape(net_n.mlp_tex.ani_al.shape).cpu())
    params, *_ = GO.check_against_oracle(net_n, a_n, scene, neg, sp, rays, 16, 16, label="ani_al -0.2: ")
    assert torch.equal(params["mlp_tex.ani_al"].reshape(()).cpu(), gn["d_ani_al"].cpu())   # through autograd, same G, same bits


# ---- 6. non-square sources and clamped taps --------------------------------------------------------------------------------
def test_non_square_sources_and_border_taps():
    """64 x 24 sources, where the hull overflows the short side: valid samples project into the validity slack past the image
    edge (|u| or |v| in (1, 1.01]), where make_taps clamps; the map gradients match grid_sample(padding_mode="border")'s."""
    scene, weights, sp, net, a, rays = GO.setup(3, 18, 3, 12, src_size=64, src_height=24)
    assert scene["img"].shape[-2:] == (24, 64)
    *_, ref_out, fwd = GO.check_against_oracle(net, a, scene, weights, sp, rays, 64, 16, label="64 x 24 sources: ")
    border = 0
    for z in (ref_out["z"], fwd["z_fine"].cpu()):
        v, xy = _valid(scene, rays, z)
        mag = xy.abs().amax(-1)
        border += int((((mag > 1.0) & (mag <= 1.01)).any(0) & v).sum())
    print(f"valid samples on clamped border taps: {border}")
    assert border > 0


# ---- 7. the tensor-core engines --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("engine", [0, 2])
def test_tensor_core_engines_against_oracle(engine):
    """render_rays_grad with net.engine = 0 (the default) and 2 differentiates the fp32 recomputation at the fine depths that
    engine's forward resampled."""
    scene, weights, sp, net, a, rays = GO.setup(3, 18, 3, 12)
    net.engine = engine
    GO.check_against_oracle(net, a, scene, weights, sp, rays, 16, 16, label=f"engine {engine}: ")


def test_own_resampling_equals_the_engine1_depths():
    """Without z_fine_override the backward resamples itself: the same dW, db and d ani_al bits as at the engine-1 forward's z_fine."""
    scene, weights, sp, net, a, rays = GO.setup(3, 18, 3, 12)
    m = _marcher(net, a)
    r = [t.to(DEV) for t in rays]
    kw = dict(S_c=16, S_f=16, fine=True)
    z = m.render_rays(*r, engine=1, debug=True, **kw)["z_fine"]
    G = {k: v.to(DEV) for k, v in GO.loss_weights(r[0].shape[0]).items()}
    own = _raw(m.render_rays_backward(*r, G, **kw))
    given = _raw(m.render_rays_backward(*r, G, z_fine_override=z, **kw))
    assert _bits_equal(own, given)
    m.check_health()


# ---- 8. reproducibility ----------------------------------------------------------------------------------------------------
def test_weight_gradients_are_reproducible():
    """Five backward calls on the 32 x 32 patch with 64 + 64 samples, an unrelated call between each two: dW, db and d ani_al are
    the same bits every time; the feature-map gradients (float atomics) agree to 1e-5 (measured on an H100: 1.5e-6).  Without the
    canonical work list every repeat differed."""
    scene, weights, sp, net, a, rays = GO.setup(3, 24, 3, 32)
    m = _marcher(net, a)
    r = [t.to(DEV) for t in rays]
    kw = dict(S_c=64, S_f=64, fine=True)
    G = {k: v.to(DEV) for k, v in GO.loss_weights(r[0].shape[0]).items()}
    other = [t[::3].contiguous() for t in r]
    Go = {k: v[..., ::3].contiguous() for k, v in G.items()}
    runs, maps = [], []
    for i in range(5):
        g = m.render_rays_backward(*r, G, **kw)
        runs.append(_raw(g))
        maps.append([g["d_" + k].cpu() for k in GO.MAPS])
        if i % 2:
            m.render_rays_backward(*other, Go, **kw)
        else:
            m.render_rays(*other, engine=0, **kw)
    differ = [i for i in range(1, 5) if not _bits_equal(runs[0], runs[i])]
    mdist = max(float((x - y).norm() / y.norm()) for mp in maps[1:] for x, y in zip(mp, maps[0]))
    print(f"repeats whose dW / db / d ani_al differ from the first: {len(differ)} of 4; feature maps: largest rel L2 {mdist:.2e}")
    assert not differ and mdist <= 1e-5
    m.check_health()


# ---- 9. several chunks -----------------------------------------------------------------------------------------------------
def _grads(res, prefix=""):
    p = {k[len(prefix) + 2:]: torch.from_numpy(v) for k, v in res.items() if k.startswith(prefix + "p/")}
    mp = {k[len(prefix) + 2:]: torch.from_numpy(v) for k, v in res.items() if k.startswith(prefix + "m/")}
    return p, mp


_rel = GO.rel_l2


def test_several_chunks_in_a_child_process(tmp_path):
    """1300 rays x (64 + 64) samples with KPN_CHUNK_SAMPLES = 65536: three chunks of at most 512 rays, the last one partial, each
    reading the fine depths, dL/d outputs and gradient planes at its own offset.  Its gradients pass the oracle gate, equal the
    one-chunk gradients but for the summation order, and the gradients of the three ray ranges add up to those of their union
    (both within 1e-5 relative L2; measured on an H100: 3.1e-6 and 3.7e-6)."""
    assert "KPN_CHUNK_SAMPLES" not in os.environ, "the in-process side must use the default chunk size"
    env = dict(os.environ, KPN_CHUNK_SAMPLES="65536")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "grad_chunk_worker.py"), str(tmp_path)], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    print(p.stdout[-2000:], p.stderr[-4000:])
    assert p.returncode == 0 and "GRAD_CHUNK_WORKER_OK" in p.stdout
    child = dict(np.load(os.path.join(tmp_path, "grad_chunks.npz")))
    rc = 65536 // (W.S_C + W.S_F) // 128 * 128
    subsets = [(lo, min(lo + rc, W.N_RAYS)) for lo in range(0, W.N_RAYS, rc)]
    assert len(subsets) == 3 and subsets[-1][1] - subsets[-1][0] < rc
    here = W.grad_config(subsets)
    # the child really ran chunk by chunk (at least 3 launches per pass of every extra chunk)
    assert int(child["launches"]) >= int(here["launches"]) + 2 * 3 * (len(subsets) - 1), (int(child["launches"]), int(here["launches"]))
    assert np.array_equal(child["z_fine"], here["z_fine"])
    scene, weights, target, rays, G = W.inputs()
    w_ref, m_ref, _ = GO.oracle_grads(scene, weights, W.SP, rays, W.S_C, W.S_F, here["z_fine"], G)
    # this batch's geometry and density gradients amplify fp32 round-off: the fp32 oracle itself is up to 5e-4 from exact there.
    # As for the gradient goldens, a tensor is gated at twice the fp32 oracle's own error where that exceeds GATE / 2.
    w32, m32, _ = GO.oracle_grads(scene, weights, W.SP, rays, W.S_C, W.S_F, here["z_fine"], G, dtype=torch.float32)
    pc, mc = _grads(child)
    got, exact, f32 = dict(pc, **mc), dict(w_ref, **m_ref), dict(w32, **m32)
    rep, good = [], True
    for k, v in got.items():
        if k == "mlp_tex.out_layer.4.bias":   # exact gradient 0
            ok = float(v.abs().max()) <= GO.GATE * float(w_ref["mlp_tex.out_layer.4.weight"].abs().max())
        else:
            e, e32 = GO.rel_errors(v, exact[k].reshape(v.shape)), GO.rel_errors(f32[k].reshape(v.shape), exact[k].reshape(v.shape))
            gate = 1e-3 if k == "mlp_tex.ani_al" else GO.GATE
            ok = all(x <= max(gate, 2.0 * y) for x, y in zip(e, e32))
            if not ok or max(e) > gate / 10:
                rep.append(f"{k}: {e[0]:.1e}/{e[1]:.1e} (fp32 oracle {e32[0]:.1e}/{e32[1]:.1e})")
        good &= ok
    print("three chunks vs exact (rel L2 / max): " + ("; ".join(rep) or "all within 1e-5"))
    assert good, rep
    ph, mh = _grads(here)
    d_chunks = max(_rel(pc[k], ph[k]) for k in ph if k != "mlp_tex.out_layer.4.bias")
    d_chunks = max([d_chunks] + [_rel(mc[k], mh[k]) for k in mh])
    parts = [_grads(here, f"s{i}/") for i in range(len(subsets))]
    d_sum = max(_rel(sum(q[0][k] for q in parts), ph[k]) for k in ph if k != "mlp_tex.out_layer.4.bias")
    d_sum = max([d_sum] + [_rel(sum(q[1][k] for q in parts), mh[k]) for k in mh])
    print(f"three chunks vs one chunk: largest rel L2 {d_chunks:.2e}; sum of the three ranges vs their union: {d_sum:.2e}")
    assert d_chunks <= 1e-5 and d_sum <= 1e-5
