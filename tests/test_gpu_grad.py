"""Gradients of explicit ray batches on the GPU (kpn_render_rays_backward, RayMarcher.render_rays_backward,
KeypointNeRF.render_rays_grad) against torch autograd through the fp64 oracle.

The loss is a seeded linear combination of every output of both passes.  The oracle renders at the fine depths the GPU's own
forward resampled (the reference computes them under torch.no_grad, so they are constants of the backward), which leaves the
arithmetic as the only difference.  Gates per gradient tensor: relative L2 error <= 1e-4 and largest absolute error <= 1e-4 x the
largest absolute reference value.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from keypointnerf_b200 import _lib as L
from keypointnerf_b200 import synthetic as syn
from keypointnerf_b200.model import KeypointNeRF, param_grads
from keypointnerf_b200.renderer import RayMarcher
from keypointnerf_b200.testing import build_model, scene_tensors
from tests import grad_oracle as GO

pytestmark = pytest.mark.gpu

DEV = GO.DEV
MAPS = GO.MAPS
GATE = GO.GATE
SP3 = {"sp_level": 3, "scale": 1.0, "sigma": 0.1}
_setup = GO.setup
_loss_weights = GO.loss_weights


def _check_against_oracle(n_views, n_kpt, sp_level, n, S_c, S_f):
    scene, weights, sp, net, a, rays = _setup(n_views, n_kpt, sp_level, n)
    GO.check_against_oracle(net, a, scene, weights, sp, rays, S_c, S_f, label=f"{n_kpt} kpt, sp_level {sp_level}: ")


@pytest.mark.parametrize("n_views", [1, 2, 3, 4])
def test_every_view_count_against_oracle(n_views):
    _check_against_oracle(n_views, 18, 3, 12, 16, 16)


@pytest.mark.parametrize("n_kpt", [1, 17, 24, 32])
def test_keypoint_counts_against_oracle(n_kpt):
    _check_against_oracle(3, n_kpt, 3, 12, 16, 16)


@pytest.mark.parametrize("sp_level", [0, 2, 4])
def test_sp_levels_against_oracle(sp_level):
    _check_against_oracle(3, 18, sp_level, 12, 16, 16)


def test_training_patch_against_oracle():
    """A 32 x 32 patch with 64 + 64 samples at the reference's default of 24 keypoints."""
    _check_against_oracle(3, 24, 3, 32, 64, 64)


@pytest.mark.parametrize("engine", [0, 1])
def test_outputs_equal_render_rays(engine):
    scene, weights, sp, net, a, rays = _setup(3, 18, 3, 12)
    net.engine = engine
    cfg = dict(sample_per_ray_c=16, sample_per_ray_f=16, fine=True, uniform=True, src_foreground_mask=a["fg"], bounds=a["bounds"],
               feat_geo=a["feat_geo"], feat_tex=a["feat_tex"])
    r = [t.to(DEV) for t in rays]
    ref = net.render_rays(net, a["img"], a["cam"], *r, sp_data=a["sp_data"], **cfg)
    got = net.render_rays_grad(net, a["img"], a["cam"], *r, sp_data=a["sp_data"], **cfg)
    assert set(got) == set(ref)
    for k in ref:
        assert got[k].grad_fn is not None, k
        assert torch.equal(got[k].detach().view(torch.int32), ref[k].view(torch.int32)), k
    host = net.render_rays_grad(net, a["img"], a["cam"], *rays, sp_data=a["sp_data"], **cfg)   # CPU rays: CPU outputs, as render_rays
    for k in ref:
        assert not host[k].is_cuda and torch.equal(host[k].detach(), ref[k].cpu()), k


def _all_grads(g):
    return list(g["dW"]) + list(g["db"]) + [g["d_ani_al"], g["d_feat64"], g["d_feat8"], g["d_feat_tex"]]


def test_no_valid_sample_and_empty_batch_give_zero_gradients():
    scene, weights, sp, net, a, rays = _setup(3, 18, 3, 8)
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    o, d, nf = (t.to(DEV) for t in rays)
    away = -d   # rays that leave the scene: no valid sample
    G = {k: v.to(DEV) for k, v in _loss_weights(o.shape[0]).items()}
    kw = dict(S_c=16, S_f=16, fine=True)
    assert float(m.render_rays(o, away, nf, engine=1, **kw)["alpha"].abs().max()) == 0.0
    for g in (m.render_rays_backward(o, away, nf, G, **kw), m.render_rays_backward(o[:0], d[:0], nf[:0], {}, **kw)):
        for t in _all_grads(g):
            assert bool((t == 0).all())
    g = m.render_rays_backward(o, d, nf, G, **kw)
    assert float(g["d_feat64"].abs().max()) > 0 and float(g["dW"][0].abs().max()) > 0
    m.check_health()


def test_refusals():
    scene, weights, sp, net, a, rays = _setup(3, 18, 3, 8)
    r = [t.to(DEV) for t in rays]
    cfg = dict(sample_per_ray_c=16, sample_per_ray_f=16, fine=True, uniform=True, src_foreground_mask=a["fg"], bounds=a["bounds"],
               feat_geo=a["feat_geo"], feat_tex=a["feat_tex"])
    for bad in (dict(uniform=False), dict(rand_noise_std=0.1), dict(ert_eps=1e-3)):
        with pytest.raises(NotImplementedError):
            net.render_rays_grad(net, a["img"], a["cam"], *r, sp_data=a["sp_data"], **dict(cfg, **bad))
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    with pytest.raises(L.KpnError, match="status -4"):
        m.render_rays_backward(*r, {}, S_c=16, S_f=16, fine=True, ert_eps=1e-3)
    # weights but no scene: KPN_ERR_STATE
    fresh = RayMarcher(0)
    fresh.set_weights({k: torch.from_numpy(np.asarray(v)) for k, v in weights.items()}, n_kpt=18)
    rays_c, op, gout, gr = L.KpnRays(), L.KpnOpts(), L.KpnOut(), L.KpnGrads()
    buf = torch.zeros(1024, device=DEV)
    rays_c.origins, rays_c.dirs, rays_c.near_far, rays_c.n = r[0].data_ptr(), r[1].data_ptr(), r[2].data_ptr(), r[0].shape[0]
    op.sample_per_ray_c = 16
    for i in range(L.KPN_NUM_LAYERS):
        gr.dW[i], gr.db[i] = buf.data_ptr(), buf.data_ptr()
    gr.d_ani_al = gr.d_feat64 = gr.d_feat8 = gr.d_feat_tex = buf.data_ptr()
    rc = fresh.lib.kpn_render_rays_backward(fresh.ctx, C.byref(rays_c), C.byref(op), C.byref(gout), C.byref(gr), fresh._stream())
    assert rc == -3
    gr.d_feat8 = None
    rc = fresh.lib.kpn_render_rays_backward(fresh.ctx, C.byref(rays_c), C.byref(op), C.byref(gout), C.byref(gr), fresh._stream())
    assert rc == -1
    fresh.close()
    m.check_health()


def test_backward_reaches_the_encoders():
    """Without feat_geo / feat_tex the encoders run with autograd: loss.backward() leaves finite, non-zero gradients on the hot-path
    parameters and on the encoders' parameters."""
    scene, weights, sp, net, a, rays = _setup(3, 18, 3, 12, src_size=256)   # the encoders downsample 64x
    assert net.geo_encoder is not None and net.tex_encoder is not None
    cfg = dict(sample_per_ray_c=16, sample_per_ray_f=16, fine=True, uniform=True, src_foreground_mask=a["fg"], bounds=a["bounds"])
    for seed in range(26, 46):   # the first weights whose density is positive somewhere on the encoders' (random) features
        net.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in syn.make_weights(18, seed=seed).items()}, strict=False)
        with torch.no_grad():
            if float(net.render_rays(net, a["img"], a["cam"], *(t.to(DEV) for t in rays), sp_data=a["sp_data"], **cfg)["alpha"].max()) > 0.05:
                break
    net.zero_grad(set_to_none=True)
    out = net.render_rays_grad(net, a["img"], a["cam"], *(t.to(DEV) for t in rays), sp_data=a["sp_data"], **cfg)
    G = _loss_weights(rays[0].shape[0])
    sum((out[k] * G[k].to(DEV)).sum() for k in G).backward()
    for name, mod in (("hot", net.hot_parameters()), ("geo_encoder", list(net.geo_encoder.parameters())),
                      ("tex_encoder", list(net.tex_encoder.parameters()))):
        grads = [p.grad for p in mod if p.grad is not None]
        assert grads, name
        assert all(bool(torch.isfinite(g).all()) for g in grads), name
        assert sum(float(g.abs().sum()) for g in grads) > 0, name
    net.marcher().check_health()


def test_adam_fits_a_render_of_other_weights():
    """20 Adam steps on the hot-path parameters lower the L1 loss against a render of different weights."""
    scene, weights, sp, net, a, rays = _setup(3, 18, 3, 16)
    r = [t.to(DEV) for t in rays]
    cfg = dict(sample_per_ray_c=32, sample_per_ray_f=32, fine=True, uniform=True, src_foreground_mask=a["fg"], bounds=a["bounds"],
               feat_geo=a["feat_geo"], feat_tex=a["feat_tex"])
    other = build_model(syn.make_weights(18, seed=27), 18, DEV, sp_args=sp)
    other.engine = 1
    with torch.no_grad():
        tgt = other.render_rays(other, a["img"], a["cam"], *r, sp_data=a["sp_data"], **cfg)
    opt = torch.optim.Adam(net.hot_parameters(), lr=1e-3)
    losses = []
    for _ in range(20):
        opt.zero_grad()
        out = net.render_rays_grad(net, a["img"], a["cam"], *r, sp_data=a["sp_data"], **cfg)
        loss = sum((out[k] - tgt[k]).abs().mean() for k in ("tex_fg", "alpha", "tex_fg_fine", "alpha_fine"))
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    print("L1 per step: " + " ".join(f"{x:.4f}" for x in losses))
    assert min(losses[1:]) < losses[0] and losses[-1] < losses[0]
    net.marcher().check_health()


@pytest.mark.parametrize("name", GO.GRAD_CASES)
def test_gradients_match_reference_goldens(name):
    """At the unmodified reference's rays and fine depths (tests/golden/make_golden_grad.py): every gradient within 1e-4 (relative
    L2 and largest absolute error) of the exact one, the fp64 oracle's, which tests/test_grad_cpu.py pins to the reference's autograd.
    Where the reference's own fp32 gradient is further than 5e-5 from exact (grad_v4_k17's geometry and density layers: up to
    1.2e-4, with the fp32 oracle 2.8e-5 away from it), the case amplifies fp32 round-off for every implementation, and the gate is
    twice the reference's own error instead.  The distance to the reference's gradients is printed."""
    g, meta, scene, weights, rays, G = GO.load_grad_case(name)
    net = build_model(weights, meta["n_kpt"], DEV, sp_args=SP3)
    a = scene_tensors(scene, syn.make_target(8), DEV)
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    res = m.render_rays_backward(*(t.to(DEV) for t in rays), {k: v.to(DEV) for k, v in G.items()}, S_c=meta["S_c"], S_f=meta["S_f"],
                                 fine=True, z_fine_override=torch.from_numpy(g["z_fine"]))
    names = [n + s for n, _, _, wn in syn.layer_table(meta["n_kpt"]) for s in ((".weight_v", ".weight_g", ".bias") if wn else (".weight", ".bias"))]
    got = dict(zip(names + ["mlp_tex.ani_al"], param_grads(net, res, net.hot_parameters())))
    got.update({"feat64": res["d_feat64"], "feat8": res["d_feat8"], "feat_tex": res["d_feat_tex"]})
    w64, m64, _ = GO.oracle_grads(scene, weights, SP3, rays, meta["S_c"], meta["S_f"], g["z_fine"], G)
    exact = dict(w64, **m64)
    scale = float(torch.from_numpy(g["g/mlp_tex.out_layer.4.weight"]).abs().max())
    rep, good = [], True
    for k, v in got.items():
        v = v.detach().cpu()
        assert bool(torch.isfinite(v).all()), k
        if k == "mlp_tex.out_layer.4.bias":   # exact gradient 0 (the softmax over views is shift invariant)
            ok = float(v.abs().max()) <= GATE * scale
        else:
            gate = 1e-3 if k == "mlp_tex.ani_al" else GATE   # see GO.check_ani_al
            x = exact[k].reshape(v.shape)
            e, ex, e64 = GO.rel_errors(v, g["g/" + k]), GO.rel_errors(v, x), GO.rel_errors(x, g["g/" + k])
            ok = all(x <= max(gate, 2.0 * y) for x, y in zip(ex, e64))
            if not ok or max(e) > gate / 10:
                rep.append(f"{k}: vs exact {ex[0]:.1e}/{ex[1]:.1e}, vs reference {e[0]:.1e}/{e[1]:.1e} (exact vs reference "
                           f"{e64[0]:.1e}/{e64[1]:.1e})")
        good &= ok
    print(f"{name}: " + ("; ".join(rep) or "every gradient within 1e-5 of the reference"))
    assert good, rep
    m.check_health()
