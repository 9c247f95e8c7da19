"""Gradients of the oracle's eval branch on explicit rays by torch autograd, the gradient goldens of
tests/golden/make_golden_grad.py, and the comparison of the GPU's gradients with the oracle's that tests/test_gpu_grad.py and
tests/test_gpu_grad_edges.py make.  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import numpy as np
import torch

from keypointnerf_b200 import synthetic as syn
from oracle import kpnerf_oracle as O
from tests import rays_oracle as RO
from tests.util import checksum, load_golden, scene_from_meta

MAPS = ("feat64", "feat8", "feat_tex")
OUT_KEYS = ["tex_fg", "depth", "alpha", "tex_fg_fine", "depth_fine", "alpha_fine", "sdf"]
COARSE_KEYS = OUT_KEYS[:3]
GRAD_CASES = ["grad_v3_k18", "grad_v4_k17"]
DEV = "cuda:0"
# per gradient tensor: relative L2 error <= GATE and largest absolute error <= GATE x the largest absolute reference value
GATE = 1e-4


def oracle_grads(scene, weights, sp, rays, S_c, S_f, z_fine, G, dtype=torch.float64, fine=True):
    """dL/d every weight (by state_dict name) and feature map (by scene key) of L = sum_k <out_k, G_k>, G_k in kpn_out's plane
    layout ((3, n) / (n,)), with the fine pass (fine=True) at the constant depths z_fine.  Parameters and maps the loss does not
    reach get zeros.  Also returns the outputs."""
    with O.precision(dtype):
        w = {k: torch.tensor(np.asarray(v), dtype=dtype, requires_grad=True) for k, v in weights.items()}
        sc = dict(scene)
        for k in MAPS:
            sc[k] = torch.tensor(scene[k], dtype=dtype, requires_grad=True)
        zo = torch.as_tensor(z_fine).to(dtype) if fine else None
        out = RO.render_rays(sc, O.fold_weights(w), *rays, S_c, S_f, fine, sp, z_fine_override=zo)
        G = {k: torch.as_tensor(v) for k, v in G.items() if v is not None}
        loss = sum((out[k] * (G[k].t() if k.startswith("tex_fg") else G[k]).to(dtype)).sum() for k in G)
        loss.backward()
    grad = lambda v: v.grad if v.grad is not None else torch.zeros_like(v)
    return {k: grad(v) for k, v in w.items()}, {k: grad(sc[k]) for k in MAPS}, out


def load_grad_case(name):
    """(golden arrays, meta, scene, weights, rays (o, d, near_far) as torch fp32, loss weights G)."""
    g, meta, sha = load_golden(name)
    g = {k: np.array(v, copy=True, order="C") for k, v in g.items()}
    scene, weights, _ = scene_from_meta(meta)
    assert checksum(scene, weights) == sha
    rays = tuple(torch.from_numpy(g[k]) for k in ("rays_o", "rays_d", "near_far"))
    G = {k: torch.from_numpy(g["G/" + k]) for k in OUT_KEYS}
    return g, meta, scene, weights, rays, G


def rel_errors(got, ref):
    """(relative L2 error, largest absolute error / largest absolute reference value)."""
    got = torch.as_tensor(got).double().reshape(-1)
    ref = torch.as_tensor(ref).double().reshape(-1)
    nrm, mx = float(ref.norm()), float(ref.abs().max())
    return float((got - ref).norm()) / nrm, float((got - ref).abs().max()) / mx


# ---- the GPU side -----------------------------------------------------------------------------------------------------------
def lattice_rays(target, n):
    """The rays of an n x n lattice of the target camera (fp32, as the library marches them)."""
    pix = O.pixel_lattice(n, n, 1, 0, 0)
    o, d, n_r, f_r = O.ray_setup(pix, target["K"], target["RT"], float(target["znear"]), float(target["zfar"]))
    return o.expand(d.shape[0], 3).contiguous(), d.contiguous(), torch.cat([n_r, f_r], -1).contiguous()


def loss_weights(n, seed=11, keys=OUT_KEYS):
    gen = torch.Generator().manual_seed(seed)
    return {k: torch.randn((3, n) if k.startswith("tex_fg") else (n,), generator=gen) for k in keys}


def bind(scene, weights, sp, target, n_kpt, engine=1):
    """(model on engine `engine`, scene tensors) of a seeded scene."""
    from keypointnerf_b200.testing import build_model, scene_tensors
    net = build_model(weights, n_kpt, DEV, sp_args=sp)
    net.engine = engine
    return net, scene_tensors(scene, target, DEV)


def setup(n_views, n_kpt, sp_level, n, src_size=64, src_height=None):
    """Scene (hull masks), weights, sp, model on engine 1, scene tensors and the rays of an n x n lattice."""
    scene = syn.make_scene(src_size=src_size, n_views=n_views, n_kpt=n_kpt, fg_mode="hull", src_height=src_height)
    target = syn.make_target(size=n, zoom=2.0)
    sp = {"sp_level": sp_level, "scale": 1.0, "sigma": 0.1}
    weights = syn.make_weights(n_kpt, sp_level=sp_level)
    net, a = bind(scene, weights, sp, target, n_kpt)
    return scene, weights, sp, net, a, lattice_rays(target, n)


def gpu_grads(net, a, rays, S_c, S_f, G, fine=True):
    """loss.backward() through render_rays_grad on net.engine: (parameters by name, d maps by scene key, outputs)."""
    feats = [a["feat_geo"][0].clone().requires_grad_(), a["feat_geo"][1].clone().requires_grad_(), a["feat_tex"].clone().requires_grad_()]
    net.zero_grad(set_to_none=True)
    cfg = dict(sample_per_ray_c=S_c, sample_per_ray_f=S_f, fine=fine, uniform=True, src_foreground_mask=a["fg"], bounds=a["bounds"],
               feat_geo=feats[:2], feat_tex=feats[2])
    out = net.render_rays_grad(net, a["img"], a["cam"], *(t.to(DEV) for t in rays), sp_data=a["sp_data"], **cfg)
    loss = sum((out[k] * G[k].to(DEV)).sum() for k in G)
    loss.backward()
    torch.cuda.synchronize()
    return dict(net.named_parameters()), dict(zip(MAPS, (f.grad for f in feats))), out


def compare(got, ref, name, rep, gate=GATE):
    got, ref = got.detach().double().cpu().reshape(-1), ref.detach().double().cpu().reshape(-1)
    nrm = float(ref.norm())
    rel = float((got - ref).norm()) / nrm if nrm > 0 else float(got.norm())
    mx = float((got - ref).abs().max()) / max(float(ref.abs().max()), 1e-30) if nrm > 0 else float(got.abs().max())
    ok = rel <= gate and mx <= gate
    if not ok or rel > gate / 10:
        rep.append(f"{name}: rel L2 {rel:.2e}, max {mx:.2e}")
    return ok


def check_ani_al(g, ref, n_views, rep):
    """ani_al reaches the loss only through the blend weights Om_v = w_v / (sum w + 1e-8), w_v = ex_v - min ex.  Where a view's ex
    nearly ties with the minimum, its w_v is a difference of nearly equal exponentials that the fp32 forward resolves only to
    ~1e-7 / w_v relative (the backward rebuilds w_v with expm1, but the forward's Om_v and dot products carry that error), and dOm_v
    carries it into d ani_al: this one scalar is gated at 1e-3 relative.  With two views, w of one view is 0 and the other's
    Om = w / (w + 1e-8) depends on ani_al only through the 1e-8 term: its gradient is pure 1 / w^2 conditioning, and only its sign
    and size (within 2x) are checked.  A reference of exactly 0 (a loss without colour) wants exactly 0."""
    got, want = float(g), float(ref)
    ok = abs(got - want) <= 1e-3 * abs(want) if n_views != 2 else (got * want > 0 and 0.5 < got / want < 2.0) or got == want == 0.0
    if not ok or abs(got - want) > GATE * abs(want):
        rep.append(f"mlp_tex.ani_al: {got:.6e} vs {want:.6e}")
    return ok


def rel_l2(got, ref):
    got, ref = got.detach().double().cpu().reshape(-1), ref.detach().double().cpu().reshape(-1)
    return float((got - ref).norm()) / max(float(ref.norm()), 1e-30)


def compare_all(params, dmaps, w_ref, m_ref, n_views, rep, cancelling=()):
    """Every parameter gradient (params: name -> tensor) and every map gradient against the oracle's.  The biases
    named in `cancelling` (sums of many signed per-sample terms in the given case) are gated like the last colour bias: their
    largest absolute error against GATE x the largest absolute gradient of the same layer's weight."""
    good = True
    for k, ref in w_ref.items():
        g = params[k]
        assert g is not None and bool(torch.isfinite(g).all()), k
        if k in cancelling:
            wk = k[: -len(".bias")] + (".weight" if k[: -len(".bias")] + ".weight" in w_ref else ".weight_v")
            scale = float(w_ref[wk].abs().max())
            err = float((g.detach().double().cpu().reshape(-1) - ref.double().reshape(-1)).abs().max())
            ok = err <= GATE * scale
            rep.append(f"{k}: max error {err:.2e} = {err / scale:.1e} x max |d {wk}| (rel L2 {rel_l2(g, ref):.1e})")
            good &= ok
            continue
        if k == "mlp_tex.out_layer.4.bias":
            # the softmax over the views is shift invariant: the exact gradient of the last colour layer's bias is 0 (fp64 leaves
            # ~1e-17), so its error is gated against the scale of the same layer's weight gradient
            scale = float(w_ref["mlp_tex.out_layer.4.weight"].abs().max())
            ok = float(g.abs().max()) <= GATE * scale and float(ref.abs().max()) <= 1e-9 * scale
            if not ok:
                rep.append(f"{k}: |got| {float(g.abs().max()):.2e}, |ref| {float(ref.abs().max()):.2e}, scale {scale:.2e}")
            good &= ok
            continue
        if k == "mlp_tex.ani_al":
            good &= check_ani_al(g, ref, n_views, rep)
            continue
        good &= compare(g, ref.reshape(g.shape), k, rep)
    for k in MAPS:
        good &= compare(dmaps[k], m_ref[k], k, rep)
    return good


def check_against_oracle(net, a, scene, weights, sp, rays, S_c, S_f, fine=True, G=None, label="", cancelling=()):
    """render_rays_grad on net.engine against fp64 oracle autograd.  A debug render on the same engine gives the fine depths that
    render_rays_grad's forward resampled; the oracle renders at those, which leaves the arithmetic as the only difference.  G:
    dL/d outputs (default: seeded, every output of the passes run).  Returns (GPU parameter gradients by name, GPU map
    gradients, oracle weight gradients, oracle map gradients, oracle outputs, the debug render)."""
    n_views = int(np.asarray(scene["img"]).shape[0])
    m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
    fwd = m.render_rays(*(t.to(DEV) for t in rays), S_c=S_c, S_f=S_f, fine=fine, engine=net.engine, debug=True)
    z_fine = fwd["z_fine"].cpu() if fine else None
    if G is None:
        G = loss_weights(rays[0].shape[0], keys=OUT_KEYS if fine else COARSE_KEYS)
    params, dmaps, out = gpu_grads(net, a, rays, S_c, S_f, G, fine)
    assert set(out) == set(OUT_KEYS if fine else COARSE_KEYS)
    w_ref, m_ref, ref_out = oracle_grads(scene, weights, sp, rays, S_c, S_f, z_fine, G, fine=fine)
    assert float(fwd["alpha_fine" if fine else "alpha"].max()) > 0.05, "empty frame"
    rep = []
    good = compare_all({k: p.grad for k, p in params.items()}, dmaps, w_ref, m_ref, n_views, rep, cancelling=cancelling)
    print(f"{label}{n_views} views, {rays[0].shape[0]} rays, S {S_c}+{S_f if fine else 0}, engine {net.engine}: "
          + ("; ".join(rep) or "all within 1e-5"))
    assert good, rep
    m.check_health()
    return {k: p.grad for k, p in params.items()}, dmaps, w_ref, m_ref, ref_out, fwd
