"""The oracle's gradients (torch autograd through oracle/kpnerf_oracle.py) against the gradients of the unmodified reference
(tests/golden/make_golden_grad.py: batch_render_pifu_nerf's eval branch with autograd, uniform=True).  CPU only.

The oracle runs in fp32 like the reference, at the reference's rays and fine depths.  Gate per tensor: relative L2 error and
largest absolute error (over the largest absolute reference value) within 1e-5, or within the fp64 oracle's own distance from the
golden where the reference's fp32 round-off is larger than that: the fp32 oracle is then no further from the reference than the
exact gradient is (grad_v4_k17's density head: the reference's fp32 gradients are 1.2e-4 from the fp64 ones).  The last colour
layer's bias has exact gradient 0 (the softmax over views is shift invariant): both values must be round-off below 1e-4 of that
layer's weight gradient.
"""
import pytest
import torch

from tests import grad_oracle as GO

SP = {"sp_level": 3, "scale": 1.0, "sigma": 0.1}
GATE = 1e-5
ZERO_GRAD = "mlp_tex.out_layer.4.bias"


@pytest.mark.parametrize("name", GO.GRAD_CASES)
def test_oracle_gradients_match_reference(name):
    g, meta, scene, weights, rays, G = GO.load_grad_case(name)
    args = (scene, weights, SP, rays, meta["S_c"], meta["S_f"], g["z_fine"], G)
    w32, m32, out = GO.oracle_grads(*args, dtype=torch.float32)
    w64, m64, _ = GO.oracle_grads(*args, dtype=torch.float64)
    for k in GO.OUT_KEYS:   # the forward the gradients belong to
        o = out[k].detach()
        assert float((o.t() if k.startswith("tex_fg") else o).sub(torch.from_numpy(g[k])).abs().max()) < 1e-5, k
    rep, good = [], True
    scale = float(torch.from_numpy(g["g/mlp_tex.out_layer.4.weight"]).abs().max())
    for k, got, exact in [(k, w32[k], w64[k]) for k in w32] + [(k, m32[k], m64[k]) for k in GO.MAPS]:
        ref = g["g/" + k]
        if k == ZERO_GRAD:
            ok = float(got.abs().max()) <= 1e-4 * scale and float(abs(ref).max()) <= 1e-4 * scale
        else:
            e32, e64 = GO.rel_errors(got, ref), GO.rel_errors(exact, ref)
            ok = all(a <= max(GATE, b) for a, b in zip(e32, e64))
            if not ok or max(e32) > GATE:
                rep.append(f"{k}: fp32 {e32[0]:.1e}/{e32[1]:.1e}, fp64 {e64[0]:.1e}/{e64[1]:.1e}")
        good &= ok
    print(name + ": " + ("; ".join(rep) or "every gradient within 1e-5"))
    assert good, rep
