"""The backward of explicit ray batches (kpn_render_rays_backward) on one GPU.

    python tools/bench_grad.py [--steps 10] [--warmup 3] [--out FILE]

Shape: a 64 x 64 training patch (the reference's train_out_h / train_out_w) in the middle of the 512 x 512 bench frame, bench
scene (512^2 sources, 3 views), 64 coarse + 64 fine samples, 18 and 24 keypoints.  Reported per keypoint count, CUDA events on the
launch stream around each call (scene bound once): the forward (render_rays) on engines 0 and 1, the backward, the weight
re-upload a training step pays after an optimiser step (KeypointNeRF.marcher() after an in-place parameter update, host clock
around a synchronised call), and valid samples per second through the backward (both passes).  The oracle builds its tensors on
the CPU, so no torch-autograd baseline is measured on the GPU.  The card's name, power limit and max SM clock are read in the same
run.  Prints one JSON line per keypoint count; --out also writes them.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SIZE, PATCH, S_C, S_F = 512, 64, 64, 64


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    import __graft_entry__ as G
    from keypointnerf_b200 import synthetic as syn
    from keypointnerf_b200.testing import build_model, scene_tensors

    G.build()
    dev = "cuda:0"
    assert torch.cuda.is_available(), "bench_grad needs a CUDA device"
    lines = []
    for n_kpt in (18, 24):
        scene = syn.make_scene(src_size=SIZE, n_kpt=n_kpt)
        target = syn.make_target(size=SIZE)
        net = build_model(syn.make_weights(n_kpt), n_kpt, dev)
        a = scene_tensors(scene, target, dev)
        m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
        x0 = y0 = (SIZE - PATCH) // 2
        o, d, nf = m.camera_rays(K=a["cam_tar"]["K"], RT=a["cam_tar"]["RT"], znear=2.0, zfar=5.0, nx=SIZE, ny=SIZE)
        idx = torch.arange(PATCH, device=dev)
        sel = ((y0 + idx)[:, None] * SIZE + (x0 + idx)[None, :]).reshape(-1)
        o, d, nf = o[sel].contiguous(), d[sel].contiguous(), nf[sel].contiguous()
        n = o.shape[0]
        gen = torch.Generator(device=dev).manual_seed(0)
        gout = {k: torch.randn((3, n) if k.startswith("tex_fg") else (n,), generator=gen, device=dev)
                for k in ("tex_fg", "depth", "alpha", "tex_fg_fine", "depth_fine", "alpha_fine", "sdf")}
        st = torch.cuda.current_stream()

        def timed(fn):
            for _ in range(args.warmup):
                fn()
            ms = []
            for _ in range(args.steps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                fn()
                e1.record(st)
                e1.synchronize()
                ms.append(e0.elapsed_time(e1))
            return statistics.median(ms), min(ms), max(ms)

        kw = dict(S_c=S_C, S_f=S_F, fine=True)
        res = {"card": card(), "n_kpt": n_kpt, "rays": n, "samples_per_ray": S_C + S_F}
        for eng in (0, 1):
            res[f"forward_engine{eng}_ms"] = timed(lambda: m.render_rays(o, d, nf, engine=eng, **kw))
        res["backward_ms"] = timed(lambda: m.render_rays_backward(o, d, nf, gout, **kw))
        valid = m.stats()["samples_valid"]
        res["backward_valid_samples"] = valid
        res["backward_valid_samples_per_s"] = valid / (res["backward_ms"][0] * 1e-3)
        up = []
        p = net.mlp_tex.out_layer[4].bias
        for _ in range(args.steps):
            with torch.no_grad():
                p.add_(0.0)   # bumps the version, as an optimiser step does
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            net.marcher()
            torch.cuda.synchronize()
            up.append((time.perf_counter() - t0) * 1e3)
        res["weight_upload_ms"] = (statistics.median(up), min(up), max(up))
        res["oracle_autograd_baseline"] = "not measured (the oracle runs on CPU tensors)"
        line = json.dumps(res)
        print(line)
        lines.append(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
