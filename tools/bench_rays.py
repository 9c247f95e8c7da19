"""Explicit ray batches (kpn_render_rays) against the lattice render they replace, on one GPU.

    python tools/bench_rays.py [--runs 3] [--steps 10] [--warmup 3] [--out FILE]

Three comparisons, the two arms of each alternating (--runs of each, --steps timed calls per run), CUDA events on the launch
stream around each call with the scene bound once (the atlases are not re-packed), L2 flushed between calls:
  frame      config-2 frame (512x512 target, 128 samples/ray, bench scene, 3 views, 18 keypoints): render vs camera_rays +
             render_rays of the same rays;
  turntable  90 cameras of 128x128 around the subject, 128 samples/ray: render_views-style per-camera render calls vs ONE
             render_rays call over the concatenated rays (built by camera_rays outside the timed region);
  silhouette the silhouette ("hull") scene's 512x512 frame vs render_rays of only its mask_at_box pixels (the rays that meet the
             bounding box, selected outside the timed region).
The card's name, power limit and max SM clock are read in the same run.  Prints one JSON line per run and a summary; --out also
writes the summary.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SIZE, S_C, N_KPT = 512, 128, 18


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    import __graft_entry__ as G
    from keypointnerf_b200 import synthetic as syn
    from keypointnerf_b200.testing import build_model, scene_tensors
    from oracle import kpnerf_oracle as O

    G.build()
    dev = "cuda:0"
    assert torch.cuda.is_available(), "bench_rays needs a CUDA device"
    net = build_model(syn.make_weights(N_KPT), N_KPT, dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def bind(scene):
        a = scene_tensors(scene, syn.make_target(8), dev)
        return net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])

    def lattice(t):
        return dict(K=torch.from_numpy(t["K"]).to(dev), RT=torch.from_numpy(t["RT"]).to(dev), znear=2.0, zfar=5.0, x0=0, y0=0,
                    step=1, nx=int(t["width"]), ny=int(t["height"]))

    def timed(fn, steps):
        ms = []
        for _ in range(steps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        return statistics.median(ms)

    benches = {}
    # config-2 frame
    m = bind(syn.make_scene(512, 3, N_KPT, fg_mode="ones"))
    lat2 = lattice(syn.make_target(SIZE, azimuth=1.0))
    m.reserve(SIZE * SIZE, S_C)
    benches["frame"] = (m, lambda: m.render(**lat2, S_c=S_C, out_device="cuda"),
                        lambda: m.render_rays(*m.camera_rays(**lat2), S_c=S_C), SIZE * SIZE)
    # 90-camera 128^2 turntable
    cams = [lattice(syn.make_target(128, azimuth=2 * np.pi * i / 90, zoom=1.0)) for i in range(90)]
    rays = [torch.cat(x, 0) for x in zip(*[m.camera_rays(**c) for c in cams])]
    benches["turntable"] = (m, lambda: [m.render(**c, S_c=S_C, out_device="cuda") for c in cams],
                            lambda: m.render_rays(*rays, S_c=S_C), 90 * 128 * 128)
    # silhouette scene: full frame vs its mask_at_box pixels
    hull = syn.make_scene(512, 3, N_KPT, fg_mode="hull")
    net2 = build_model(syn.make_weights(N_KPT), N_KPT, dev)
    ah = scene_tensors(hull, syn.make_target(8), dev)
    mh = net2._bind_scene(ah["cam"], ah["feat_geo"], ah["feat_tex"], ah["sp_data"], ah["img"], ah["fg"], ah["bounds"])
    mh.reserve(SIZE * SIZE, S_C)
    oh, dh, nfh = mh.camera_rays(**lat2)
    box = O.ray_bbox(hull["bounds"], oh.cpu(), dh.cpu())[2][:, 0].to(dev)
    sel = [oh[box].contiguous(), dh[box].contiguous(), nfh[box].contiguous()]
    benches["silhouette"] = (mh, lambda: mh.render(**lat2, S_c=S_C, out_device="cuda"), lambda: mh.render_rays(*sel, S_c=S_C),
                             SIZE * SIZE)

    name = card()
    summary = {"card": name, "steps": args.steps, "runs": args.runs, "note": "median CUDA-event ms per call of each run"}
    for key, (mm, base, new, rays_n) in benches.items():
        for _ in range(args.warmup):
            base(); new()
        torch.cuda.synchronize()
        rb, rn = [], []
        for r in range(args.runs):
            rb.append(timed(base, args.steps))
            rn.append(timed(new, args.steps))
            print(json.dumps({"bench": key, "run": r, "lattice_ms": rb[-1], "rays_ms": rn[-1]}), flush=True)
        summary[key] = {"lattice_ms": rb, "rays_ms": rn, "rays_per_call": rays_n,
                        "rays_batch": int(sel[0].shape[0]) if key == "silhouette" else rays_n}
    mh.check_health()
    m.check_health()
    print(json.dumps(summary))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
