"""Config-2 frame (512x512 target, 128 samples/ray, bench scene, 18 keypoints, 512^2 sources) with 3 and with 4 source views.

    python tools/bench_views.py [--runs 3] [--steps 20] [--warmup 3] [--simt-steps 3] [--out FILE]

The 3- and 4-view runs alternate (--runs of each, --steps timed frames per run), then the fp32 engine (engine 1) renders the
4-view frame once.  A step is what bench.py times: re-bind the scene (the atlases are re-packed) and render the frame, CUDA
events on the launch stream, L2 flushed between steps.  A fourth view changes which samples are valid (every view must see a
sample), so besides ms/frame and rays/s each line gives samples_valid and ms per million valid samples.  The card's name and
power limit are read in the same run.  Prints one JSON line per run and a summary; --out also writes the summary.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SIZE, S_C, N_KPT = 512, 128, 18
AZIMUTHS = (0.0, 2.1, 4.2, 5.25)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def make_runner(n_views, dev):
    import torch
    from keypointnerf_b200 import synthetic as syn
    from keypointnerf_b200.testing import build_model, scene_tensors

    scene = syn.make_scene(512, n_views, N_KPT, fg_mode="ones", src_azimuths=AZIMUTHS)
    target = syn.make_target(SIZE, azimuth=1.0)
    net = build_model(syn.make_weights(N_KPT), N_KPT, dev)
    a = scene_tensors(scene, target, dev)
    m = net.marcher()
    m.reserve(SIZE * SIZE, S_C)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def step(engine):
        m.set_scene(KRT=a["cam"]["KRT"], extrin=a["sp_data"]["extrin"], kpt3d=a["sp_data"]["kpt3d"].reshape(-1, 3),
                    bounds=a["bounds"], feat64=a["feat_geo"][0], feat8=a["feat_geo"][1], feat_tex=a["feat_tex"], img=a["img"],
                    fg=a["fg"], width=scene["width"], height=scene["height"], znear=scene["znear"], zfar=scene["zfar"],
                    nml_scale=scene["nml_scale"])
        return m.render(K=a["cam_tar"]["K"], RT=a["cam_tar"]["RT"], znear=target["znear"], zfar=target["zfar"], x0=0, y0=0,
                        step=1, nx=SIZE, ny=SIZE, S_c=S_C, S_f=0, fine=False, engine=engine, out_device="cuda")

    def run(engine, steps, warmup):
        for _ in range(warmup):
            step(engine)
        torch.cuda.synchronize()
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        for e0, e1 in evs:
            flush.zero_()
            e0.record()
            step(engine)
            e1.record()
        torch.cuda.synchronize()
        ms = sum(e0.elapsed_time(e1) for e0, e1 in evs) / steps
        valid = m.stats()["samples_valid"]
        m.check_health()
        return {"n_views": n_views, "engine": engine, "steps": steps, "ms_per_frame": round(ms, 3),
                "rays_per_s": round(SIZE * SIZE / (ms * 1e-3)), "samples_valid": int(valid),
                "ms_per_million_valid": round(ms / (valid * 1e-6), 4) if valid else None}

    return run


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--simt-steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import __graft_entry__ as G

    G.build()
    assert torch.cuda.is_available(), "bench_views needs a CUDA device"
    runners = {v: make_runner(v, "cuda:0") for v in (3, 4)}
    lines = []
    for _ in range(args.runs):
        for v in (3, 4):
            r = runners[v](0, args.steps, args.warmup)
            lines.append(r)
            print(json.dumps(r), flush=True)
    r = runners[4](1, args.simt_steps, 1)
    lines.append(r)
    print(json.dumps(r), flush=True)
    summary = {"workload": f"{SIZE}x{SIZE} frame, {S_C} samples/ray, bench scene, {N_KPT} keypoints, 512^2 sources",
               "card": card(), "runs": lines}
    print(json.dumps(summary))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
