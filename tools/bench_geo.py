"""Splits the shading time of one bench.py frame between its kernels: geo_front_kernel, geo_tail_kernel, the colour work list and
shade_color_kernel, plus everything else the frame launches (ray setup, compositing, the atlas re-layout).

    python tools/bench_geo.py [--config 2] [--scene ones] [--n-kpt 18] [--steps 10] [--warmup 3] [--out FILE]

The frame is bench.py's (same seeded scene, weights and target; config 2 by default: 512x512, 128 samples/ray, 3 views).  After
--warmup untimed frames, --steps frames run under torch.profiler with CPU and CUDA activities; each kernel's device time is
summed by name and divided by --steps.  The L2 flush before each frame runs inside its own record_function range, and the
kernels linked to it are subtracted.  The profiler adds host overhead between launches but not to the kernels' own device time.  The
card's name, power limit and maximum SM clock are read in the same run and printed with the result (one JSON line).

The line also sets geo_tail_kernel's time against the two floors its shapes give, at the H100 SXM data sheet's rates (3.35 TB/s
HBM3, 989 TFLOP/s dense fp16; figures the card is not claimed to reach): the bytes it must move (the 512-byte pooled row of every
valid sample in, its 8-byte alpha / sdf record and, for samples with density > 0, the 48-byte latent out) and the MMA work it
executes (per 64-sample tile, engine 0: P0|compress 26 m64n96k16 and P1 14 m64n64k16).  shade_color_kernel (colour_list
reported beside it) is set against the same two floors: the MMA work it executes (128 rows x 15 104 MAC per tile of 40 samples,
3 views) and the bytes its loads and stores request (per coloured sample: the 8-byte work-list entry, the ray's 32 bytes, the
48-byte latent, four 16-byte img and four 32-byte feat_tex taps per view, and the 12-byte colour out).
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

CONFIGS = {2: dict(size=512, S_c=128, S_f=0, fine=False, ert=0.0),
           3: dict(size=512, S_c=64, S_f=64, fine=True, ert=1e-4),
           4: dict(size=1024, S_c=128, S_f=0, fine=False, ert=0.0)}
GROUPS = ("geo_front_kernel", "geo_tail_kernel", "colour_list", "shade_color_kernel")
DATASHEET_BYTES_S = 3.35e12   # H100 SXM, HBM3
DATASHEET_FLOP_S = 989e12     # H100 SXM, dense fp16 tensor
TAIL_TILE_FLOP = 2 * 64 * 16 * (26 * 96 + 14 * 64)   # executed MMA work of one 64-sample tile with two-term weights (engine 0)
# executed MMA work of one colour tile (128 rows): sum of Kp x Np over RE1, BASE0, BASE1, VIS1A, VIS1B, VIS2A, OUT0
COLOUR_TILE_FLOP = 2 * 128 * (32 * 48 + 112 * 64 + 64 * 32 + 32 * 32 + 32 * 48 + 32 * 32 + 48 * 16)


def tail_floors(valid: int, coloured: int, tail_ms: float) -> dict:
    """geo_tail_kernel against the data sheet: the bytes it must move and the MMA work it executes, over its measured time."""
    nbytes = 512 * valid + 8 * valid + 48 * coloured
    flop = TAIL_TILE_FLOP * ((valid + 63) // 64)
    s = tail_ms * 1e-3
    return {"required_bytes": nbytes, "achieved_GB_s": round(nbytes / s / 1e9, 1) if s else None,
            "datasheet_GB_s": DATASHEET_BYTES_S / 1e9, "byte_floor_ms": round(nbytes / DATASHEET_BYTES_S * 1e3, 3),
            "executed_mma_flop": flop, "achieved_TFLOP_s": round(flop / s / 1e12, 1) if s else None,
            "datasheet_TFLOP_s": DATASHEET_FLOP_S / 1e12, "mma_floor_ms": round(flop / DATASHEET_FLOP_S * 1e3, 3)}


def colour_floors(coloured: int, n_views: int, list_ms: float, colour_ms: float) -> dict:
    """shade_color_kernel against the data sheet: the bytes its loads and stores request and the MMA work it executes."""
    spt = 4 * (32 // n_views)
    nbytes = coloured * (8 + 32 + 48 + 12 + n_views * 4 * (16 + 32))
    flop = COLOUR_TILE_FLOP * ((coloured + spt - 1) // spt)
    s = colour_ms * 1e-3
    return {"colour_list_ms": round(list_ms, 3), "shade_color_kernel_ms": round(colour_ms, 3), "requested_bytes": nbytes,
            "achieved_GB_s": round(nbytes / s / 1e9, 1) if s else None, "byte_floor_ms": round(nbytes / DATASHEET_BYTES_S * 1e3, 3),
            "executed_mma_flop": flop, "achieved_TFLOP_s": round(flop / s / 1e12, 1) if s else None,
            "mma_floor_ms": round(flop / DATASHEET_FLOP_S * 1e3, 3)}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError) as e:
        return f"nvidia-smi unavailable ({e})"


def group_of(name: str) -> str:
    for g in GROUPS:
        if g in name:
            return g
    return "other"


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--config", type=int, default=2, choices=sorted(CONFIGS))
    ap.add_argument("--scene", default="ones", choices=["ones", "hull"])
    ap.add_argument("--n-kpt", type=int, default=18)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile, record_function

    import __graft_entry__ as G
    from keypointnerf_b200 import synthetic as syn
    from keypointnerf_b200.testing import build_model, scene_tensors

    G.build()
    if not torch.cuda.is_available():
        sys.exit("bench_geo needs a CUDA device")
    cfg = CONFIGS[args.config]
    dev = "cuda:0"
    size = cfg["size"]
    scene = syn.make_scene(512, 3, args.n_kpt, fg_mode=args.scene)
    target = syn.make_target(size, azimuth=1.0)
    net = build_model(syn.make_weights(args.n_kpt), args.n_kpt, dev)
    a = scene_tensors(scene, target, dev)
    m = net.marcher()
    m.reserve(size * size, cfg["S_c"] + cfg["S_f"])
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def step():
        m.set_scene(KRT=a["cam"]["KRT"], extrin=a["sp_data"]["extrin"], kpt3d=a["sp_data"]["kpt3d"].reshape(-1, 3),
                    bounds=a["bounds"], feat64=a["feat_geo"][0], feat8=a["feat_geo"][1], feat_tex=a["feat_tex"], img=a["img"],
                    fg=a["fg"], width=scene["width"], height=scene["height"], znear=scene["znear"], zfar=scene["zfar"],
                    nml_scale=scene["nml_scale"])
        m.render(K=a["cam_tar"]["K"], RT=a["cam_tar"]["RT"], znear=target["znear"], zfar=target["zfar"], x0=0, y0=0, step=1,
                 nx=size, ny=size, S_c=cfg["S_c"], S_f=cfg["S_f"], fine=cfg["fine"], engine=0, ert_eps=cfg["ert"],
                 out_device="cuda")

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            with record_function("l2_flush"):   # L2 flush between frames, as bench.py does; left out of the sums below
                flush.zero_()
            step()
        torch.cuda.synchronize()
    CPU, CUDA = torch.autograd.DeviceType.CPU, torch.autograd.DeviceType.CUDA
    # device time of the kernels the flush launched, by name: the kernels linked to the CPU ops inside its range
    flush_us = {}

    def walk(ev):
        for k in ev.kernels:
            flush_us[k.name] = flush_us.get(k.name, 0.0) + k.duration
        for c in ev.cpu_children:
            walk(c)

    for ev in prof.events():
        if ev.name == "l2_flush" and ev.device_type == CPU:
            walk(ev)
    us = {}
    for ev in prof.events():
        if ev.device_type == CUDA and ev.name != "l2_flush":   # device activity, without the flush's annotation range
            us[ev.name] = us.get(ev.name, 0.0) + (ev.time_range.end - ev.time_range.start)
    ms = {g: 0.0 for g in GROUPS + ("other",)}
    for name, t in us.items():
        ms[group_of(name)] += (t - flush_us.get(name, 0.0)) / 1e3 / args.steps
    geo = ms["geo_front_kernel"] + ms["geo_tail_kernel"]
    st = m.stats()
    line = {"card": card(), "config": args.config, "scene": args.scene, "n_kpt": args.n_kpt, "steps": args.steps,
            "samples_valid": int(st["samples_valid"]), "samples_coloured": int(st["samples_coloured"]),
            "ms_per_frame": {k: round(v, 3) for k, v in ms.items()},
            "flush_ms_excluded": round(sum(flush_us.values()) / 1e3 / args.steps, 3),
            "geometry_ms": round(geo, 3), "front_share_of_geometry": round(ms["geo_front_kernel"] / geo, 3) if geo else None,
            "tail_vs_datasheet": tail_floors(int(st["samples_valid"]), int(st["samples_coloured"]), ms["geo_tail_kernel"]),
            "colour_vs_datasheet": colour_floors(int(st["samples_coloured"]), 3, ms["colour_list"], ms["shade_color_kernel"])}
    m.check_health()
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    main()
