"""Times the mesh path on the bench scene (512 x 512 sources, 3 views, 18 keypoints): the geometry-only grid query
(kpn_query_grid), kpn_query on the same points (host-built pts / view arrays, what a caller of query would do), and marching
cubes (kpn_mesh_begin + kpn_mesh_emit) of the density field valid * relu(rad).  Prints the card and its power limit first
(read in the same run), then one JSON line per (mask, engine, resolution).

    python tools/bench_mesh.py [--res 128 256 512] [--engines 0 1] [--masks ones hull] [--reps 3]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from keypointnerf_b200 import synthetic as syn  # noqa: E402
from keypointnerf_b200.model import KeypointNeRF  # noqa: E402
from keypointnerf_b200.testing import build_model, scene_tensors  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # the timings below still say which device they ran on
        q = f"nvidia-smi unavailable ({e}); torch: {torch.cuda.get_device_name(0)}"
    return q


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return min(ts), sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, nargs="+", default=[128, 256, 512])
    ap.add_argument("--engines", type=int, nargs="+", default=[0, 1])
    ap.add_argument("--masks", nargs="+", default=["ones", "hull"])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-query-points", type=int, default=1 << 31, help="skip kpn_query above this many points")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_mesh needs a CUDA device")
    print(json.dumps({"card": card(), "torch_device": torch.cuda.get_device_name(0)}), flush=True)
    dev = "cuda:0"
    net = build_model(syn.make_weights(18), 18, dev)
    for mask in args.masks:
        scene = syn.make_scene(512, 3, 18, fg_mode=mask)
        a = scene_tensors(scene, syn.make_target(size=16), dev)
        m = net._bind_scene(a["cam"], a["feat_geo"], a["feat_tex"], a["sp_data"], a["img"], a["fg"], a["bounds"])
        for engine in args.engines:
            for res in args.res:
                origin, spacing, dims = KeypointNeRF.mesh_grid(a["bounds"], res)
                n = dims[0] * dims[1] * dims[2]
                row = {"mask": mask, "engine": engine, "res": res, "dims": dims, "points": n}
                box = {}

                def grid():
                    box["q"] = m.query_grid(origin, spacing, dims, engine=engine)

                grid()   # warm-up (module load, workspace growth)
                row["query_grid_ms"] = timed(grid, args.reps)
                out2, valid = box["q"]
                row["valid_fraction"] = float(valid.float().mean())
                dens = out2[..., 1].clamp_min(0) * valid
                pos = dens[dens > 0]
                level = float(pos.median()) if pos.numel() else 0.5
                field = torch.nn.functional.pad(dens, (1, 1, 1, 1, 1, 1)).contiguous()
                po = tuple(o - h for o, h in zip(origin, spacing))

                def mesh():
                    box["mesh"] = m.marching_cubes(field, po, spacing, level)

                mesh()
                row["mesh_begin_emit_ms"] = timed(mesh, args.reps)
                row["vertices"], row["faces"] = int(box["mesh"][0].shape[0]), int(box["mesh"][1].shape[0])
                del box["mesh"]
                if n <= args.max_query_points:
                    ax = [origin[i] + spacing[i] * torch.arange(dims[i], device=dev, dtype=torch.float32) for i in range(3)]
                    Z, Y, X = torch.meshgrid(ax[2], ax[1], ax[0], indexing="ij")
                    pts = torch.stack([X, Y, Z], -1).reshape(-1, 3)
                    del X, Y, Z
                    view = torch.zeros_like(pts)
                    view[:, 2] = 1.0

                    def query():
                        box["p"] = m.query(pts, view, engine=engine)

                    query()
                    row["kpn_query_ms"] = timed(query, args.reps)
                    del box["p"], pts, view
                else:
                    row["kpn_query_ms"] = "not measured"
                del box["q"], out2, valid, dens, field
                torch.cuda.empty_cache()
                print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
