"""numpy restatement of the marching-cubes kernels (csrc/kpn_mesh.cu) and mesh checks shared by the mesh tests.

Grid point (i, j, k) of an (nz, ny, nx) field sits at p[a] = origin[a] + spacing[a] * idx_a, rounded in fp32 with no fused
multiply-add.  Vertices come in the kernels' order: by (linear index of the edge's lower corner, axis x < y < z); faces by cell
linear index, then table order (tools/gen_mc_table.py)."""
from __future__ import annotations

import importlib.util
import os

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def mc_table_module():
    spec = importlib.util.spec_from_file_location("gen_mc_table", os.path.join(_ROOT, "tools", "gen_mc_table.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def grid_axis(origin, spacing, n):
    """fp32 coordinates of n grid points along one axis: origin + spacing * idx, both roundings explicit."""
    idx = np.arange(n, dtype=np.float32)
    return (np.float32(origin) + (np.float32(spacing) * idx).astype(np.float32)).astype(np.float32)


def grid_points(origin, spacing, dims):
    """(nz, ny, nx, 3) fp32 points of the grid, x fastest."""
    nx, ny, nz = dims
    xs, ys, zs = (grid_axis(origin[a], spacing[a], n) for a, n in enumerate((nx, ny, nz)))
    Z, Y, X = np.meshgrid(zs, ys, xs, indexing="ij")
    return np.stack([X, Y, Z], axis=-1)


def _inside(f, level):
    return np.greater(f, np.float32(level))   # NaN compares false: outside


def marching_cubes(field, origin, spacing, level):
    """Returns (vertices (V,3) fp32, faces (F,3) int64) in the kernels' order."""
    f = np.asarray(field, dtype=np.float32)
    nz, ny, nx = f.shape
    lv = np.float32(level)
    P = grid_points(origin, spacing, (nx, ny, nz))
    ins = _inside(f, lv)
    # crossings owned by each point along x, y, z
    cross = np.zeros((nz, ny, nx, 3), dtype=bool)
    cross[:, :, :-1, 0] = ins[:, :, :-1] != ins[:, :, 1:]
    cross[:, :-1, :, 1] = ins[:, :-1, :] != ins[:, 1:, :]
    cross[:-1, :, :, 2] = ins[:-1, :, :] != ins[1:, :, :]
    flat = cross.reshape(-1, 3)
    cnt = flat.sum(1)
    vofs = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    pid, ax = np.nonzero(flat)                      # row-major: (point, axis) order
    k, j, i = np.unravel_index(pid, (nz, ny, nx))
    kb, jb, ib = k + (ax == 2), j + (ax == 1), i + (ax == 0)
    fa, fb = f[k, j, i], f[kb, jb, ib]
    with np.errstate(invalid="ignore", divide="ignore"):
        t = ((lv - fa).astype(np.float32) / (fb - fa).astype(np.float32)).astype(np.float32)
    t = np.where(np.isfinite(t), t, np.float32(0.5)).astype(np.float32)
    pa, pb = P[k, j, i], P[kb, jb, ib]
    verts = pa.copy()
    sel = np.arange(len(ax))
    d = (pb[sel, ax] - pa[sel, ax]).astype(np.float32)
    verts[sel, ax] = (pa[sel, ax] + (t * d).astype(np.float32)).astype(np.float32)
    # faces
    tab = mc_table_module().table()
    if nx < 2 or ny < 2 or nz < 2:
        return verts, np.zeros((0, 3), dtype=np.int64)
    case = np.zeros((nz - 1, ny - 1, nx - 1), dtype=np.int64)
    for c in range(8):
        dx, dy, dz = c & 1, (c >> 1) & 1, (c >> 2) & 1
        case |= ins[dz:nz - 1 + dz, dy:ny - 1 + dy, dx:nx - 1 + dx].astype(np.int64) << c
    rank = np.cumsum(cross, axis=-1) - cross        # rank of an owned crossing among the point's crossings
    faces = []
    edges = []
    for e in range(12):
        ax_e, r = divmod(e, 4)
        o = [(1, 2), (0, 2), (0, 1)][ax_e]
        off = [0, 0, 0]
        off[o[0]], off[o[1]] = r & 1, (r >> 1) & 1
        edges.append((ax_e, off))
    for cid, cs in enumerate(case.reshape(-1)):
        if not tab[cs]:
            continue
        ck, cj, ci = np.unravel_index(cid, case.shape)
        for tri in tab[cs]:
            ids = []
            for e in tri:
                ax_e, off = edges[e]
                pi, pj, pk = ci + off[0], cj + off[1], ck + off[2]
                p = (pk * ny + pj) * nx + pi
                ids.append(int(vofs[p] + rank[pk, pj, pi, ax_e]))
            faces.append(ids)
    return verts, np.asarray(faces, dtype=np.int64).reshape(-1, 3)


def edge_counts(faces):
    """(directed edge -> count, undirected edge -> count)."""
    d = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    ud = np.sort(d, axis=1)
    dirc = np.unique(d, axis=0, return_counts=True)
    undc = np.unique(ud, axis=0, return_counts=True)
    return dirc, undc


def is_closed_manifold(faces):
    (_, dc), (_, uc) = edge_counts(faces)
    return bool(np.all(uc == 2) and np.all(dc == 1))


def euler(verts, faces):
    (_, _), (ue, _) = edge_counts(faces)
    used = np.unique(faces)
    return len(used) - len(ue) + len(faces)


def signed_volume(verts, faces):
    v = verts.astype(np.float64)
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    return float(np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0)
