"""Generates keypointnerf_b200/csrc/kpn_mc_table.cuh, the 256-case triangle table of the marching-cubes kernels.

Conventions (the same in the kernels and in tests/mesh_ref.py):
  corner c = dx + 2 dy + 4 dz of a cell; bit c of the case byte is set when that corner is inside (f > level);
  edge e: axis e // 4 (x, y, z); for x edges (e % 4) = dy + 2 dz, for y edges dx + 2 dz, for z edges dx + 2 dy.
  An edge's vertex belongs to its lower corner.

Every cube face is cut the same way in both cells that share it: a face with two crossing edges gets one segment; a face with
four (its two inside corners on a diagonal) gets two segments, each cutting off one inside corner.  The segments are oriented
so that the inside corners lie on their right when the face is seen from outside the cell, which makes them closed cycles;
each cycle is triangulated with diagonals whose two vertices share no cube face, so that no triangle edge other than a face
segment can be seen from a neighbouring cell.  Triangles are counter-clockwise seen from the side where f <= level.

    python tools/gen_mc_table.py            # rewrite the header
    python tools/gen_mc_table.py --check    # exit 1 if the header differs
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "keypointnerf_b200", "csrc", "kpn_mc_table.cuh")


def corner_pos(c):
    return np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1], dtype=np.float64)


def edge_corners(e):
    """(lower corner, upper corner) of edge e."""
    ax, r = divmod(e, 4)
    o = [(1, 2), (0, 2), (0, 1)][ax]   # the two other axes, low bit first
    lo = [0, 0, 0]
    lo[o[0]], lo[o[1]] = r & 1, (r >> 1) & 1
    hi = list(lo)
    hi[ax] = 1
    return lo[0] + 2 * lo[1] + 4 * lo[2], hi[0] + 2 * hi[1] + 4 * hi[2]


EDGES = [edge_corners(e) for e in range(12)]
EDGE_ID = {frozenset(p): e for e, p in enumerate(EDGES)}
# faces: (axis, side); corners in cyclic order, outward normal
FACES = []
for ax in range(3):
    for side in range(2):
        cs = [c for c in range(8) if ((c >> ax) & 1) == side]
        ring = [min(cs)]
        while len(ring) < 4:   # walk along cube edges inside the face
            nxt = [c for c in cs if c not in ring and frozenset((ring[-1], c)) in EDGE_ID]
            ring.append(nxt[0])
        n = np.zeros(3)
        n[ax] = 1.0 if side else -1.0
        FACES.append((ring, n))
EDGE_FACES = [{fi for fi, (ring, _) in enumerate(FACES) if set(EDGES[e]) <= set(ring)} for e in range(12)]


def edge_mid(e):
    a, b = EDGES[e]
    return 0.5 * (corner_pos(a) + corner_pos(b))


def face_segments(case, ring, n):
    ins = [(case >> c) & 1 for c in ring]
    cross = [EDGE_ID[frozenset((ring[i], ring[(i + 1) % 4]))] for i in range(4) if ins[i] != ins[(i + 1) % 4]]
    segs = []
    if len(cross) == 2:
        segs.append((cross[0], cross[1], next(ring[i] for i in range(4) if ins[i])))
    elif len(cross) == 4:
        for i in range(4):
            if ins[i]:
                c = ring[i]
                e1 = EDGE_ID[frozenset((c, ring[(i + 1) % 4]))]
                e2 = EDGE_ID[frozenset((c, ring[(i - 1) % 4]))]
                segs.append((e1, e2, c))
    out = []
    for p, q, c in segs:   # orient: the inside corner on the right seen from outside
        P, Q, Cc = edge_mid(p), edge_mid(q), corner_pos(c)
        if np.dot(np.cross(Q - P, Cc - P), n) > 0:
            p, q = q, p
        out.append((p, q))
    return out


def share_face(a, b):
    return bool(EDGE_FACES[a] & EDGE_FACES[b])


def triangulate(cyc):
    """Triangulation of a cycle of edge ids by ear clipping, with every diagonal joining two edges that share no cube face (the
    first one found in a fixed search order); triangles keep the cycle's orientation."""
    def rec(poly):
        if len(poly) == 3:
            return [tuple(poly)]
        k = len(poly)
        # clip an ear (poly[i-1], poly[i], poly[i+1]) whose closing diagonal is allowed
        for i in range(k):
            a, b, c = poly[i - 1], poly[i], poly[(i + 1) % k]
            if share_face(a, c) and k > 3:
                continue
            rest = poly[:i] + poly[i + 1:]
            sub = rec(rest)
            if sub is not None:
                return [(a, b, c)] + sub
        return None

    tris = rec(list(cyc))
    if tris is None:
        raise RuntimeError(f"no admissible triangulation of cycle {cyc}")
    return tris


def case_triangles(case):
    nxt = {}
    for ring, n in FACES:
        for p, q in face_segments(case, ring, n):
            assert p not in nxt
            nxt[p] = q
    tris, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        cyc, e = [], start
        while e not in seen:
            seen.add(e)
            cyc.append(e)
            e = nxt[e]
        assert e == start
        tris += triangulate(cyc)
    return tris


def table():
    return [case_triangles(c) for c in range(256)]


def render(tab):
    width = max(len(t) for t in tab)
    lines = ["// Generated by tools/gen_mc_table.py: do not edit.  Conventions (corners, edges, orientation) are in that script.",
             "#pragma once", "", "namespace kpn {", "",
             f"constexpr int MC_MAX_TRIS = {width};",
             "// number of triangles of each case",
             "__constant__ unsigned char c_mc_ntri[256] = {"]
    cnt = [len(t) for t in tab]
    for i in range(0, 256, 32):
        lines.append("    " + ", ".join(str(x) for x in cnt[i:i + 32]) + ",")
    lines.append("};")
    lines.append("// the cell edges of each triangle, three per triangle (unused entries 0)")
    lines.append(f"__constant__ unsigned char c_mc_tri[256][{3 * width}] = {{")
    for c, t in enumerate(tab):
        flat = [e for tri in t for e in tri] + [0] * (3 * (width - len(t)))
        lines.append("    {" + ", ".join(str(x) for x in flat) + "},")
    lines += ["};", "", "}  // namespace kpn", ""]
    return "\n".join(lines)


def main():
    text = render(table())
    if "--check" in sys.argv:
        ok = os.path.exists(HEADER) and open(HEADER).read() == text
        print("up to date" if ok else f"{HEADER} differs from the generator")
        sys.exit(0 if ok else 1)
    with open(HEADER, "w") as f:
        f.write(text)
    print(f"wrote {HEADER}")


if __name__ == "__main__":
    main()
