"""Derive the marching-cubes triangle table from first principles and write instantavatar_b200/csrc/ia_mc_table.cuh.

Numbering (shared by the generator, the kernels in ia_mesh.cu and oracle/marching_cubes_ref.py):
  corner c in 0..7 sits at offset (c >> 2 & 1, c >> 1 & 1, c & 1) from the cube's lower lattice point (x slowest);
  the case index of a cube is sum over corners of (v_c > level) << c;
  edge e in 0..11 runs along axis e // 4 from its lower end, whose offsets on the other two axes (ascending axis order)
  are (e >> 1 & 1, e & 1).

For each case:
  1. every cube face gets its crossing segments: a face with two crossing edges joins them; a face with four (the
     ambiguous diagonal pattern) joins the two edges around each above corner, so the segments cut off the above
     corners.  The rule reads only that face's four signs, so the two cubes sharing a face agree.
  2. each segment is oriented so that, seen from outside the cube, the above corners lie on its left; the segments then
     chain into closed loops around the above region of the cube's surface (every crossing edge has one segment in, one
     out).  Loops start at their smallest unvisited edge.
  3. each loop is fan-triangulated from its first edge, where the loop starts at the first edge (in loop order from the
     traversal's start) whose fan draws no chord between two edges of one cube face.  A chord in a face could join the
     same two vertices as a triangle of the neighbouring cube, and the mesh would no longer be a closed manifold.
     A triangle's normal (right-hand rule) points towards the above side; the kernel swaps two indices when the object
     is the above set.

    python scripts/gen_mc_table.py          # rewrite the header
    python scripts/gen_mc_table.py --check  # exit 1 if the committed header differs
"""
from __future__ import annotations

import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "instantavatar_b200", "csrc", "ia_mc_table.cuh")


def corner_offset(c):
    return (c >> 2 & 1, c >> 1 & 1, c & 1)


def edge_geometry(e):
    """(axis, lower-end offset, corner index of the lower end, corner index of the upper end)"""
    axis = e // 4
    others = [a for a in range(3) if a != axis]
    off = [0, 0, 0]
    off[others[0]] = e >> 1 & 1
    off[others[1]] = e & 1
    hi = list(off)
    hi[axis] = 1
    lo_c = off[0] * 4 + off[1] * 2 + off[2]
    hi_c = hi[0] * 4 + hi[1] * 2 + hi[2]
    return axis, tuple(off), lo_c, hi_c


EDGES = [edge_geometry(e) for e in range(12)]


def face_geometry(axis, side):
    """corners and edges of the cube face at offset `side` on `axis`, and its outward normal"""
    corners = [c for c in range(8) if corner_offset(c)[axis] == side]
    edges = [e for e in range(12) if EDGES[e][0] != axis and EDGES[e][1][axis] == side]
    normal = [0, 0, 0]
    normal[axis] = 1 if side else -1
    return corners, edges, tuple(normal)


FACES = [face_geometry(a, s) for a in range(3) for s in range(2)]


def crossing_edges(case):
    return [e for e in range(12) if (case >> EDGES[e][2] & 1) != (case >> EDGES[e][3] & 1)]


def _midpoint(e):
    axis, off, _, _ = EDGES[e]
    p = [float(o) for o in off]
    p[axis] += 0.5
    return p


def _left_of(p, q, a, n):
    """sign of ((q - p) x (a - p)) . n"""
    u = [q[i] - p[i] for i in range(3)]
    w = [a[i] - p[i] for i in range(3)]
    cr = (u[1] * w[2] - u[2] * w[1], u[2] * w[0] - u[0] * w[2], u[0] * w[1] - u[1] * w[0])
    return sum(cr[i] * n[i] for i in range(3))


def face_segments(case):
    """oriented segments (edge_from, edge_to) of every face, by the face rule of the module docstring"""
    cross = set(crossing_edges(case))
    segs = []
    for corners, edges, normal in FACES:
        fe = [e for e in edges if e in cross]
        if not fe:
            continue
        above = [c for c in corners if case >> c & 1]
        if len(fe) == 2:
            pairs = [(fe[0], fe[1], above[0])]
        else:
            assert len(fe) == 4 and len(above) == 2
            pairs = []
            for c in above:
                inc = [e for e in fe if c in (EDGES[e][2], EDGES[e][3])]
                assert len(inc) == 2
                pairs.append((inc[0], inc[1], c))
        for a, b, c in pairs:
            s = _left_of(_midpoint(a), _midpoint(b), [float(o) for o in corner_offset(c)], normal)
            assert s != 0
            segs.append((a, b) if s > 0 else (b, a))
    return segs


def loops(case):
    nxt = {}
    for a, b in face_segments(case):
        assert a not in nxt, "two segments leave one edge"
        nxt[a] = b
    assert sorted(nxt) == sorted(nxt.values()) == crossing_edges(case)
    out, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = nxt[e]
        assert e == start
        out.append(loop)
    return out


def share_face(a, b):
    return any(a in fe and b in fe for _, fe, _ in FACES)


def fan_start(loop):
    """the loop rotated to its first vertex whose fan adds no chord between two edges of one cube face (such a chord
    would lie in the face, where the neighbouring cube may draw the same vertex pair)"""
    for k in range(len(loop)):
        r = loop[k:] + loop[:k]
        if not any(share_face(r[0], r[i]) for i in range(2, len(r) - 1)):
            return r
    raise AssertionError(f"no chord-free fan for loop {loop}")


def triangles(case):
    tris = []
    for loop in loops(case):
        loop = fan_start(loop)
        for i in range(1, len(loop) - 1):
            tris.append((loop[0], loop[i], loop[i + 1]))
    return tris


def generate() -> str:
    table = [triangles(c) for c in range(256)]
    max_tris = max(len(t) for t in table)
    lines = [
        "// ia_mc_table.cuh -- marching-cubes case table, GENERATED by scripts/gen_mc_table.py (do not edit).",
        "// Corner c: offset (c>>2&1, c>>1&1, c&1); case = sum (v_c > level) << c; edge e: axis e/4, lower end at",
        "// offsets (e>>1&1, e&1) on the other two axes.  Triangles (edge triples) point their normals to the above side.",
        "#pragma once",
        "",
        f"#define IA_MC_MAX_TRIS {max_tris}",
        "",
        "// number of triangles of each case",
        "static __device__ const unsigned char kMcNumTris[256] = {",
    ]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(len(t)) for t in table[r:r + 32]) + ",")
    lines += ["};", "", "// edges of each case's triangles, IA_MC_MAX_TRIS triples per case (unused slots 255)",
              "static __device__ const unsigned char kMcTriEdges[256][IA_MC_MAX_TRIS * 3] = {"]
    for c, t in enumerate(table):
        flat = [e for tri in t for e in tri] + [255] * (3 * (max_tris - len(t)))
        lines.append("    {" + ", ".join(str(e) for e in flat) + "},  // " + str(c))
    lines += ["};", ""]
    return "\n".join(lines)


def main():
    text = generate()
    if "--check" in sys.argv[1:]:
        same = os.path.exists(HEADER) and open(HEADER).read() == text
        print("ia_mc_table.cuh is " + ("up to date" if same else "STALE"))
        sys.exit(0 if same else 1)
    with open(HEADER, "w") as f:
        f.write(text)
    print(f"wrote {HEADER}: max {max(len(triangles(c)) for c in range(256))} triangles per cube")


if __name__ == "__main__":
    main()
