#!/usr/bin/env python3
"""Write relightable3dgaussian_b200/csrc/mc_table.cuh, the marching-cubes triangle table of csrc/tsdf.cu, from one
rule, so that the table is crack-free by construction rather than typed in.

  python tools/gen_mc_table.py [--check]      # --check: exit 1 if the committed header differs from the output

Conventions (shared with csrc/tsdf.cu and tests/tsdf_oracle.py):
  corner c = 0..7 sits at offset (c & 1, (c >> 1) & 1, (c >> 2) & 1) from the cell's lower corner (i, j, k);
  bit c of the cube index is set when corner c is inside (tsdf < 0);
  edge e = 0..11 joins corners (a, a | bit) along axis e // 4: x-edges 0..3 start at corners 0, 2, 4, 6, y-edges
  4..7 at 0, 1, 4, 5 and z-edges 8..11 at 0, 1, 2, 3.

The rule: on each of the cell's six faces, every maximal run of face-adjacent inside corners (walking the face's
four corners cyclically) is cut off by one segment between the two crossing edges that bound it.  Two diagonal inside
corners are two runs, so an ambiguous face always separates its inside corners.  A face's segments depend only on its
own four corners, so the two cells that share a face draw the same segments on it: no cracks.  Each crossing edge
lies on two faces, so the segments close into loops.  Each loop is fanned into triangles from a vertex whose chords
never join two edges of one face, so no chord is shared with the neighbouring cell (an edge of four triangles).  Every
segment is directed so that the loop runs counter-clockwise seen from the outside (tsdf > 0) side, so triangle
normals (right-hand rule) point from inside to outside.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "relightable3dgaussian_b200", "csrc", "mc_table.cuh")

EDGES = ([(a, a | 1) for a in (0, 2, 4, 6)] + [(a, a | 2) for a in (0, 1, 4, 5)] + [(a, a | 4) for a in (0, 1, 2, 3)])


def corner(c):
    return (c & 1, (c >> 1) & 1, (c >> 2) & 1)


def edge_of(a, b):
    return EDGES.index((min(a, b), max(a, b)))


def faces():
    """The six faces as (outward normal, four corners in cyclic order)."""
    out = []
    for d in range(3):
        u, v = (d + 1) % 3, (d + 2) % 3
        for s in (0, 1):
            cyc = []
            for (cu, cv) in ((0, 0), (1, 0), (1, 1), (0, 1)):
                cyc.append((s << d) | (cu << u) | (cv << v))
            n = [0, 0, 0]
            n[d] = 1 if s else -1
            out.append((tuple(n), cyc))
    return out


def edge_faces(e):
    """The two cube faces (axis, side) that contain edge e."""
    a, b = EDGES[e]
    return {(d, (a >> d) & 1) for d in range(3) if (a >> d) & 1 == (b >> d) & 1}


def _sub(p, q):
    return tuple(a - b for a, b in zip(p, q))


def _cross(p, q):
    return (p[1] * q[2] - p[2] * q[1], p[2] * q[0] - p[0] * q[2], p[0] * q[1] - p[1] * q[0])


def _dot(p, q):
    return sum(a * b for a, b in zip(p, q))


def _mid(e):
    a, b = EDGES[e]
    return tuple((x + y) / 2 for x, y in zip(corner(a), corner(b)))


def segments(cube):
    """Directed segments (edge from, edge to) the rule draws on the cell's faces for cube index `cube`."""
    inside = [(cube >> c) & 1 for c in range(8)]
    segs = []
    for n, cyc in faces():
        flags = [inside[c] for c in cyc]
        if all(flags) or not any(flags):
            continue
        for start in range(4):
            if not flags[start] or flags[start - 1]:
                continue                       # a run starts after an outside corner
            run = [start]
            while flags[(run[-1] + 1) % 4]:
                run.append((run[-1] + 1) % 4)
            e1 = edge_of(cyc[start - 1], cyc[start])
            e2 = edge_of(cyc[run[-1]], cyc[(run[-1] + 1) % 4])
            pts = [corner(cyc[r]) for r in run]
            cen = tuple(sum(p[i] for p in pts) / len(pts) for i in range(3))
            p1, p2 = _mid(e1), _mid(e2)
            N = _sub(tuple((a + b) / 2 for a, b in zip(p1, p2)), cen)    # inside -> outside, in the face
            if _dot(_sub(p2, p1), _cross(N, n)) < 0:
                e1, e2 = e2, e1
            segs.append((e1, e2))
    return segs


def triangles(cube):
    nxt = {}
    for e1, e2 in segments(cube):
        assert e1 not in nxt, (cube, e1)
        nxt[e1] = e2
    assert sorted(nxt) == sorted(nxt.values()), cube
    tris, left = [], set(nxt)
    while left:
        e0 = min(left)
        loop = [e0]
        while nxt[loop[-1]] != e0:
            loop.append(nxt[loop[-1]])
        left -= set(loop)
        # fan apex: the first vertex (from the lowest edge on) none of whose chords joins two edges of one cube face.
        # Such a chord could also be a chord of the neighbour that shares the face (both cells would then own an
        # edge between the same two vertices: four triangles on one edge); chords between edges with no common face
        # belong to one cell only.
        n = len(loop)
        for a in range(n):
            if all(not (edge_faces(loop[a]) & edge_faces(loop[(a + d) % n])) for d in range(2, n - 1)):
                break
        else:
            raise AssertionError(f"cube {cube}: no fan apex for loop {loop}")
        loop = loop[a:] + loop[:a]
        tris += [(loop[0], loop[i], loop[i + 1]) for i in range(1, n - 1)]
    return tris


def render():
    tabs = [triangles(c) for c in range(256)]
    mx = max(len(t) for t in tabs)
    lines = ["// Generated by tools/gen_mc_table.py from its rule (see there); do not edit.  Marching-cubes triangles per",
             "// cube index: corner c at offset (c & 1, (c >> 1) & 1, (c >> 2) & 1), bit c set when corner c is inside;",
             "// edge e joins corners kMcEdge[e] = (a, b), a < b, and lies along axis e / 4.  Every ambiguous face",
             "// separates its inside corners, so neighbouring cells agree on every shared face; triangles are wound",
             "// counter-clockwise seen from the outside (tsdf > 0).",
             "#pragma once",
             "#include <cstdint>",
             "",
             "namespace r3dg {",
             "",
             f"constexpr int kMcMaxTris = {mx};",
             "",
             "static __device__ const uint8_t kMcEdge[12][2] = {" +
             ", ".join("{%d, %d}" % e for e in EDGES) + "};",
             "",
             "// triangle count per cube index",
             "static __device__ const uint8_t kMcCount[256] = {"]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(len(t)) for t in tabs[r:r + 32]) + ",")
    lines += ["};", "",
              "// edges of each triangle; unused slots are 255",
              f"static __device__ const uint8_t kMcTris[256][{3 * mx}] = {{"]
    for c, t in enumerate(tabs):
        flat = [e for tri in t for e in tri] + [255] * (3 * (mx - len(t)))
        lines.append("    {" + ", ".join(str(e) for e in flat) + "},")
    lines += ["};", "", "}  // namespace r3dg", ""]
    return "\n".join(lines)


if __name__ == "__main__":
    text = render()
    if "--check" in sys.argv:
        sys.exit(0 if open(OUT).read() == text else 1)
    with open(OUT, "w") as f:
        f.write(text)
    print(OUT)
