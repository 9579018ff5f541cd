"""Generates nerfshop_b200/csrc/nsb_mc_table.h, the marching-cubes case table, from the cube's geometry.

  python tools/gen_mc_table.py           writes the header
  python tools/gen_mc_table.py --check   exits 1 if the committed header differs from what this script generates

Corner and edge numbering are the reference's (marching_cubes.cu:198-213): corners 0-3 are (0,0,0) (1,0,0) (1,1,0) (0,1,0),
corners 4-7 the same at z = 1; edges 0-3 run 0-1, 1-2, 3-2, 0-3, edges 4-7 the same at z = 1, edges 8-11 go +z from corners 0-3.
Bit i of a configuration is set when corner i is inside (density > threshold).

For each configuration:
  1. On every face, walk the corners counter-clockwise as seen from outside the cube. Each maximal run of inside corners
     gives one segment, from the crossing where the walk leaves the run back to the crossing where it entered it. A face with four
     crossings (inside corners diagonal) therefore always separates its two inside corners. The rule reads only the face's four
     signs, so the two cells sharing a face build the same segments, in opposite directions: closed surfaces are watertight.
  2. Every crossing edge lies on two faces, where it ends one segment and starts the next: the segments chain into cycles.
  3. Each cycle is triangulated without a diagonal between two crossings on one face (see _triangulate), so no edge is built by two cells
     unless it is a face segment they share.
Triangle winding is the reference's: configuration 1 (corner 0 inside) gives the triangle (0, 8, 3), whose normal by the
right-hand rule points from the inside corner to the outside.
"""
from __future__ import annotations

import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "..", "nerfshop_b200", "csrc", "nsb_mc_table.h")

CORNERS = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]
EDGES = [(0, 1), (1, 2), (3, 2), (0, 3), (4, 5), (5, 6), (7, 6), (4, 7), (0, 4), (1, 5), (2, 6), (3, 7)]
# the six faces as (axis, side); corners ordered counter-clockwise seen from outside below
FACES = [(0, 0), (0, 1), (1, 0), (1, 1), (2, 0), (2, 1)]


def _edge(a: int, b: int) -> int:
    return EDGES.index((a, b)) if (a, b) in EDGES else EDGES.index((b, a))


def _face_loop(axis: int, side: int):
    """The face's four corners, counter-clockwise about its outward normal."""
    cs = [i for i, c in enumerate(CORNERS) if c[axis] == side]
    u, v = [a for a in range(3) if a != axis]
    order = sorted(cs, key=lambda i: {(0, 0): 0, (1, 0): 1, (1, 1): 2, (0, 1): 3}[(CORNERS[i][u], CORNERS[i][v])])
    p = [CORNERS[i] for i in order[:3]]
    a = [p[1][k] - p[0][k] for k in range(3)]
    b = [p[2][k] - p[1][k] for k in range(3)]
    normal_along_axis = a[(axis + 1) % 3] * b[(axis + 2) % 3] - a[(axis + 2) % 3] * b[(axis + 1) % 3]
    if (normal_along_axis > 0) != (side == 1):  # outward is +axis on side 1, -axis on side 0
        order = order[::-1]
    return order


def face_segments(cfg: int):
    """Directed segments (from_edge, to_edge) on all six faces of configuration cfg."""
    segs = []
    for axis, side in FACES:
        loop = _face_loop(axis, side)
        ins = [(cfg >> c) & 1 for c in loop]
        if all(ins) or not any(ins):
            continue
        # start the walk just after an outside corner so every inside run is contiguous
        k0 = next(k for k in range(4) if not ins[k])
        enter = None
        for s in range(1, 5):
            k, prev = (k0 + s) % 4, (k0 + s - 1) % 4
            if ins[k] and not ins[prev]:
                enter = _edge(loop[prev], loop[k])
            elif not ins[k] and ins[prev]:
                segs.append((_edge(loop[prev], loop[k]), enter))
    return segs


def cycles(cfg: int):
    nxt = {}
    for a, b in face_segments(cfg):
        assert a not in nxt, (cfg, a)
        nxt[a] = b
    out, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        cyc, e = [], start
        while e not in seen:
            seen.add(e)
            cyc.append(e)
            e = nxt[e]
        assert e == start, (cfg, cyc)
        out.append(cyc)
    return out


def _faces_of_edge(e: int):
    a, b = EDGES[e]
    return {f for f, (axis, side) in enumerate(FACES) if CORNERS[a][axis] == side and CORNERS[b][axis] == side}


def _triangulate(poly):
    """A triangulation of the cycle whose diagonals never join two crossings on one cube face: such a diagonal could also be
    built by the cell across that face, and the edge would then have more than two triangles. The first one found, searching
    triangles on (poly[0], poly[1]) by apex in cycle order, recursively."""
    if len(poly) == 3:
        return [tuple(poly)]
    for k in range(2, len(poly)):
        parts = []
        ok = True
        for sub, outer in ((poly[1:k + 1], k > 2), (poly[k:] + poly[:1], k < len(poly) - 1)):
            if not outer:
                continue
            if _faces_of_edge(sub[0]) & _faces_of_edge(sub[-1]):
                ok = False
                break
            t = _triangulate(sub)
            if t is None:
                ok = False
                break
            parts.append(t)
        if ok:
            return [(poly[0], poly[1], poly[k])] + [t for p in parts for t in p]
    return None


def triangles(cfg: int):
    tris = []
    for cyc in cycles(cfg):
        t = _triangulate(cyc)
        assert t is not None, (cfg, cyc)
        tris += t
    return tris


def four_crossing_configs():
    """Configurations with at least one face whose inside corners are diagonal (the faces the separation rule decides)."""
    out = []
    for cfg in range(256):
        for axis, side in FACES:
            ins = [(cfg >> c) & 1 for c in _face_loop(axis, side)]
            if ins in ([1, 0, 1, 0], [0, 1, 0, 1]):
                out.append(cfg)
                break
    return out


def table():
    return [triangles(cfg) for cfg in range(256)]


def render() -> str:
    t = table()
    max_tris = max(len(x) for x in t)
    width = 3 * max_tris + 1
    lines = [
        "/* nsb_mc_table.h — marching-cubes case table. GENERATED by tools/gen_mc_table.py; do not edit.",
        " * Corner / edge numbering of the reference's marching_cubes.cu:198-213. Row c lists the triangles of configuration c",
        " * (bit i = corner i inside) as edge triples, -1 terminated; NSB_MC_TRI_COUNT[c] is their number.",
        " * Faces with two crossings give the only possible segment; a face with four separates its two inside corners. */",
        "#ifndef NSB_MC_TABLE_H",
        "#define NSB_MC_TABLE_H",
        "",
        f"#define NSB_MC_MAX_TRIS {max_tris}",
        f"#define NSB_MC_ROW {width}",
        "",
        "#define NSB_MC_TRI_COUNT_INIT { \\",
    ]
    counts = [len(x) for x in t]
    for r in range(0, 256, 32):
        lines.append("\t" + ", ".join(str(c) for c in counts[r:r + 32]) + ", \\")
    lines.append("}")
    lines.append("")
    lines.append("#define NSB_MC_TRI_TABLE_INIT { \\")
    for cfg, tris in enumerate(t):
        flat = [e for tri in tris for e in tri]
        flat += [-1] * (width - len(flat))
        lines.append("\t{" + ", ".join(str(e) for e in flat) + "}, \\")
    lines.append("}")
    lines.append("")
    lines.append("#endif /* NSB_MC_TABLE_H */")
    return "\n".join(lines) + "\n"


def main(argv):
    text = render()
    if "--check" in argv:
        with open(OUT) as fh:
            same = fh.read() == text
        print("nsb_mc_table.h is up to date" if same else "nsb_mc_table.h differs from the generator's output")
        return 0 if same else 1
    with open(OUT, "w") as fh:
        fh.write(text)
    print(OUT)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
