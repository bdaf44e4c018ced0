"""Marching-cubes case table, generated from a stated rule (pure Python, no dependencies).

Cube geometry.  Corner i sits at offset (x, y, z) = (i & 1, (i >> 1) & 1, (i >> 2) & 1) from the cell's origin; bit i of
the case index is set when corner i is inside (sdf <= thresh).  Edge e runs along axis a = e >> 2 (0 = x, 1 = y, 2 = z)
from corner EDGE_CORNER[e] (bit a clear) to EDGE_CORNER[e] | (1 << a); the other two axes' bits of that corner, in
ascending axis order, are the bits of e & 3.

Rule.
  1. On each of the six faces, join the face's crossing edges into segments: with two crossings, the one segment between
     them; with four (the inside corners on a diagonal), one segment per inside corner, across that corner.  This choice
     depends only on the face's four signs, so the two cells that share a face cut it the same way and the mesh has no
     cracks.
  2. Orient each segment so that the loops run counter-clockwise seen from the outside side (sdf > thresh): the segment's
     direction is u x n, with n the face's outward normal and u the in-face direction from its inside side to its outside
     side.  A face shared by two cells gets opposite directions in the two, so the mesh is an oriented 2-manifold away from
     the lattice's border.
  3. Chain the segments into loops through their shared crossing edges (each crossing edge lies on two faces, so it ends
     one segment and starts another).  Loops are taken in the order of their lowest edge.  Each loop is fan-triangulated,
     (e0, e_i, e_i+1) for i = 1 .. k - 2, from its lowest edge e0 that shares no cube face with a loop edge other than its
     two neighbours in the loop.  Without that condition a fan diagonal can join two crossing edges of an ambiguous face;
     the cell on the face's other side can draw the same diagonal, and that mesh edge then has four faces.  With it every
     diagonal runs through the cell's interior and belongs to that cell alone.  Every loop of the 256 cases has such an
     edge (the generator asserts it); for all but 18 loops it is the loop's lowest edge.

``python -m selfocc_b200.mc_table`` prints the header checked in as csrc/mc_table.cuh.
"""

AXES = 3


def _edge_corner(e):
    a, k = e >> 2, e & 3
    others = [b for b in range(AXES) if b != a]
    return ((k & 1) << others[0]) | ((k >> 1) << others[1])


EDGE_CORNER = tuple(_edge_corner(e) for e in range(12))


def _corner_pos(c):
    return (c & 1, (c >> 1) & 1, (c >> 2) & 1)


def _edge_of(c0, c1):
    a = (c0 ^ c1).bit_length() - 1
    lo = min(c0, c1)
    return next(e for e in range(12) if e >> 2 == a and EDGE_CORNER[e] == lo)


def _faces():
    """(corners in cyclic order, outward normal) of the six cube faces."""
    out = []
    for a in range(AXES):
        b, c = [x for x in range(AXES) if x != a]
        for side in (0, 1):
            base = side << a
            ring = [base, base | (1 << b), base | (1 << b) | (1 << c), base | (1 << c)]
            n = [0, 0, 0]
            n[a] = 1 if side else -1
            out.append((ring, tuple(n)))
    return out


def _sub(p, q):
    return tuple(x - y for x, y in zip(p, q))


def _cross(p, q):
    return (p[1] * q[2] - p[2] * q[1], p[2] * q[0] - p[0] * q[2], p[0] * q[1] - p[1] * q[0])


def _dot(p, q):
    return sum(x * y for x, y in zip(p, q))


def _mid(e):
    c0 = _corner_pos(EDGE_CORNER[e])
    c1 = _corner_pos(EDGE_CORNER[e] | (1 << (e >> 2)))
    return tuple((x + y) / 2 for x, y in zip(c0, c1))


def _mean(ps):
    return tuple(sum(p[i] for p in ps) / len(ps) for i in range(3))


def _oriented(e0, e1, u, n):
    """(e0, e1) or (e1, e0): the direction of the segment that follows u x n."""
    return (e0, e1) if _dot(_sub(_mid(e1), _mid(e0)), _cross(u, n)) > 0 else (e1, e0)


def case_segments(case):
    """Directed segments (edge, edge) of one case, face by face."""
    inside = lambda c: (case >> c) & 1
    segs = []
    for ring, n in _faces():
        ins = [c for c in ring if inside(c)]
        if len(ins) in (0, 4):
            continue
        crossing = [_edge_of(ring[i], ring[(i + 1) % 4]) for i in range(4) if inside(ring[i]) != inside(ring[(i + 1) % 4])]
        if len(crossing) == 2:
            outs = [c for c in ring if not inside(c)]
            u = _sub(_mean([_corner_pos(c) for c in outs]), _mean([_corner_pos(c) for c in ins]))
            segs.append(_oriented(crossing[0], crossing[1], u, n))
        else:                                   # ambiguous face: cut off each inside corner
            for c in ins:
                i = ring.index(c)
                e0, e1 = _edge_of(ring[i - 1], c), _edge_of(c, ring[(i + 1) % 4])
                u = _sub(_mean([_mid(e0), _mid(e1)]), _corner_pos(c))
                segs.append(_oriented(e0, e1, u, n))
    return segs


def _faces_of(e):
    """The cube faces (axis, side) edge e lies on."""
    c0 = EDGE_CORNER[e]
    return {(a, (c0 >> a) & 1) for a in range(AXES) if a != e >> 2}


def _fan_apex(loop):
    """Index of the loop's lowest edge that shares no cube face with a loop edge other than its two neighbours."""
    k = len(loop)
    ok = [i for i in range(k)
          if all(not (_faces_of(loop[i]) & _faces_of(e)) for j, e in enumerate(loop) if (j - i) % k not in (0, 1, k - 1))]
    assert ok, loop
    return min(ok, key=lambda i: loop[i])


def case_loops(case):
    """The case's loops of crossing edges in the order of their lowest edge, each starting at its fan apex."""
    nxt = {}
    for a, b in case_segments(case):
        assert a not in nxt, (case, a)
        nxt[a] = b
    assert sorted(nxt) == sorted(nxt.values()), case          # every crossing edge starts one segment and ends one
    loops, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = nxt[e]
        assert e == start, case
        i = _fan_apex(loop)
        loops.append(loop[i:] + loop[:i])
    return loops


def case_triangles(case):
    tris = []
    for loop in case_loops(case):
        tris += [(loop[0], loop[i], loop[i + 1]) for i in range(1, len(loop) - 1)]
    return tris


def edge_mask(case):
    """Bit e set when edge e crosses: its two corners are on different sides."""
    return sum(1 << e for e in range(12) if ((case >> EDGE_CORNER[e]) ^ (case >> (EDGE_CORNER[e] | (1 << (e >> 2))))) & 1)


def tables():
    """(edge masks [256], triangle lists [256] of edge triples, maximum triangle count)."""
    tris = [case_triangles(c) for c in range(256)]
    return [edge_mask(c) for c in range(256)], tris, max(len(t) for t in tris)


def header():
    masks, tris, max_tri = tables()
    lines = ['// Generated by selfocc_b200/mc_table.py (python -m selfocc_b200.mc_table); do not edit.',
             '// Marching-cubes case table: corner i at offset (i & 1, (i >> 1) & 1, (i >> 2) & 1), bit i of the case set when',
             '// corner i is inside (sdf <= thresh); edge e along axis e >> 2 from corner kMcEdgeCorner[e].  kMcTri[case] lists',
             '// kMcNumTri[case] triangles as edge triples, counter-clockwise seen from the outside (sdf > thresh), padded with -1.',
             '// Global memory, not __constant__: neighbouring threads look up different cases, which the constant cache serialises.',
             '#pragma once',
             '#include <stdint.h>',
             '',
             'namespace so {',
             '',
             'constexpr int kMcMaxTri = %d;' % max_tri,
             '',
             '__device__ uint8_t kMcEdgeCorner[12] = {%s};' % ', '.join(str(c) for c in EDGE_CORNER),
             '',
             '__device__ uint16_t kMcEdgeMask[256] = {']
    for r in range(0, 256, 8):
        lines.append('    ' + ', '.join('0x%03x' % m for m in masks[r:r + 8]) + ',')
    lines += ['};', '', '__device__ uint8_t kMcNumTri[256] = {']
    for r in range(0, 256, 16):
        lines.append('    ' + ', '.join(str(len(t)) for t in tris[r:r + 16]) + ',')
    lines += ['};', '', '__device__ int8_t kMcTri[256][3 * kMcMaxTri] = {']
    for c in range(256):
        flat = [e for t in tris[c] for e in t] + [-1] * (3 * (max_tri - len(tris[c])))
        lines.append('    {%s},  // %d' % (', '.join(str(e) for e in flat), c))
    lines += ['};', '', '}  // namespace so', '']
    return '\n'.join(lines)


if __name__ == '__main__':
    print(header(), end='')
