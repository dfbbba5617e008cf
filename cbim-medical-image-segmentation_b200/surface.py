"""Surfel-area table of the 3D surface-distance metric (metric/lookup_tables.py:591-639,
create_table_neighbour_code_to_surface_area), derived here from a marching-cubes triangulation of the 2x2x2 cell.

A neighbour code describes the 8 voxels p-1 .. p of a 2x2x2 cell; corner (a, b, c) (a along axis 0) carries the bit
weight 2**(7 - (4a + 2b + c)), so 128 is offset (-1,-1,-1) and 1 is offset (0,0,0)
(ENCODE_NEIGHBOURHOOD_3D_KERNEL, lookup_tables.py:45).  The surface of a code is the classic marching-cubes surface
with its vertices at the midpoints of the cell edges whose two corners differ:

* codes with more than four inside corners are triangulated as their complement (same surface, same area);
* on a face whose inside corners lie on a diagonal, each inside corner is cut off on its own;
* each closed polygon is triangulated as a fan.  Triangles, quads and the planar hexagon give the same area from
  any apex.  The two non-planar polygons fan from a fixed vertex, identified by how many inside neighbours the
  inside and the outside corner of its cell edge have: the pentagon of three corners on one face (an L) from the
  edge normal to that face at an end of the L, (1, 1); the hexagon of a four-corner zig-zag from (1, 2).

table[code] = sum over triangles of |(n0 s1 s2, n1 s0 s2, n2 s0 s1)|, with n the triangle's area vector in voxel
units and s the spacing: the area of the triangle after scaling the cell to the spacing."""
import functools
import itertools

import numpy as np

_CORNERS = [(a, b, c) for a in (0, 1) for b in (0, 1) for c in (0, 1)]          # index 4a + 2b + c
_EDGES = [(i, j) for i, j in itertools.combinations(range(8), 2)
          if sum(abs(x - y) for x, y in zip(_CORNERS[i], _CORNERS[j])) == 1]
_FACES = [[i for i in range(8) if _CORNERS[i][ax] == v] for ax in range(3) for v in (0, 1)]
_NEIGHBOURS = [[j for j in range(8) if (min(i, j), max(i, j)) in _EDGES] for i in range(8)]
_FAN_APEX = {5: (1, 1), 6: (1, 2)}      # polygon size -> (inside, outside) neighbour counts of the apex's corners


def _inside(code):
    return [(code >> (7 - i)) & 1 for i in range(8)]


def _polygons(inside):
    """Closed loops of cut cell edges, each a list of edges in boundary order."""
    cut = [e for e in _EDGES if inside[e[0]] != inside[e[1]]]
    link = {e: [] for e in cut}
    for face in _FACES:
        fe = [e for e in cut if e[0] in face and e[1] in face]
        if len(fe) == 2:
            pairs = [fe]
        else:                           # 0 or 4: with 4 the inside corners are diagonal; cut each one off
            pairs = [[e for e in fe if k in e] for k in face if inside[k]] if fe else []
        for a, b in pairs:
            link[a].append(b)
            link[b].append(a)
    loops, seen = [], set()
    for start in cut:
        if start in seen:
            continue
        loop, prev, cur = [start], None, start
        seen.add(start)
        while True:
            nxt = link[cur][0] if link[cur][0] != prev else link[cur][1]
            if nxt == start:
                break
            loop.append(nxt)
            seen.add(nxt)
            prev, cur = cur, nxt
        loops.append(loop)
    return loops


def _apex(loop, inside):
    want = _FAN_APEX.get(len(loop))
    if want is None:
        return 0
    corners = {i if inside[i] else j for i, j in loop}               # the loop's own inside corners
    for k, (i, j) in enumerate(loop):
        cin, cout = (i, j) if inside[i] else (j, i)
        if (sum(n in corners for n in _NEIGHBOURS[cin]), sum(n in corners for n in _NEIGHBOURS[cout])) == want:
            return k
    return 0                            # planar hexagon (a corner and its three neighbours): every apex is equal


@functools.lru_cache(maxsize=None)
def _triangle_normals():
    """[256] lists of area vectors (voxel units) of each code's triangles."""
    out = [[] for _ in range(256)]
    mid = lambda e: np.array([(_CORNERS[e[0]][k] + _CORNERS[e[1]][k]) / 2.0 for k in range(3)])
    for code in range(1, 255):
        inside = _inside(code)
        if sum(inside) > 4:
            inside = [1 - x for x in inside]
        for loop in _polygons(inside):
            k = _apex(loop, inside)
            loop = loop[k:] + loop[:k]
            p0 = mid(loop[0])
            for i in range(1, len(loop) - 1):
                out[code].append(0.5 * np.cross(mid(loop[i]) - p0, mid(loop[i + 1]) - p0))
    return out


@functools.lru_cache(maxsize=64)
def _table(spacing):
    s0, s1, s2 = spacing
    t = np.zeros(256)
    for code, normals in enumerate(_triangle_normals()):
        area = 0.0
        for n in normals:
            area += np.linalg.norm(np.array([n[0] * s1 * s2, n[1] * s0 * s2, n[2] * s0 * s1]))
        t[code] = area
    return t


def surface_area_table(spacing):
    """float64 [256]: surfel area of every neighbour code at voxel spacing (s0, s1, s2); cached per spacing."""
    s = tuple(float(x) for x in spacing)
    if len(s) != 3:
        raise ValueError("spacing must have 3 entries, got %d" % len(s))
    return _table(s).copy()
