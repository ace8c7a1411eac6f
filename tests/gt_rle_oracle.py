"""numpy restatement of COCO.annToRLE for list segmentations (pycocotools coco.py annToRLE, _mask.pyx frPyObjects /
frBbox / frPoly / frUncompressedRLE, maskApi.c rleFrBbox / rleMerge), statement by statement, on top of the literal
rleFrPoly of tests/proposal_target_oracle.py; and the toggle formulation the kernel uses (csrc/poly.cuh, csrc/gt_rle.cu)
at an h x w canvas.  pycocotools is absent and not vendored by the reference, so parity with it is pinned to the
published algorithm, not to executed code.

Uncompressed RLEs are {'size': [h, w], 'counts': uint32 run lengths}.
"""
import math

import numpy as np

from proposal_target_oracle import rle_fr_poly
from oracle import oracle as O


# ------------------------------------------------------------------------------------------------
# maskApi.c / _mask.pyx, as written
# ------------------------------------------------------------------------------------------------
def rle_merge(R, intersect=0):
    """maskApi.c rleMerge(R, M, n, intersect) on a list of {'size', 'counts'}."""
    n = len(R)
    if n == 0:
        return {'size': [0, 0], 'counts': np.zeros(0, np.uint32)}
    h, w = R[0]['size']
    if n == 1:
        return {'size': [h, w], 'counts': np.asarray(R[0]['counts'], np.uint32).copy()}
    cnts = [int(c) for c in R[0]['counts']]
    m = len(cnts)
    for i in range(1, n):
        B = R[i]
        if list(B['size']) != [h, w]:
            h = w = m = 0
            cnts = []
            break
        A = cnts[:m]
        Bc = [int(c) for c in B['counts']]
        ca, cb = A[0], Bc[0]
        v = va = vb = 0
        m = 0
        a = b = 1
        cc = 0
        ct = 1
        out = []
        while ct > 0:
            c = min(ca, cb)
            cc += c
            ct = 0
            ca -= c
            if not ca and a < len(A):
                ca = A[a]
                a += 1
                va = not va
            ct += ca
            cb -= c
            if not cb and b < len(Bc):
                cb = Bc[b]
                b += 1
                vb = not vb
            ct += cb
            vp = v
            v = (va and vb) if intersect else (va or vb)
            if v != vp or ct == 0:
                out.append(cc)
                m += 1
                cc = 0
        cnts = out
    return {'size': [h, w], 'counts': np.asarray(cnts[:m], np.uint32)}


def rle_fr_bbox(bb, h, w):
    """maskApi.c rleFrBbox: each [x, y, bw, bh] row as the polygon [xs, ys, xs, ye, xe, ye, xe, ys] through rleFrPoly."""
    out = []
    for row in np.asarray(bb, np.float64).reshape(-1, 4):
        xs, ys = float(row[0]), float(row[1])
        xe, ye = xs + float(row[2]), ys + float(row[3])
        out.append({'size': [h, w], 'counts': np.asarray(rle_fr_poly([xs, ys, xs, ye, xe, ye, xe, ys], h, w), np.uint32)})
    return out


def fr_poly(poly, h, w):
    """_mask.pyx frPoly: rleFrPoly of every polygon, k = int(len(p) / 2)."""
    return [{'size': [h, w], 'counts': np.asarray(rle_fr_poly(np.asarray(p, np.float64), h, w), np.uint32)}
            for p in poly]


def fr_uncompressed_rle(uc, h, w):
    """_mask.pyx frUncompressedRLE: the counts as uint32, the size of the dict (not h, w)."""
    return [{'size': [int(r['size'][0]), int(r['size'][1])], 'counts': np.array(r['counts'], dtype=np.uint32)}
            for r in uc]


def fr_py_objects(pyobj, h, w):
    """_mask.pyx frPyObjects, branch by branch (the forms annToRLE reaches)."""
    if type(pyobj) == np.ndarray:
        return rle_fr_bbox(pyobj, h, w)
    elif type(pyobj) == list and len(pyobj[0]) == 4:
        bb = np.array(pyobj, dtype=np.double)               # frBbox's 2-D double buffer
        if bb.ndim != 2:
            raise ValueError("Buffer has wrong number of dimensions")
        return rle_fr_bbox(bb, h, w)
    elif type(pyobj) == list and len(pyobj[0]) > 4:
        return fr_poly(pyobj, h, w)
    elif type(pyobj) == list and type(pyobj[0]) == dict and 'counts' in pyobj[0] and 'size' in pyobj[0]:
        return fr_uncompressed_rle(pyobj, h, w)
    elif type(pyobj) == dict and 'counts' in pyobj and 'size' in pyobj:
        return fr_uncompressed_rle([pyobj], h, w)[0]
    raise Exception('input type is not supported.')


def ann_to_rle(segm, h, w):
    """COCO.annToRLE with the image record's (h, w); a compressed RLE is returned decoded to its run lengths."""
    if type(segm) == list:
        return rle_merge(fr_py_objects(segm, h, w))
    elif type(segm['counts']) == list:
        return fr_py_objects(segm, h, w)
    return {'size': [int(segm['size'][0]), int(segm['size'][1])], 'counts': O.rle_from_string(segm['counts'])}


# ------------------------------------------------------------------------------------------------
# the kernel's formulation at h x w: toggles, a prefix XOR per polygon, the union, its boundaries
# ------------------------------------------------------------------------------------------------
def _vert(c):
    """(int)(5 * c + .5) of a double."""
    return int(math.trunc(5.0 * c + .5))


def edge_toggles(X0, Y0, X1, Y1, h, w):
    """Column-major indices n * h + y toggled by one edge (csrc/poly.cuh): crossed columns 0 <= n <= w - 1, y clamped
    to h, so a point with y = h lands on row 0 of column n + 1 and h * w is off the canvas."""
    out = []
    dx, dy = abs(X1 - X0), abs(Y1 - Y0)

    def toggle(n, yv):
        yd = (float(yv) + .5) / 5.0 - .5
        yd = 0.0 if yd < 0 else (float(h) if yd > h else yd)
        out.append(n * h + int(math.ceil(yd)))

    def cols(lo, hi):
        return range(max(0, -(-(lo - 2) // 5)), min(w - 1, (hi - 3) // 5) + 1)

    if dx >= dy:
        if dx == 0:
            return out
        flip = X0 > X1
        xs, ys, ye = (X1, Y1, Y0) if flip else (X0, Y0, Y1)
        s = (ye - ys) / dx

        def v(t):
            return int(math.trunc(ys + s * t + .5))
        for n in cols(xs, xs + dx):
            ta = 5 * n + 2 - xs
            toggle(n, min(v(ta), v(ta + 1)))
    else:
        flip = Y0 > Y1
        xs, xe, ys = (X1, X0, Y1) if flip else (X0, X1, Y0)
        s = (xe - xs) / dy

        def u(t):
            return int(math.trunc(xs + s * t + .5))
        u0, u1 = u(0), u(dy)
        for n in cols(min(u0, u1), max(u0, u1)):
            xd = 5 * n + 2
            a, b = 0, dy
            while b - a > 1:
                m = (a + b) // 2
                if (u(m) >= xd + 1) if s > 0 else (u(m) <= xd):
                    b = m
                else:
                    a = m
            toggle(n, ys + b - 1)
    return out


def toggle_flat(xy, h, w):
    """One polygon -> its column-major uint8 [h * w] mask by toggles and a prefix XOR."""
    xy = np.asarray(xy, np.float64)
    k = len(xy) // 2
    X = [_vert(c) for c in xy[0:2 * k:2]]
    Y = [_vert(c) for c in xy[1:2 * k:2]]
    bits = np.zeros(h * w + 1, np.uint8)
    for j in range(k):
        for a in edge_toggles(X[j], Y[j], X[(j + 1) % k], Y[(j + 1) % k], h, w):
            bits[a] ^= 1
    return np.bitwise_xor.accumulate(bits[:h * w])


def encode_flat(flat):
    """The canonical runs of a column-major mask: boundaries differenced from 0, then h * w (zeros first)."""
    flat = np.asarray(flat, np.uint8)
    b = np.flatnonzero(np.diff(np.concatenate([[0], flat])) != 0)
    return np.diff(np.concatenate([[0], b, [flat.size]])).astype(np.uint32)


def toggle_union_rle(polys, h, w):
    """The union of the polygons as the kernel computes it -> canonical run lengths."""
    u = np.zeros(h * w, np.uint8)
    for p in polys:
        u |= toggle_flat(p, h, w)
    return encode_flat(u)


# ------------------------------------------------------------------------------------------------
# seeded polygons
# ------------------------------------------------------------------------------------------------
def random_polygon(rng, h, w, kind):
    """A flat [x0, y0, ...] polygon of one of six kinds: 0 star inside the image, 1 star crossing the border (negative
    vertices included), 2 self-intersecting star, 3 long steep and shallow edges (full width / height), 4 coordinates
    on the 5c + .5 boundary with repeated and collinear vertices, 5 a tiny polygon."""
    k = int(rng.integers(3, 24))
    if kind in (0, 1, 2):
        cx, cy = rng.uniform(0, w), rng.uniform(0, h)
        r = float(np.exp(rng.uniform(np.log(2), np.log(max(h, w) / (2 if kind == 1 else 4)))))
        a = rng.uniform(0, 2 * np.pi, k) if kind == 2 else np.sort(rng.uniform(0, 2 * np.pi, k))
        rr = r * rng.uniform(0.3, 1.0, k)
        xy = np.stack([cx + rr * np.cos(a), cy + rr * np.sin(a) * rng.uniform(0.3, 3.0)], 1)
        if kind == 1:
            xy = xy * rng.uniform(1.0, 1.6) - rng.uniform(0, 0.3) * np.array([w, h])
    elif kind == 3:
        xy = np.array([[rng.uniform(-3, 2), rng.uniform(0, h)], [w + rng.uniform(-2, 3), rng.uniform(0, h)],
                       [rng.uniform(0, w), h + rng.uniform(-2, 3)], [rng.uniform(0, w), rng.uniform(-3, 2)]])
    elif kind == 4:
        xy = np.round(rng.uniform(-2, 1.05, (k, 2)) * [w, h] * 5) / 5 + 0.1
        xy = np.repeat(xy, rng.integers(1, 3, k), axis=0)             # repeated consecutive vertices
        mid = (xy[:1] + xy[1:2]) / 2
        xy = np.concatenate([xy[:1], mid, xy[1:]])                     # a collinear point
    else:
        x, y = rng.uniform(0, w), rng.uniform(0, h)
        xy = np.array([[x, y], [x + rng.uniform(0, 1.5), y], [x, y + rng.uniform(0, 1.5)]])
    return [float(v) for v in np.asarray(xy).reshape(-1)]
