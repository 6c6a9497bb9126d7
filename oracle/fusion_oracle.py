"""numpy restatement of TSDF fusion and marching-tetrahedra extraction (sam6d_b200/fusion.py; the rules are documented at
sam6d_tsdf_integrate and sam6d_tsdf_mesh_count / _emit in include/sam6d_b200.h).

integrate(..., dtype=np.float32) performs the kernel's operations in its order, each rounded to float32, and is the bit-exact
target of csrc/fusion.cu; dtype=np.float64 runs the same rule in double precision (for geometric bounds).  mesh() is written
from the extraction rule: tetrahedra are enumerated from the axis permutations, and each triangle is oriented by the sign of
its tetrahedron's corner determinant rather than from a table."""
import itertools

import numpy as np


def integrate(rgb, depth_mm, mask, K4, P12, dims, bbox_min, voxel, trunc, znear, state=None, dtype=np.float32):
    """rgb (T,H,W,3) u8, depth_mm (T,H,W) (0 = missing), mask (T,H,W) u8 or None, K4 (T,4) fx, fy, cx, cy, P12 (T,12) R row-major
    then t, dims (nx, ny, nz), bbox_min (3,), voxel, trunc, znear; state: a previous result to continue from (default: tsdf 1,
    the rest 0) -> dict tsdf (nz,ny,nx) dtype, weight i32, csum (nz,ny,nx,3) u32, ccount i32"""
    f = np.dtype(dtype).type
    nx, ny, nz = dims
    T, H, W = depth_mm.shape
    if state is None:
        st = dict(tsdf=np.ones((nz, ny, nx), dtype), weight=np.zeros((nz, ny, nx), np.int32),
                  csum=np.zeros((nz, ny, nx, 3), np.uint32), ccount=np.zeros((nz, ny, nx), np.int32))
    else:
        st = {k: v.copy() for k, v in state.items()}
    s, w = st["tsdf"].reshape(-1), st["weight"].reshape(-1)
    cs, cc = st["csum"].reshape(-1, 3), st["ccount"].reshape(-1)
    b = np.asarray(bbox_min, dtype).astype(dtype)
    voxel, trunc, znear = f(voxel), f(trunc), f(znear)
    half = f(0.5)
    iz, iy, ix = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    px = (b[0] + (ix.reshape(-1).astype(dtype) + half) * voxel).astype(dtype)
    py = (b[1] + (iy.reshape(-1).astype(dtype) + half) * voxel).astype(dtype)
    pz = (b[2] + (iz.reshape(-1).astype(dtype) + half) * voxel).astype(dtype)
    K4, P12 = np.asarray(K4).astype(dtype), np.asarray(P12).astype(dtype)
    depth = np.asarray(depth_mm).astype(dtype)
    one = f(1.0)
    with np.errstate(all="ignore"):
        for k in range(T):
            R, t = P12[k, :9], P12[k, 9:]
            qz = ((R[6] * px + R[7] * py) + R[8] * pz) + t[2]
            qx = ((R[0] * px + R[1] * py) + R[2] * pz) + t[0]
            qy = ((R[3] * px + R[4] * py) + R[5] * pz) + t[1]
            fx, fy, cx, cy = K4[k]
            u = (fx * qx) / qz + cx
            v = (fy * qy) / qz + cy
            c, r = np.floor(u + half), np.floor(v + half)
            vis = (qz > znear) & (c >= 0) & (c < W) & (r >= 0) & (r < H)
            ci, ri = np.where(vis, c, 0).astype(np.int64), np.where(vis, r, 0).astype(np.int64)
            d = depth[k][ri, ci]
            obj = np.ones_like(vis) if mask is None else mask[k][ri, ci] != 0
            sdf = d - qz
            upd_obj = vis & obj & (d != 0) & ~(sdf < -trunc)
            carve = vis & ~obj & ~((d > 0) & (qz > d - trunc))
            obs = np.where(upd_obj, np.minimum(one, sdf / trunc), one).astype(dtype)
            upd = upd_obj | carve
            wf = w.astype(dtype)
            s[:] = np.where(upd, (s * wf + obs) / (w + 1).astype(dtype), s)
            w += upd
            col = upd_obj & (np.abs(sdf) < trunc)
            cs += np.where(col[:, None], rgb[k][ri, ci].astype(np.uint32), 0).astype(np.uint32)
            cc += col
    return st


PERMS = list(itertools.permutations(range(3)))       # lexicographic: the tetrahedron order


def tetrahedra():
    """the 6 Kuhn tetrahedra as paths of cube corners (bits x = 1, y = 2, z = 4): 0 -> e_a -> e_a + e_b -> 7"""
    return [[0, 1 << a, (1 << a) | (1 << b), 7] for a, b, _ in PERMS]


def _bits(c):
    return np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1])


def _parity(p):
    return sum(1 for i in range(len(p)) for j in range(i + 1, len(p)) if p[i] > p[j]) % 2


def mesh(tsdf, weight, csum, ccount, bbox_min, voxel, min_weight=1):
    """marching tetrahedra -> (vertices (V,3) f32 mm, colours (V,3) u8, faces (F,3) int64), ordered as the rule orders them"""
    nz, ny, nx = tsdf.shape
    ts, wt = tsdf.reshape(-1).astype(np.float32), weight.reshape(-1)
    cz, cy, cx = np.meshgrid(np.arange(nz - 1), np.arange(ny - 1), np.arange(nx - 1), indexing="ij")
    pts = ((cz * ny + cy) * nx + cx).reshape(-1).astype(np.int64)
    cube = np.arange(len(pts))
    off = np.array([(c & 1) + ((c >> 1) & 1) * nx + ((c >> 2) & 1) * nx * ny for c in range(8)], np.int64)
    rows = []            # (cube, tet, sub, key a, key b, key c)
    for t, path in enumerate(tetrahedra()):
        cid = pts[:, None] + off[path]
        ins = ts[cid] < 0
        good = (wt[cid] >= min_weight).all(axis=1)
        pattern = (ins * (1 << np.arange(4))).sum(axis=1)
        corner = [_bits(c) for c in path]

        def key(sel, i, j):
            a, b_ = path[min(i, j)], path[max(i, j)]
            return (pts[sel] + off[a]) * 7 + (a ^ b_) - 1

        def det(i, j, k, l):
            return np.linalg.det(np.stack([corner[j] - corner[i], corner[k] - corner[i], corner[l] - corner[i]]).astype(float))

        for pat in range(1, 15):
            sel = np.nonzero(good & (pattern == pat))[0]
            if len(sel) == 0:
                continue
            inside = [i for i in range(4) if (pat >> i) & 1]
            outside = [i for i in range(4) if not (pat >> i) & 1]
            if len(inside) in (1, 3):
                lone = inside[0] if len(inside) == 1 else outside[0]
                j, k, l = [x for x in range(4) if x != lone]
                # facing away from the lone corner when det > 0; a lone outside corner faces the other way
                away = det(lone, j, k, l) > 0
                if away != (len(inside) == 1):
                    k, l = l, k
                tri = [(key(sel, lone, j), key(sel, lone, k), key(sel, lone, l))]
            else:
                i, j = inside
                k, l = outside
                if _parity([i, j, k, l]):
                    k, l = l, k
                A, B, C, D = key(sel, i, k), key(sel, i, l), key(sel, j, l), key(sel, j, k)
                if det(i, j, k, l) < 0:
                    B, D = D, B
                tri = [(A, B, C), (A, C, D)]
            for sub, (a, b_, c) in enumerate(tri):
                rows.append(np.stack([cube[sel], np.full(len(sel), t), np.full(len(sel), sub), a, b_, c], axis=1))
    if not rows:
        return np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint8), np.zeros((0, 3), np.int64)
    rows = np.concatenate(rows)
    rows = rows[np.lexsort((rows[:, 2], rows[:, 1], rows[:, 0]))]
    keys = np.unique(rows[:, 3:].reshape(-1))
    faces = np.searchsorted(keys, rows[:, 3:]).astype(np.int64)
    p, d = keys // 7, keys % 7 + 1
    q = p + off[d]
    a, b = ts[p], ts[q]
    with np.errstate(all="ignore"):
        t = a / (a - b)
    f32 = np.float32
    bm = np.asarray(bbox_min, np.float32)
    idx = [p % nx, (p // nx) % ny, p // (nx * ny)]
    verts = np.stack([bm[ax] + ((idx[ax].astype(f32) + f32(0.5)) + np.where((d >> ax) & 1, t, f32(0))) * f32(voxel)
                      for ax in range(3)], axis=1).astype(np.float32)
    cs, cc = csum.reshape(-1, 3), ccount.reshape(-1)
    ha, hb = cc[p] > 0, cc[q] > 0
    with np.errstate(all="ignore"):
        ma = cs[p].astype(f32) / cc[p].astype(f32)[:, None]
        mb = cs[q].astype(f32) / cc[q].astype(f32)[:, None]
        both = ma + t[:, None] * (mb - ma)
    col = np.where((ha & hb)[:, None], both, np.where(ha[:, None], ma, np.where(hb[:, None], mb, f32(128))))
    cols = np.clip(np.rint(col), 0, 255).astype(np.uint8)
    return verts, cols, faces
