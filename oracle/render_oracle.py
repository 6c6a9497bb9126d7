"""numpy restatement of the template rasteriser (sam6d_b200/csrc/render.cu): float32 operations in the kernel's order, integer
edge functions, the same (depth bits << 32 | face id) visibility key.  It specifies this renderer -- triangle id, mask, depth
and the f16 object coordinates must match the GPU bit for bit, colours within 1 -- not the reference's Cycles images.

Rules (one view):
  vertex    p = ((R0 x + R1 y) + R2 z) + t per row; u = fx p_x / p_z + cx, v = fy p_y / p_z + cy; valid iff p_z > znear and
            |u|, |v| <= 2^14; fixed point X = rint(256 u), Y = rint(256 v) (half to even)
  triangle  dropped if a vertex is invalid; area = (b-a) x (c-a) in int64, skipped if 0, b and c swapped if negative
  coverage  pixel centre P = (256 x + 128, 256 y + 128); E0 = edge(b, c), E1 = edge(c, a), E2 = edge(a, b) with
            edge(s, e) = (e.x - s.x)(P.y - s.y) - (e.y - s.y)(P.x - s.x); covered iff every E_i > 0, or E_i == 0 on a top-left
            edge (dy < 0, or dy == 0 and dx > 0)
  depth     q_i = (f32(E_i) / f32(area)) * (1 / z_i), invz = (q0 + q1) + q2, z = 1 / invz; key = bits(z) << 32 | face id,
            the smallest key wins
  resolve   w_i = q_i / invz, xyz = (w0 x0 + w1 x1) + w2 x2; albedo from vertex colours, the bilinear texture (texel centres,
            clamp to edge, v = 0 at the bottom row) or the base colour; rgb = min(255, floor(albedo (a + (1 - a) max(0, n.l))
            255 + 1/2)) with n the camera-facing face normal and l towards the light at -1.5 t"""
import numpy as np

f32 = np.float32
GUARD = f32(16384.0)
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


def vertex_pass(V, P, K, znear):
    """V (n,3) f32, P (4,4) f32 -> X, Y int64 fixed point, z f32 camera depth, ok bool"""
    V = np.asarray(V, f32)
    P = np.asarray(P, f32)
    x, y, z = V[:, 0], V[:, 1], V[:, 2]
    p = [((P[r, 0] * x + P[r, 1] * y) + P[r, 2] * z) + P[r, 3] for r in range(3)]
    fx, fy, cx, cy = f32(K[0, 0]), f32(K[1, 1]), f32(K[0, 2]), f32(K[1, 2])
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        u = (fx * p[0]) / p[2] + cx
        v = (fy * p[1]) / p[2] + cy
        ok = (p[2] > f32(znear)) & (np.abs(u) <= GUARD) & (np.abs(v) <= GUARD)
        X = np.where(ok, np.rint(np.where(ok, u, 0) * f32(256)), 0).astype(np.int64)
        Y = np.where(ok, np.rint(np.where(ok, v, 0) * f32(256)), 0).astype(np.int64)
    return X, Y, p[2].astype(f32), ok


def setup(F, X, Y, Z, ok):
    """-> per face: state (1 rasterise, 0 zero area, -1 dropped), the swapped vertex indices (F,3), ax..cy, area, 1/z_i"""
    F = np.asarray(F, np.int64)
    i0, i1, i2 = F[:, 0].copy(), F[:, 1].copy(), F[:, 2].copy()
    valid = ok[i0] & ok[i1] & ok[i2]
    area = (X[i1] - X[i0]) * (Y[i2] - Y[i0]) - (Y[i1] - Y[i0]) * (X[i2] - X[i0])
    neg = area < 0
    i1[neg], i2[neg] = F[neg, 2], F[neg, 1]
    area = np.abs(area)
    state = np.where(~valid, -1, np.where(area == 0, 0, 1))
    with np.errstate(divide="ignore"):
        iz = [f32(1) / Z[i] for i in (i0, i1, i2)]
    return dict(state=state, idx=np.stack([i0, i1, i2], 1), ax=X[i0], ay=Y[i0], bx=X[i1], by=Y[i1], cx=X[i2], cy=Y[i2], area=area,
                iza=iz[0], izb=iz[1], izc=iz[2])


def _inside(e, dx, dy):
    return (e > 0) | ((e == 0) & ((dy < 0) | ((dy == 0) & (dx > 0))))


def cover(s, f, x, y):
    """s = setup(); f, x, y equal-length arrays of face / pixel -> covered bool, q0, q1, q2, invz (float32)"""
    px, py = x.astype(np.int64) * 256 + 128, y.astype(np.int64) * 256 + 128
    ax, ay, bx, by, cx, cy = (s[k][f] for k in ("ax", "ay", "bx", "by", "cx", "cy"))
    e0 = (cx - bx) * (py - by) - (cy - by) * (px - bx)
    e1 = (ax - cx) * (py - cy) - (ay - cy) * (px - cx)
    e2 = (bx - ax) * (py - ay) - (by - ay) * (px - ax)
    cov = _inside(e0, cx - bx, cy - by) & _inside(e1, ax - cx, ay - cy) & _inside(e2, bx - ax, by - ay)
    fa = s["area"][f].astype(f32)
    with np.errstate(divide="ignore", invalid="ignore"):
        q0 = (e0.astype(f32) / fa) * s["iza"][f]
        q1 = (e1.astype(f32) / fa) * s["izb"][f]
        q2 = (e2.astype(f32) / fa) * s["izc"][f]
    return cov, q0, q1, q2, (q0 + q1) + q2


def visibility(s, H, W):
    """-> (H*W) uint64 keys of one view (EMPTY where nothing covers the pixel centre)"""
    ax, ay, bx, by, cx, cy = (s[k] for k in ("ax", "ay", "bx", "by", "cx", "cy"))
    mnx, mxx = np.minimum(ax, np.minimum(bx, cx)), np.maximum(ax, np.maximum(bx, cx))
    mny, mxy = np.minimum(ay, np.minimum(by, cy)), np.maximum(ay, np.maximum(by, cy))
    x0, x1 = np.maximum(0, -((128 - mnx) >> 8)), np.minimum(W - 1, (mxx - 128) >> 8)
    y0, y1 = np.maximum(0, -((128 - mny) >> 8)), np.minimum(H - 1, (mxy - 128) >> 8)
    live = np.flatnonzero((s["state"] == 1) & (x0 <= x1) & (y0 <= y1))
    vis = np.full(H * W, EMPTY, dtype=np.uint64)
    if len(live) == 0:
        return vis
    bw, bh = (x1 - x0 + 1)[live], (y1 - y0 + 1)[live]
    n = bw * bh
    end = np.cumsum(n)
    start = end - n
    chunk = 1 << 22                                                   # bound the per-pass pixel lists
    lo = 0
    while lo < len(live):
        hi = max(lo + 1, int(np.searchsorted(end, start[lo] + chunk, side="right")))
        sel = np.arange(lo, hi)
        rep = np.repeat(sel, n[sel])
        k = np.arange(len(rep)) - (start[rep] - start[lo])
        f = live[rep]
        x = x0[f] + k % bw[rep]
        y = y0[f] + k // bw[rep]
        cov, _, _, _, invz = cover(s, f, x, y)
        with np.errstate(divide="ignore"):
            z = f32(1) / invz[cov]
        key = (z.view(np.uint32).astype(np.uint64) << np.uint64(32)) | f[cov].astype(np.uint64)
        np.minimum.at(vis, y[cov] * W + x[cov], key)
        lo = hi
    return vis


def _albedo(mesh, fi, w, base):
    n = len(w)
    if mesh.get("uv") is not None and mesh.get("texture") is not None:
        uv = np.asarray(mesh["uv"], f32)
        tex = np.asarray(mesh["texture"], np.uint8).astype(f32)
        th, tw = tex.shape[:2]
        su = w[:, 0] * uv[fi[:, 0], 0] + w[:, 1] * uv[fi[:, 1], 0] + w[:, 2] * uv[fi[:, 2], 0]
        sv = w[:, 0] * uv[fi[:, 0], 1] + w[:, 1] * uv[fi[:, 1], 1] + w[:, 2] * uv[fi[:, 2], 1]
        tx = np.clip(su * f32(tw) - f32(0.5), -1, tw)
        ty = np.clip((f32(1) - sv) * f32(th) - f32(0.5), -1, th)
        x0, y0 = np.floor(tx), np.floor(ty)
        ax, ay = (tx - x0)[:, None], (ty - y0)[:, None]
        x0, y0 = x0.astype(np.int64), y0.astype(np.int64)

        def t(xx, yy):
            return tex[np.clip(yy, 0, th - 1), np.clip(xx, 0, tw - 1)]
        top = (1 - ax) * t(x0, y0) + ax * t(x0 + 1, y0)
        bot = (1 - ax) * t(x0, y0 + 1) + ax * t(x0 + 1, y0 + 1)
        return ((1 - ay) * top + ay * bot) / f32(255)
    if mesh.get("colors") is not None:
        c = np.asarray(mesh["colors"], np.uint8).astype(f32)
        return (w[:, 0:1] * c[fi[:, 0]] + w[:, 1:2] * c[fi[:, 1]] + w[:, 2:3] * c[fi[:, 2]]) / f32(255)
    return np.broadcast_to(np.asarray(base, f32), (n, 3))


def render_view(mesh, P, K, H, W, ambient=0.3, base_color=(0.8, 0.8, 0.8), znear=1e-3):
    """mesh: dict with vertices (V,3), faces (F,3) and optional colors / uv + texture (numpy); P (4,4) object -> camera
    -> dict rgb (H,W,3) u8, mask (H,W) u8, xyz (H,W,3) f16, tri (H,W) i32, depth (H,W) f32, dropped int, and xyz32 (H,W,3):
    the float32 object coordinates before the f16 store"""
    V = np.asarray(mesh["vertices"], f32)
    P = np.asarray(P, f32)
    X, Y, Z, ok = vertex_pass(V, P, K, znear)
    s = setup(mesh["faces"], X, Y, Z, ok)
    vis = visibility(s, H, W)
    out = dict(rgb=np.zeros((H * W, 3), np.uint8), mask=np.zeros(H * W, np.uint8), xyz=np.zeros((H * W, 3), np.float16),
               tri=np.full(H * W, -1, np.int32), depth=np.zeros(H * W, f32), dropped=int((s["state"] < 0).sum()),
               xyz32=np.zeros((H * W, 3), f32))
    pix = np.flatnonzero(vis != EMPTY)
    if len(pix):
        key = vis[pix]
        f = (key & np.uint64(0xFFFFFFFF)).astype(np.int64)
        _, q0, q1, q2, invz = cover(s, f, pix % W, pix // W)
        w = np.stack([q0 / invz, q1 / invz, q2 / invz], 1)
        fi = s["idx"][f]
        vx = [V[fi[:, k]] for k in range(3)]
        xyz = (w[:, 0:1] * vx[0] + w[:, 1:2] * vx[1]) + w[:, 2:3] * vx[2]
        out["xyz32"][pix] = xyz
        out["xyz"][pix] = xyz.astype(np.float16)
        out["mask"][pix] = 255
        out["tri"][pix] = f.astype(np.int32)
        out["depth"][pix] = (key >> np.uint64(32)).astype(np.uint32).view(f32)
        alb = _albedo(mesh, fi, w, base_color)
        R, t = P[:3, :3].astype(np.float64), P[:3, 3].astype(np.float64)
        pc = [vx[k].astype(np.float64) @ R.T + t for k in range(3)]
        n = np.cross(pc[1] - pc[0], pc[2] - pc[0])
        sp = xyz.astype(np.float64) @ R.T + t
        n = np.where((np.sum(n * sp, 1) > 0)[:, None], -n, n)
        l = -1.5 * t - sp
        nn, ll = np.linalg.norm(n, axis=1), np.linalg.norm(l, axis=1)
        good = (nn > 0) & (ll > 0)
        ndl = np.where(good, np.sum(n * l, 1) / np.where(good, nn * ll, 1), 0)
        shade = ambient + (1 - ambient) * np.maximum(0, ndl)
        out["rgb"][pix] = np.minimum(255, np.floor(alb * shade[:, None] * 255 + 0.5)).astype(np.uint8)
    return dict(rgb=out["rgb"].reshape(H, W, 3), mask=out["mask"].reshape(H, W), xyz=out["xyz"].reshape(H, W, 3),
                tri=out["tri"].reshape(H, W), depth=out["depth"].reshape(H, W), dropped=out["dropped"], xyz32=out["xyz32"].reshape(H, W, 3))


def render(meshes, poses, K, H, W, ambient=0.3, base_color=0.8, znear=1e-3):
    """every view of every mesh: poses (O,T,4,4) -> dict of (O,T,...) arrays and dropped (O,), as sam6d_b200.render.render"""
    O, T = np.asarray(poses).shape[:2]
    base = np.broadcast_to(np.asarray(base_color, f32), (O, 3)) if np.ndim(base_color) < 2 else np.asarray(base_color, f32)
    views = [[render_view(meshes[o], poses[o][t], K, H, W, ambient, base[o], znear) for t in range(T)] for o in range(O)]
    out = {k: np.stack([np.stack([v[k] for v in row]) for row in views]) for k in ("rgb", "mask", "xyz", "tri", "depth")}
    out["dropped"] = np.array([sum(v["dropped"] for v in row) for row in views], np.int32)
    return out


# ---- procedural meshes of the tests and tools/render_bench.py -----------------------------------------------------------

def icosphere(subdiv: int, radius: float = 1.0):
    """-> vertices (V,3) float32, faces (20 * 4^subdiv, 3) int32 of a closed, outward-wound icosphere"""
    t = (1.0 + 5 ** 0.5) / 2.0
    v = [[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t], [t, 0, -1], [t, 0, 1],
         [-t, 0, -1], [-t, 0, 1]]
    f = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6], [7, 1, 8],
         [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10], [8, 6, 7], [9, 8, 1]]
    v = [np.asarray(p, np.float64) / np.linalg.norm(p) for p in v]
    for _ in range(subdiv):
        cache, nf = {}, []

        def mid(a, b):
            key = (min(a, b), max(a, b))
            if key not in cache:
                m = v[a] + v[b]
                v.append(m / np.linalg.norm(m))
                cache[key] = len(v) - 1
            return cache[key]
        for a, b, c in f:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            nf += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        f = nf
    return (np.asarray(v) * radius).astype(np.float32), np.asarray(f, np.int32)


def cube(half: float = 1.0):
    """-> vertices (8,3) float32, faces (12,3) int32 of an axis-aligned cube"""
    v = np.array([[x, y, z] for x in (-half, half) for y in (-half, half) for z in (-half, half)], np.float32)
    f = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4],
                  [1, 5, 7], [1, 7, 3]], np.int32)
    return v, f
