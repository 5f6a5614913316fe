"""numpy restatement of the mesh culling (gssdf_mesh_cull_vertices / _faces, DESIGN 7h) in the kernel's rounding order, the reference's
Mesher::cull_mesh restated line by line in torch (include/mesher/mesher.cpp:76-160), and the knife-edge bound under which the two may
disagree when ATen rounds differently (another host ISA, or the CUDA composition)."""
import numpy as np
import torch

f32 = np.float32
TAU = 2.0 ** -20  # knife-edge bound: 16 fp32 unit roundoffs of the magnitudes a decision is computed from


def fma32(a, b, c):
    """Correctly rounded fp32 fma(a, b, c) on arrays: a*b is exact in fp64, the fp64 sum is made round-to-odd from its exact error
    (TwoSum), and rounding that to fp32 is then a single correct rounding (53 >= 2 * 24 + 2)."""
    a, b, c = (np.asarray(t, f32).astype(np.float64) for t in (a, b, c))
    p = a * b
    s = p + c
    bp = s - c
    err = (p - bp) + (c - (s - bp))  # s + err == p + c exactly (where finite)
    bits = s.view(np.int64)
    fix = np.isfinite(s) & (err != 0) & ((bits & 1) == 0)
    s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    with np.errstate(over="ignore", invalid="ignore"):
        return s.astype(f32)


def random_case(seed, N=20000, B=4, W=160, H=120, Hd=90, Wd=130):
    """Vertices in a 4 m box, cameras outside it looking at its centre, smooth random depth images whose values straddle the vertices'
    camera depths (so d + 0.02 > z goes both ways), an image size unlike the camera's, random faces. Returns (V, F, depths [B,Hd,Wd],
    c2w, w2c = the host torch.inverse of c2w, (fx, fy, cx, cy, W, H))."""
    rng = np.random.default_rng(seed)
    V = rng.uniform(-2, 2, (N, 3)).astype(f32)
    fx, fy, cx, cy = f32(90.0), f32(85.0), f32(79.5), f32(59.5)
    poses, depths = [], []
    for b in range(B):
        pos = rng.normal(size=3)
        pos = pos / np.linalg.norm(pos) * rng.uniform(4, 6)
        f = -pos / np.linalg.norm(pos) + rng.normal(scale=0.1, size=3)
        f /= np.linalg.norm(f)
        right = np.cross(f, [0.0, 0.0, 1.0])
        right /= np.linalg.norm(right)
        P = np.eye(4)
        P[:3, :3] = np.stack([right, np.cross(f, right), f], 1)
        P[:3, 3] = pos
        poses.append(P.astype(f32))
        yy, xx = np.mgrid[0:Hd, 0:Wd]
        base = np.linalg.norm(pos) - 1.0 + 1.5 * np.sin(xx / 9.0 + b) * np.cos(yy / 7.0 - b)
        depths.append((base + rng.normal(scale=0.05, size=(Hd, Wd))).astype(f32))
    poses, depths = np.stack(poses), np.stack(depths)
    w2c = torch.inverse(torch.from_numpy(poses)).numpy()
    F = rng.integers(0, N, (3 * N, 3)).astype(np.int32)
    return V, F, depths, poses, w2c, (fx, fy, cx, cy, W, H)


def _f(x):
    return np.asarray(x, f32)


def frame_sees(V, w2c, D, fx, fy, cx, cy, W, H):
    """One frame's visibility (mesher.cpp:120-153) in the kernel's order. V [N,3] fp32, w2c [4,4] fp32, D [Hd,Wd] fp32."""
    V, w, D = _f(V), _f(w2c), _f(D)
    fx, fy, cx, cy = f32(fx), f32(fy), f32(cx), f32(cy)
    Wf, Hf = f32(W), f32(H)
    Hd, Wd = D.shape
    with np.errstate(all="ignore"):
        # w2c.matmul(homo_points) (:120): ATen's batched kernel for such small matrices sums ((w0 x + w1 y) + w2 z) + w3 * 1, each
        # product and sum rounded on its own (CPU, determined: tests/test_mesh_cull_host.py)
        c = [(((w[r, 0] * V[:, 0]) + (w[r, 1] * V[:, 1])) + (w[r, 2] * V[:, 2])) + w[r, 3] for r in range(3)]
        z = c[2]
        az = np.abs(z)
        p = [c[0] / az, c[1] / az, z / az]  # cam_cord / z.abs() (:126)
        u = ((fx * p[0]) + (f32(0) * p[1])) + (cx * p[2])  # K.matmul(uv) (:127), the same kernel
        v = ((f32(0) * p[0]) + (fy * p[1])) + (cy * p[2])
        gx = (f32(2) * (u / Wf)) - f32(1)  # (:131-135): true divisions by the int W, H
        gy = (f32(2) * (v / Hf)) - f32(1)
        # grid_sample bilinear / zeros / align_corners (:138-146): ATen's vectorised CPU sampler un-normalises (g + 1) * ((size - 1) / 2)
        xs = (gx + f32(1)) * (f32(Wd - 1) / f32(2))
        ys = (gy + f32(1)) * (f32(Hd - 1) / f32(2))
        x0, y0 = np.floor(xs), np.floor(ys)
        wx = xs - x0
        e = f32(1) - wx
        n = ys - y0
        s = f32(1) - n
        ok = (0 <= z) & (u < Wf) & (u > 0) & (v < Hf) & (v > 0)  # (:149-151)
        ix = np.where(ok, x0, 0).astype(np.int64)
        iy = np.where(ok, y0, 0).astype(np.int64)

        def tap(a, b):
            inside = (a >= 0) & (a < Wd) & (b >= 0) & (b < Hd)
            return np.where(inside, D[np.clip(b, 0, Hd - 1), np.clip(a, 0, Wd - 1)], f32(0)).astype(f32)

        # (nw_val * nw) + (ne_val * ne) + (sw_val * sw) + (se_val * se): the sampler's Vectorized products and adds contract into FMAs
        d = tap(ix, iy) * (s * e)
        d = fma32(tap(ix + 1, iy), s * wx, d)
        d = fma32(tap(ix, iy + 1), n * e, d)
        d = fma32(tap(ix + 1, iy + 1), n * wx, d)
        return ok & ((d + f32(0.02)) > z)  # (:152)


def cull(V, F, depths, w2c, fx, fy, cx, cy, W, H, seen=None):
    """seen [N] bool OR-ed over the frames, and the faces with a seen vertex in order (mesher.cpp:157-159). depths [B,Hd,Wd], w2c [B,4,4]."""
    seen = np.zeros(len(V), bool) if seen is None else seen.copy()
    for b in range(len(depths)):
        m = ~seen
        if m.any():
            seen[m] |= frame_sees(V[m], w2c[b], depths[b], fx, fy, cx, cy, W, H)
    F = np.asarray(F)
    keep = seen[F].any(1) if len(F) else np.zeros(0, bool)
    return seen, F[keep].reshape(-1, 3)


def torch_cull_mesh(vertices, faces, depths, poses, K, W, H):
    """Mesher::cull_mesh (mesher.cpp:76-160) line by line on the vertices' device: depths [B,Hd,Wd,1], poses [B,4,4] c2w, K [3,3].
    Returns (~whole_mask, kept faces). The face index keeps the [K,3] shape (the reference's squeeze gives [3] for one kept face)."""
    device = vertices.device
    whole_mask = torch.ones(vertices.size(0), dtype=torch.bool, device=device)
    K = K.to(device)
    ones = torch.ones(vertices.size(0), 1, dtype=torch.float32, device=device)
    homo_points = torch.cat([vertices, ones], 1).reshape(-1, 4, 1)
    for i in range(depths.shape[0]):
        pose = poses[i].to(device)
        depth = depths[i].to(device)
        w2c = torch.inverse(pose.cpu()).to(device)  # the pose inverse stays on the host (DESIGN 7h)
        cam_cord_homo = w2c.matmul(homo_points)
        cam_cord = cam_cord_homo[:, 0:3]
        z = cam_cord[:, -1:]
        z_squeezed = z.reshape(-1)
        uv = cam_cord / z.abs()
        uv = K.matmul(uv)
        uv = uv[:, 0:2].squeeze(-1)
        grid_x = uv[:, 0:1] / W
        grid_y = uv[:, 1:] / H
        grid = torch.cat([grid_x, grid_y], 1)
        grid = 2 * grid - 1
        inp = depth.unsqueeze(0).unsqueeze(1).squeeze(-1)
        flow_field = grid.unsqueeze(0).unsqueeze(1)
        depth_samples = torch.nn.functional.grid_sample(inp, flow_field, mode="bilinear", padding_mode="zeros",
                                                        align_corners=True).reshape(-1)
        mask = ((0 <= z_squeezed) & (uv[:, 0] < W) & (uv[:, 0] > 0) & (uv[:, 1] < H) & (uv[:, 1] > 0)
                & ((depth_samples + 0.02) > z_squeezed))
        whole_mask &= ~mask
    face_mask = ~(whole_mask[faces.long()].all(1))
    valid_face_idx = face_mask.nonzero().reshape(-1)
    return ~whole_mask, faces[valid_face_idx]


def knife_edge(V, depths, w2c, fx, fy, cx, cy, W, H):
    """Vertices whose seen bit another correct fp32 rounding of the composition could flip: for some frame, every decision of mesher.cpp
    :149-152 (z >= 0, 0 < u < W, 0 < v < H, d + 0.02 > z) holds or lies within its bound of the boundary, and at least one lies within
    it, while no frame sees the vertex with every margin clear. Margins are fp64 evaluations from the same fp32 inputs; the bound of
    each is TAU times the magnitudes it is computed from, propagated to first order (camera coordinates -> u, v -> sample position ->
    bilinear depth, whose slope is bounded by the spread of the four taps). Fixed before any comparison was run."""
    V = _f(V).astype(np.float64)
    N = len(V)
    robust = np.zeros(N, bool)
    edge = np.zeros(N, bool)
    for b in range(len(depths)):
        w = _f(w2c[b]).astype(np.float64)
        D = _f(depths[b]).astype(np.float64)
        Hd, Wd = D.shape
        with np.errstate(all="ignore"):
            c = V @ w[:3, :3].T + w[:3, 3]
            S = np.abs(V) @ np.abs(w[:3, :3]).T + np.abs(w[:3, 3])
            z = c[:, 2]
            ez = TAU * S[:, 2]
            az = np.maximum(np.abs(z), 1e-30)
            p0, p1 = c[:, 0] / az, c[:, 1] / az
            u, v = fx * p0 + cx, fy * p1 + cy
            eu = TAU * (np.abs(fx * p0) + abs(cx)) + fx * (TAU * S[:, 0] + np.abs(p0) * ez) / az
            ev = TAU * (np.abs(fy * p1) + abs(cy)) + fy * (TAU * S[:, 1] + np.abs(p1) * ez) / az
            xs = u / W * (Wd - 1)
            ys = v / H * (Hd - 1)
            x0, y0 = np.floor(xs), np.floor(ys)
            ix, iy = np.clip(x0, -1, Wd).astype(np.int64), np.clip(y0, -1, Hd).astype(np.int64)

            def tap(a, bb):
                inside = (a >= 0) & (a < Wd) & (bb >= 0) & (bb < Hd)
                return np.where(inside, D[np.clip(bb, 0, Hd - 1), np.clip(a, 0, Wd - 1)], 0.0)

            t = np.stack([tap(ix, iy), tap(ix + 1, iy), tap(ix, iy + 1), tap(ix + 1, iy + 1)])
            wx, wy = xs - x0, ys - y0
            d = (t[0] * (1 - wx) + t[1] * wx) * (1 - wy) + (t[2] * (1 - wx) + t[3] * wx) * wy
            spread = t.max(0) - t.min(0)
            exs = eu * (Wd - 1) / W + TAU * Wd
            eys = ev * (Hd - 1) / H + TAU * Hd
            ed = spread * (exs + eys) + TAU * np.abs(t).max(0)
            md = d + 0.02 - z
            emd = ed + TAU * (np.abs(d) + 0.02 + np.abs(z)) + ez
            margins = [(z, ez), (u, eu), (W - u, eu), (v, ev), (H - v, ev), (md, emd)]
        clear = np.ones(N, bool)
        possible = np.ones(N, bool)
        for m, e in margins:
            clear &= m > e
            possible &= ~(m < -e)  # NaN margins (z = 0) are never possible
            possible &= ~np.isnan(m)
        robust |= clear
        edge |= possible & ~clear
    return edge & ~robust
