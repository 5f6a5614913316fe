"""Seeded synthetic scenes standing in for Replica / FAST-LIVO2 (SURVEY.md section 8d).

`box_scene(N, seed)` places N 2D splats on the inside faces of a Replica-room sized box;
`camera(i, W, H)` draws a pinhole camera inside it. Everything is numpy float32 so the CPU
oracle, the golden generators and the CUDA path consume identical bits.
"""
import math

import numpy as np

BOX = np.array([3.0, 2.0, 1.5], np.float64)  # half extents [m]; Replica room scale (replica.yaml:25 map 14 m)
NEAR, FAR = 0.05, 300.0  # config/base.yaml:41-42


def box_scene(N, sh_degree=3, seed=0, scale_mult=None):
    """Activated splat parameters as `NeuralGS::generate_gaussian` hands them to the renderer
    (neural_gaussian.cpp:480-492): means[N,3], quats[N,4] (w,x,y,z, unnormalised), scales[N,3]
    (already exp'ed), opacities[N] (already sigmoid'ed), sh[N,K,3]."""
    rng = np.random.default_rng(seed)
    hx, hy, hz = BOX
    areas = np.array([hy * hz, hy * hz, hx * hz, hx * hz, hx * hy, hx * hy]) * 4
    face = rng.choice(6, size=N, p=areas / areas.sum())
    uv = rng.uniform(-1, 1, size=(N, 2))
    means = np.zeros((N, 3))
    axis = face // 2
    sign = np.where(face % 2 == 0, -1.0, 1.0)
    for a in range(3):
        m = axis == a
        o = [i for i in range(3) if i != a]
        means[m, a] = sign[m] * BOX[a]
        means[m, o[0]] = uv[m, 0] * BOX[o[0]]
        means[m, o[1]] = uv[m, 1] * BOX[o[1]]
    if scale_mult is None:
        scale_mult = math.sqrt(1.0e6 / N)  # keep screen coverage constant as N changes
    s_xy = np.exp(rng.uniform(math.log(0.005), math.log(0.05), size=(N, 2))) * scale_mult
    scales = np.concatenate([s_xy, np.full((N, 1), 1e-6)], 1)  # gs.ply convention scale_2 = 1e-6
    quats = rng.normal(size=(N, 4))
    opac = rng.uniform(0.05, 0.95, size=N)
    K = (sh_degree + 1) ** 2
    sh = np.zeros((N, K, 3))
    sh[:, 0] = rng.uniform(0, 1, size=(N, 3))
    if K > 1:
        sh[:, 1:] = rng.normal(0, 0.05, size=(N, K - 1, 3))
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    return dict(means=f32(means), quats=f32(quats), scales=f32(scales), opacities=f32(opac), sh=f32(sh))


def camera(i, W, H, seed_base=1000):
    """viewmat[4,4] (world->camera, OpenCV axes: x right, y down, z forward) and K[3,3]."""
    rng = np.random.default_rng(seed_base + i)
    pos = rng.uniform(-0.5, 0.5, size=3) * BOX
    yaw = rng.uniform(0, 2 * math.pi)
    pitch = rng.uniform(-0.3, 0.3)
    f = np.array([math.cos(pitch) * math.cos(yaw), math.cos(pitch) * math.sin(yaw), math.sin(pitch)])
    up = np.array([0.0, 0.0, 1.0])
    right = np.cross(f, up)
    right /= np.linalg.norm(right)
    down = np.cross(f, right)
    R_c2w = np.stack([right, down, f], 1)
    V = np.eye(4)
    V[:3, :3] = R_c2w.T
    V[:3, 3] = -R_c2w.T @ pos
    K = np.array([[W / 2.0, 0, (W - 1) / 2.0], [0, W / 2.0, (H - 1) / 2.0], [0, 0, 1.0]])
    return np.ascontiguousarray(V, np.float32), np.ascontiguousarray(K, np.float32)


def cameras(ids, W, H):
    vs, ks = zip(*[camera(i, W, H) for i in ids])
    return np.stack(vs), np.stack(ks)


def randns(n, seed=7):
    return np.random.default_rng(seed).standard_normal(size=(n, 2)).astype(np.float32)


def cotangents(C, H, W, seed=11):
    """Direct cotangent images for kernel-level backward parity (SURVEY 8d: v_* ~ N(0,1) seed 11)."""
    rng = np.random.default_rng(seed)
    g = lambda *s: rng.standard_normal(size=s).astype(np.float32)
    return dict(v_render_colors=g(C, H, W, 3), v_render_depths=g(C, H, W, 1), v_render_alphas=g(C, H, W, 1),
                v_render_normals=g(C, H, W, 3), v_render_median=g(C, H, W, 1))


CONFIGS = {
    # BASELINE.json configs (c1..c5) as concrete splat-path inputs
    "c1": dict(W=256, H=256, N=50_000, sh_degree=0),
    "c2": dict(W=1200, H=680, N=500_000, sh_degree=3),
    "c3": dict(W=1920, H=1080, N=2_000_000, sh_degree=3),
    "c4": dict(W=1920, H=1080, N=1_000_000, sh_degree=3),  # per scene / per GPU
    "c5": dict(W=3840, H=2160, N=5_000_000, sh_degree=3),
}


def box_signed_distance(x):
    """Signed distance to the walls of the BOX room, positive inside (free space), float64 numpy or torch [n,3]."""
    if hasattr(x, "detach"):
        import torch
        b = torch.as_tensor(BOX, dtype=x.dtype, device=x.device)
        q = x.abs() - b
        outside = q.clamp_min(0).norm(dim=-1)
        inside = q.max(-1).values.clamp_max(0)
        return -(outside + inside)
    q = np.abs(x) - BOX
    return -(np.linalg.norm(np.maximum(q, 0), axis=-1) + np.minimum(q.max(-1), 0))


def box_wall_points(spacing, offsets=(0.0,)):
    """Regular samples of the six inside faces of the BOX room, shifted along the wall normal by each of `offsets` (float32 [n,3])."""
    out = []
    for a in range(3):
        o = [i for i in range(3) if i != a]
        u = np.arange(-BOX[o[0]], BOX[o[0]] + 1e-9, spacing)
        v = np.arange(-BOX[o[1]], BOX[o[1]] + 1e-9, spacing)
        uu, vv = np.meshgrid(u, v, indexing="ij")
        for sgn in (-1.0, 1.0):
            for off in offsets:
                p = np.zeros((uu.size, 3))
                p[:, a] = sgn * (BOX[a] + off)
                p[:, o[0]], p[:, o[1]] = uu.reshape(-1), vv.reshape(-1)
                out.append(p)
    return np.ascontiguousarray(np.concatenate(out), np.float32)


def box_room_sdf_net(device, inner_map_size=14.0, leaf_size=0.05, steps=1000, seed=0, pos_W_M=(0.0, 0.0, 0.0), mlp_mode=None, batch=1 << 16):
    """A SubMap holding the BOX room: (SdfNet, OctreeAS, (xyz_min_M_margin, xyz_max_M_margin)).
    Octree as SubMap::update_octree_as (sub_map.cpp:22-35): quantise, unique, 27-neighbour dilation, clamp; applied to points on the walls
    and up to one leaf to either side of them, so that the walls lie well inside the dilated octree. Level and map size as params.cpp:474-478.
    The net is fitted with the autograd mirror (sdf.SdfNet) and torch.optim.Adam to the room's signed distance, positive inside.
    Test and benchmark infrastructure (GPU)."""
    import torch

    from . import octree as OT
    from . import sdf as SD
    f = np.float32
    level = int(math.ceil(math.log2(float(f(f(inner_map_size) + f(2 * f(leaf_size))) * f(f(1.0) / f(leaf_size))))))
    map_size = float(f(f(2 ** level) * f(leaf_size)))
    pos = np.asarray(pos_W_M, np.float32)
    wall = box_wall_points(leaf_size / 2, (-leaf_size, -leaf_size / 2, 0.0, leaf_size / 2, leaf_size))
    xw = torch.from_numpy(wall).to(device)
    pos_t = torch.from_numpy(pos).to(device)
    m1p1 = ((xw - pos_t) * 2) * f(f(1.0) / f(map_size))  # SubMap::xyz_to_m1p1_pts
    q = torch.unique(OT.quantize_points(m1p1, level), dim=0)
    d = torch.tensor([[i, j, k] for i in (-1, 0, 1) for j in (-1, 0, 1) for k in (-1, 0, 1)], dtype=torch.int32, device=device)
    q = (q.to(torch.int32)[:, None, :] + d[None]).view(-1, 3).clamp(0, 2 ** level - 1).to(torch.int16)  # points_to_neighbors + clamp
    tree = OT.OctreeAS.from_quantized_points(q, level, device, origin=tuple(float(v) for v in pos), map_size=map_size)
    net = SD.SdfNet(device, origin=tuple(float(v) for v in pos), map_size=map_size, seed=1337 + seed, mlp_mode=mlp_mode)
    g = torch.Generator(device=device).manual_seed(seed)
    opt = torch.optim.Adam([{"params": [net.params_], "lr": 1e-2}, {"params": [net.decoder_], "lr": 2e-3}], eps=1e-15)
    b = torch.as_tensor(BOX, dtype=torch.float32, device=device)
    for _ in range(steps):
        # half the batch on the walls +- a 0.3 m band, half uniform in the room and around it
        idx = torch.randint(0, xw.shape[0], (batch // 2,), device=device, generator=g)
        near = xw[idx] + torch.randn(batch // 2, 3, device=device, generator=g) * 0.1
        far = (torch.rand(batch // 2, 3, device=device, generator=g) * 2 - 1) * (b + 0.5)
        x = torch.cat([near, far]).contiguous()
        target = box_signed_distance(x)
        sdf, _ = net.get_sdf(x)
        loss = (sdf[:, 0] - target).abs().mean()
        opt.zero_grad(set_to_none=False)
        loss.backward()
        opt.step()
    lo = tuple(float(f(f(-0.5 * inner_map_size) + f(0.5 * leaf_size))) for _ in range(3))  # xyz_min_M_ + 0.5 * k_leaf_size (sub_map.cpp:17-18)
    hi = tuple(float(f(f(0.5 * inner_map_size) - f(0.5 * leaf_size))) for _ in range(3))
    return net, tree, (lo, hi)


# an occluding pillar for the culling scenes: floor to ceiling, NOT part of box_room_sdf_net's SDF, in front of the cameras' cluster
PILLAR_MIN = np.array([0.5, -0.3, -BOX[2]], np.float64)
PILLAR_MAX = np.array([1.1, 0.3, BOX[2]], np.float64)
CULL_CAM_CENTER = np.array([-1.5, 0.0, 0.0], np.float64)


def box_room_cull_poses(n, seed=0, radius=0.1, max_yaw=math.radians(50.0), max_pitch=0.2):
    """c2w [n,4,4] float32 (OpenCV axes: x right, y down, z forward) for the culling scenes: positions within `radius` of
    CULL_CAM_CENTER, looking toward +x with |yaw| <= max_yaw, so the -x wall behind them is never in view, and the pillar hides the
    same patch of the +x wall from all of them."""
    rng = np.random.default_rng(seed)
    out = np.zeros((n, 4, 4))
    for i in range(n):
        d = rng.normal(size=3)
        pos = CULL_CAM_CENTER + radius * rng.uniform() ** (1 / 3) * d / np.linalg.norm(d)
        yaw, pitch = rng.uniform(-max_yaw, max_yaw), rng.uniform(-max_pitch, max_pitch)
        f = np.array([math.cos(pitch) * math.cos(yaw), math.cos(pitch) * math.sin(yaw), math.sin(pitch)])
        right = np.cross(f, [0.0, 0.0, 1.0])
        right /= np.linalg.norm(right)
        down = np.cross(f, right)
        out[i, :3, :3] = np.stack([right, down, f], 1)
        out[i, :3, 3] = pos
        out[i, 3, 3] = 1.0
    return out.astype(np.float32)


def box_room_pack(device, n_frames, ds_pt_num=10_000, W=160, H=120, seed=0):
    """A training depth pack of the BOX room (no pillar) in the layout base_parser.cpp:925-960 builds: per frame `ds_pt_num` pixels drawn
    without replacement (the per-frame downsampling of k_ds_pt_num), origin = camera centre, unit direction, depth = range along the ray,
    xyz = direction * depth + origin. Cameras anywhere in the inner half of the room, any yaw, pitch within +-0.8 rad, so every wall,
    the floor and the ceiling are seen. Returns a dict of float32 tensors on `device`: origin [N,3], direction [N,3], depth [N,1], xyz [N,3].
    Test and benchmark infrastructure."""
    import torch
    rng = np.random.default_rng(seed)
    c2w = np.zeros((n_frames, 4, 4))
    for i in range(n_frames):
        yaw, pitch = rng.uniform(0, 2 * math.pi), rng.uniform(-0.8, 0.8)
        f = np.array([math.cos(pitch) * math.cos(yaw), math.cos(pitch) * math.sin(yaw), math.sin(pitch)])
        right = np.cross(f, [0.0, 0.0, 1.0])
        right /= np.linalg.norm(right)
        c2w[i, :3, :3] = np.stack([right, np.cross(f, right), f], 1)
        c2w[i, :3, 3] = rng.uniform(-0.5, 0.5, 3) * BOX
        c2w[i, 3, 3] = 1.0
    fx = fy = W / 2.0
    cx, cy = (W - 1) / 2.0, (H - 1) / 2.0
    P = torch.from_numpy(c2w).to(device)
    z = box_room_depth(P.to(torch.float32), fx, fy, cx, cy, W, H, pillar=False)[..., 0].reshape(n_frames, -1).to(torch.float64)
    k = min(ds_pt_num, W * H)
    pix = torch.from_numpy(np.stack([rng.choice(W * H, k, replace=False) for _ in range(n_frames)])).to(device)
    j, i = (pix % W).to(torch.float64), (pix // W).to(torch.float64)
    dc = torch.stack([(j - cx) / fx, (i - cy) / fy, torch.ones_like(j)], -1)  # [B,k,3] camera ray with z = 1
    norm = dc.norm(dim=-1, keepdim=True)
    d = torch.einsum("brc,bkc->bkr", P[:, :3, :3], dc / norm)
    rng_ = (torch.gather(z, 1, pix) * norm[..., 0])[..., None]
    o = P[:, None, :3, 3].expand(-1, k, -1)
    f32 = lambda t: t.reshape(-1, t.shape[-1]).to(torch.float32).contiguous()
    origin, direction, depth = f32(o), f32(d), f32(rng_)
    return dict(origin=origin, direction=direction, depth=depth, xyz=(direction * depth + origin).contiguous())


def box_room_depth(c2w, fx, fy, cx, cy, W, H, pillar=True, batch=16):
    """Analytic z-depth images [B,H,W,1] float32 of the BOX room's inner walls (plus the occluding pillar) seen from the c2w poses
    [B,4,4] (torch, any device; rendered there `batch` frames at a time), pixel (i, j) along K^-1 [j, i, 1], as the reference's
    get_depth_image hands them to Mesher::cull_mesh. Test and benchmark infrastructure."""
    import torch
    dev = c2w.device
    j = torch.arange(W, dtype=torch.float64, device=dev)
    i = torch.arange(H, dtype=torch.float64, device=dev)
    dc = torch.stack([((j[None, :] - cx) / fx).expand(H, W), ((i[:, None] - cy) / fy).expand(H, W), torch.ones(H, W, dtype=torch.float64,
                                                                                                             device=dev)], -1)
    box = torch.as_tensor(BOX, dtype=torch.float64, device=dev)
    pmin = torch.as_tensor(PILLAR_MIN, dtype=torch.float64, device=dev)
    pmax = torch.as_tensor(PILLAR_MAX, dtype=torch.float64, device=dev)
    out = []
    for b0 in range(0, c2w.shape[0], batch):
        P = c2w[b0:b0 + batch].to(torch.float64)
        o = P[:, None, None, :3, 3]
        d = torch.einsum("brc,hwc->bhwr", P[:, :3, :3], dc)  # world direction with camera z = 1, so the ray parameter is the z-depth
        with torch.no_grad():
            t_wall = torch.where(d > 0, (box - o) / d, torch.where(d < 0, (-box - o) / d, torch.full_like(d, float("inf")))).amin(-1)
            t = t_wall
            if pillar:
                t1, t2 = (pmin - o) / d, (pmax - o) / d
                t_in = torch.minimum(t1, t2).amax(-1)
                t_out = torch.maximum(t1, t2).amin(-1)
                hit = (t_in <= t_out) & (t_in > 0)
                t = torch.where(hit, torch.minimum(t_in, t_wall), t_wall)
        out.append(t.to(torch.float32)[..., None])
    return torch.cat(out, 0)


def box_room_color(c2w, fx, fy, cx, cy, W, H, batch=16):
    """Colour images [B,H,W,3] float32 in [0.1, 0.9] of the BOX room (no pillar) seen from the c2w poses [B,4,4] (torch, any device):
    each pixel's ray along K^-1 [j, i, 1] hits a wall, whose colour there is a smooth procedural texture of the hit point (a few
    sinusoids per channel, periods 0.5 to 2 m), so that a trained render has a ground truth to converge to. Test and benchmark
    infrastructure."""
    import torch
    dev = c2w.device
    j = torch.arange(W, dtype=torch.float64, device=dev)
    i = torch.arange(H, dtype=torch.float64, device=dev)
    dc = torch.stack([((j[None, :] - cx) / fx).expand(H, W), ((i[:, None] - cy) / fy).expand(H, W), torch.ones(H, W, dtype=torch.float64,
                                                                                                             device=dev)], -1)
    box = torch.as_tensor(BOX, dtype=torch.float64, device=dev)
    freq = torch.tensor([[3.1, 1.7, 4.3], [2.3, 5.1, 1.3], [4.7, 2.9, 3.7]], dtype=torch.float64, device=dev)
    phase = torch.tensor([0.3, 1.9, 4.1], dtype=torch.float64, device=dev)
    out = []
    for b0 in range(0, c2w.shape[0], batch):
        P = c2w[b0:b0 + batch].to(torch.float64)
        o = P[:, None, None, :3, 3]
        d = torch.einsum("brc,hwc->bhwr", P[:, :3, :3], dc)
        with torch.no_grad():
            t = torch.where(d > 0, (box - o) / d, torch.where(d < 0, (-box - o) / d, torch.full_like(d, float("inf")))).amin(-1)
            x = o + t[..., None] * d
            c = 0.5 + 0.2 * torch.sin(x @ freq.T + phase) + 0.2 * torch.sin(0.5 * (x @ freq) - phase)
        out.append(c.clamp(0.1, 0.9).to(torch.float32))
    return torch.cat(out, 0)
