"""Scenes and cotangents of the splat VJP tests (tests/test_splat_vjp_host.py, tests/test_gpu_splat_vjp.py).

Each scene holds the raw parameters the trainer optimises (anchors, offsets, log-scales, logits) and their activation
(splat_vjp_oracle.activate), so the activated and the raw-parameter runs see the same splats. Everything is seeded float32.
"""
import math

import numpy as np

from gssdf_b200 import scene as S

# name: (N, W, H, SH degree, scale_mult). N is never a multiple of 256, so the last CTA of every kernel is partial.
SCENES = {
    "box": (30_001, 1200, 680, 3, None),  # the trainer's image size
    "c1": (50_000, 256, 256, 0, None),  # BASELINE.json configs[0]
    "edge": (6_007, 320, 240, 3, 6.0),
}


def _quat_from_normal(n, rng):
    """(w,x,y,z) of a rotation whose third column is the unit vector n (rows of n)."""
    a = rng.normal(size=n.shape)
    u = np.cross(n, a)
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    v = np.cross(n, u)
    R = np.stack([u, v, n], 2)  # columns u, v, n
    w = np.sqrt(np.maximum(1.0 + R[:, 0, 0] + R[:, 1, 1] + R[:, 2, 2], 1e-12)) / 2
    q = np.stack([w, (R[:, 2, 1] - R[:, 1, 2]) / (4 * w), (R[:, 0, 2] - R[:, 2, 0]) / (4 * w), (R[:, 1, 0] - R[:, 0, 1]) / (4 * w)], 1)
    bad = w < 1e-3  # rotations by ~pi: fall back to the largest diagonal entry
    if bad.any():
        for i in np.nonzero(bad)[0]:
            Ri = R[i]
            k = int(np.argmax(np.diag(Ri)))
            j, l = (k + 1) % 3, (k + 2) % 3
            t = math.sqrt(max(1.0 + Ri[k, k] - Ri[j, j] - Ri[l, l], 1e-12)) / 2
            qi = np.zeros(4)
            qi[1 + k] = t
            qi[1 + j] = (Ri[j, k] + Ri[k, j]) / (4 * t)
            qi[1 + l] = (Ri[l, k] + Ri[k, l]) / (4 * t)
            qi[0] = (Ri[l, j] - Ri[j, l]) / (4 * t)
            q[i] = qi
    return q


def _edge(sc, V, K, W, H, rng):
    """Ill-conditioned splats mixed into a box scene, one group each:
    quaternion norms 1e-3 .. 1e3 (all), near-axis quaternions with w ~ 1e-4 (15 %), scale ratios up to 1e5 (30 %),
    depths within 1e-3 of the near plane (8 %), splats seen almost edge-on (12 %: the normal tilted 10^-3.5 .. 10^-1.5 rad out of the
    plane that holds the viewing ray)."""
    N = len(sc["means"])
    means, quats, scales = sc["means"].astype(np.float64), sc["quats"].astype(np.float64), sc["scales"].astype(np.float64)
    Rcw, t = V[0, :3, :3].astype(np.float64), V[0, :3, 3].astype(np.float64)
    centre = -Rcw.T @ t
    grp = rng.permutation(N)
    near, edge, axis = grp[:N * 8 // 100], grp[N * 8 // 100:N * 20 // 100], grp[N * 20 // 100:N * 35 // 100]
    # near plane: camera depth NEAR + (1e-5 .. 1e-3), on screen
    z = S.NEAR + rng.uniform(1e-5, 1e-3, len(near))
    fx, fy, cx, cy = K[0, 0, 0], K[0, 1, 1], K[0, 0, 2], K[0, 1, 2]
    px, py = rng.uniform(0, W, len(near)), rng.uniform(0, H, len(near))
    mc = np.stack([(px - cx) / fx * z, (py - cy) / fy * z, z], 1)
    means[near] = (mc - t) @ Rcw  # R^T (mc - t)
    scales[near, :2] = rng.uniform(1e-4, 2e-3, (len(near), 2))
    # edge-on: normal perpendicular to the viewing ray, then tilted by eps towards it
    d = means[edge] - centre
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    n = np.cross(d, rng.normal(size=d.shape))
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    eps = 10 ** rng.uniform(-3.5, -1.5, len(edge))
    n = n + eps[:, None] * d * rng.choice([-1.0, 1.0], len(edge))[:, None]
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    quats[edge] = _quat_from_normal(n, rng)
    # near-axis: w ~ 0
    quats[axis, 0] = rng.uniform(-1e-4, 1e-4, len(axis))
    quats[axis, 1:] /= np.linalg.norm(quats[axis, 1:], axis=1, keepdims=True)
    # scale ratios up to 1e5 at constant area
    ratio = grp[N * 50 // 100:N * 80 // 100]
    u = rng.uniform(-5, 5, len(ratio))
    g = np.sqrt(scales[ratio, 0] * scales[ratio, 1])
    scales[ratio, 0], scales[ratio, 1] = g * 10 ** (u / 2), g * 10 ** (-u / 2)
    # quaternion norms 1e-3 .. 1e3
    quats /= np.linalg.norm(quats, axis=1, keepdims=True)
    quats *= 10 ** rng.uniform(-3, 3, (N, 1))
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    return dict(sc, means=f32(means), quats=f32(quats), scales=f32(scales)), dict(near=near, edge=edge, axis=axis, ratio=ratio)


def scene(name):
    """dict(raw, act, quats, V, K, W, H, deg, N, groups): raw = anchors / offsets / log_scales / logits, act = its activation."""
    from splat_vjp_oracle import activate
    N, W, H, deg, scale = SCENES[name]
    sc = S.box_scene(N, deg, seed=5, scale_mult=scale)
    V, K = S.cameras([0], W, H)
    rng = np.random.default_rng(17)
    groups = {}
    if name == "edge":
        sc, groups = _edge(sc, V, K, W, H, rng)
    offsets = (0.01 * rng.standard_normal((N, 3))).astype(np.float32)
    op = np.clip(sc["opacities"].astype(np.float64), 1e-3, 1 - 1e-3)
    raw = dict(anchors=(sc["means"] - offsets).astype(np.float32), offsets=offsets,
               log_scales=np.log(sc["scales"].astype(np.float64)).astype(np.float32), logits=np.log(op / (1 - op)).astype(np.float32))
    means, scales, opac = activate(raw)
    return dict(raw=raw, act=dict(means=means, scales=scales, opacities=opac), quats=sc["quats"], V=V, K=K, W=W, H=H, deg=deg, N=N,
                groups=groups)


def cotangents(nnz, seed=23):
    """One N(0,1) cotangent per branch of the projection backward, and randns uniform in [-4, 4] for the sample branch."""
    rng = np.random.default_rng(seed)
    g = lambda *s: rng.standard_normal(size=s).astype(np.float32)
    cot = dict(v_ray_transforms=g(nnz, 3, 3), v_normals=g(nnz, 3), v_samples=g(nnz, 3), v_pt_opacities=g(nnz), v_means2d=g(nnz, 2),
               v_depths=g(nnz))
    return cot, rng.uniform(-4, 4, (nnz, 2)).astype(np.float32)


def sh_scene(name, K, seed=31):
    """SH coefficients for the colour tests: DC drawn so that roughly half of the (splat, channel) colours clamp at 0, rest
    coefficients large enough that the view-direction gradient matters. dict(sh [N,K,3], dc [N,1,3], rest [N,K-1,3])."""
    N = SCENES[name][0]
    rng = np.random.default_rng(seed)
    sh = np.zeros((N, K, 3), np.float32)
    sh[:, 0] = rng.normal(-1.8, 1.5, (N, 3))  # 0.282 dc + 0.5 <= 0  <=>  dc <= -1.77
    sh[:, 1:] = rng.normal(0, 0.4, (N, K - 1, 3))
    return dict(sh=sh, dc=np.ascontiguousarray(sh[:, :1]), rest=np.ascontiguousarray(sh[:, 1:]))


# The call with all six branches scales each cotangent so that every branch moves >= 5 % of some compared gradient's entries at the
# tolerance (tests/test_splat_vjp_host.py checks it): unscaled, the ray-transform and image-space terms are 1e2..1e6 times the others.
ALL_WEIGHTS = dict(v_ray_transforms=1e-2, v_normals=1.0, v_samples=1.0, v_pt_opacities=1.0, v_means2d=1e-5, v_depths=1e1)
GRAZE_PX = 1.0e5
MAX_EXCLUDED = 0.01


def exclusions(sc, p):
    """fp64 conditioning rules of the projection comparison, as bool masks over the visible rows p (a forward's outputs), per branch
    and for the call with all six ("all"):
    knife: the normal's sign flips within fp32 noise, |n . mu_c| <= 1e-4 |n| |mu_c| (normal branch);
    grazing: |mean2d - principal point| > GRAZE_PX; the image-space VJP divides by distance = M6^2 + M7^2 - M8^2, which cancels for
    splats grazing the camera plane (v_means2d branch)."""
    means = sc["act"]["means"].astype(np.float64)
    gid = np.asarray(p["gaussian_ids"], np.int64)
    V = sc["V"][0].astype(np.float64)
    mc = means[gid] @ V[:3, :3].T + V[:3, 3]
    q = np.asarray(sc["quats"], np.float64)[gid]
    w, x, y, z = (q / np.linalg.norm(q, axis=1, keepdims=True)).T
    nw = np.stack([2 * (x * z + w * y), 2 * (y * z - w * x), 1 - 2 * (x * x + y * y)], 1)  # third column of R(q)
    nc = nw @ V[:3, :3].T
    knife = np.abs((nc * mc).sum(1)) <= 1e-4 * np.linalg.norm(nc, axis=1) * np.linalg.norm(mc, axis=1)
    pp = np.array([sc["K"][0, 0, 2], sc["K"][0, 1, 2]])
    graze = np.linalg.norm(np.asarray(p["means2d"], np.float64) - pp, axis=1) > GRAZE_PX
    none = np.zeros(len(gid), bool)
    out = {b: none for b in ("v_ray_transforms", "v_samples", "v_pt_opacities", "v_depths")}
    out.update(v_normals=knife, v_means2d=graze, all=knife | graze)
    return out
