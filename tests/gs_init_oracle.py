"""numpy restatement of the splat-initialisation epilogue (gssdf_sdf_init_gs / gssdf_rot6d_to_quat, DESIGN 7g) and of the reference lines
around it (include/neural_gaussian/neural_gaussian.cpp:19-127, 293-424; include/utils/utils.cpp:693-719).

`dtype=np.float32` rounds every operation once, in the order ATen's separate kernels do; `dtype=np.float64` is the same formula in
double, the yardstick for the fp32 path on well-conditioned rows."""
import math

import numpy as np


def normalize(v, eps, dt):
    """F::normalize(v, dim=-1, eps): v / clamp_min(||v||, eps); NaN propagates through the clamp like ATen's clamp_min."""
    v = v.astype(dt)
    with np.errstate(invalid="ignore", over="ignore"):
        nrm = np.sqrt(v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1] + v[:, 2] * v[:, 2])
        nrm = np.where(np.isnan(nrm), nrm, np.maximum(nrm, dt(eps)))
    with np.errstate(invalid="ignore", divide="ignore"):
        return v / nrm[:, None]


def rot6d_matrix(a1, a2, dt):
    """utils::rotation_6d_to_matrix(cat(a1, a2)) followed by the column permutation [b2, b3, b1] of neural_gaussian.cpp:68-69."""
    b1 = normalize(a1, 1e-12, dt)
    a2 = a2.astype(dt)
    with np.errstate(invalid="ignore", over="ignore"):
        t = ((b1[:, 0] * a2[:, 0] + b1[:, 1] * a2[:, 1]) + b1[:, 2] * a2[:, 2])[:, None]
        b2 = normalize(a2 - t * b1, 1e-12, dt)
        if dt == np.float32:  # the kernel's b1 x b2 is fma(b1[i], b2[j], -b1[j] b2[i]): an exact product, one rounding (fp64 emulation)
            b3 = np.stack([(b1[:, i].astype(np.float64) * b2[:, j] - (b1[:, j] * b2[:, i]).astype(np.float64)).astype(dt)
                           for i, j in ((1, 2), (2, 0), (0, 1))], -1)
        else:
            b3 = np.cross(b1, b2)
    return np.stack([b2, b3, b1], -1)  # M[:, r, c]


def matrix_to_quat(M, dt):
    """neural_gaussian.cpp:76-100: trace -> acos -> axis / (2 sin) -> normalize -> (cos(a/2), sin(a/2) axis) -> nan_to_num."""
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        trace = (M[:, 0, 0] + M[:, 1, 1]) + M[:, 2, 2]
        angle = np.arccos((trace - dt(1)) * dt(0.5))
        den = dt(2) * np.sin(angle)
        axis = np.stack([M[:, 2, 1] - M[:, 1, 2], M[:, 0, 2] - M[:, 2, 0], M[:, 1, 0] - M[:, 0, 1]], -1) / den[:, None]
        axis = normalize(axis, 1e-12, dt)
        h = angle * dt(0.5)
        q = np.concatenate([np.cos(h)[:, None], np.sin(h)[:, None] * axis], -1)
    big = np.finfo(np.float32).max
    return np.nan_to_num(q, nan=0.0, posinf=big, neginf=-big).astype(dt), trace


def rot6d_to_quat(a1, a2, dt=np.float32):
    return matrix_to_quat(rot6d_matrix(a1, a2, dt), dt)


def epilogue(s7, y1, delta, bce_isigma, dt=np.float32):
    """s7: [7, n] SDF values (variant 0 = the point, 1..6 = +x,-x,+y,-y,+z,-z); y1: [n] decoder output 1 of the point.
    Returns dict grad, curv_dom, quaternion, opacity (+ trace) in dtype dt."""
    s7 = s7.astype(dt)
    inv_delta = 1.0 / float(np.float32(delta))
    gcoef, hcoef = dt(0.5 * inv_delta), dt(inv_delta * inv_delta)
    s = s7[0]
    sp, sm = s7[1::2], s7[2::2]                       # [3, n]
    grad = (gcoef * (sp - sm)).T
    curv = (hcoef * ((sp + sm) - dt(2) * s)).T
    q, trace = rot6d_to_quat(normalize(grad, 1e-12, dt), normalize(curv, 1e-12, dt), dt)
    y = y1.astype(dt)
    with np.errstate(over="ignore"):
        yb = y * dt(100)
        soft = np.where(yb > dt(20), y, np.log1p(np.exp(yb)) / dt(100)).astype(dt)
    isigma = soft * dt(bce_isigma) + dt(1)
    opacity = np.exp(-(s * s) * isigma).astype(dt)
    return dict(grad=grad, curv_dom=curv, quaternion=q, opacity=opacity, trace=trace)


def quat_to_matrix(q):
    """Rotation matrix of a unit quaternion (w, x, y, z), float64."""
    q = q.astype(np.float64)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                     np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                     np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def well_conditioned(trace, margin=1e-2):
    """Rows whose axis and angle are determined to fp32 accuracy: the axis is divided by 2 sin(angle) and acos' slope is 1 / sin(angle),
    so rows within `margin` of trace = -1 (angle pi) or trace = 3 (angle 0) amplify the last-bit differences of the matrix."""
    t = trace.astype(np.float64)
    return np.isfinite(t) & (np.abs(1 + t) > margin) & (np.abs(3 - t) > margin)


def crafted_cases(seed=0):
    """(a1, a2, names): identity, exact half-turns, a1 parallel to a2, zero vectors."""
    rows = [((0, 0, 1), (1, 0, 0), "identity"),
            ((0, 0, -1), (1, 0, 0), "half-turn x"),     # M = diag(1, -1, -1)
            ((0, 0, -1), (-1, 0, 0), "half-turn y"),    # M = diag(-1, 1, -1)
            ((0, 0, 1), (-1, 0, 0), "half-turn z"),     # M = diag(-1, -1, 1)
            ((0, 0, 1), (0, 0, 2), "parallel"),
            ((1, 2, 3), (-2, -4, -6), "antiparallel"),
            ((0, 0, 0), (1, 0, 0), "zero a1"),
            ((0, 0, 1), (0, 0, 0), "zero a2"),
            ((0, 0, 0), (0, 0, 0), "zero both")]
    a1 = np.array([r[0] for r in rows], np.float32)
    a2 = np.array([r[1] for r in rows], np.float32)
    rng = np.random.default_rng(seed)  # plus near-identity frames, where the fp32 trace lands on 3 and the axis is 0 / 0
    e = rng.normal(size=(8, 4)).astype(np.float32) * np.float32(1e-4)
    a1 = np.concatenate([a1, np.stack([e[:, 0], e[:, 1], np.ones(8, np.float32)], -1)])
    a2 = np.concatenate([a2, np.stack([np.ones(8, np.float32), e[:, 2], e[:, 3]], -1)])
    return a1, a2, [r[2] for r in rows] + ["near identity"] * 8


def anchor_indices_reference(n_vertices, cap):
    """neural_gaussian.cpp:302-306 literally: valid_vertices_idx.slice(0, 0, -1, sample_step) as torch computes it."""
    import torch
    idx = torch.arange(n_vertices)
    if idx.size(0) > cap:
        step = max(idx.size(0) // cap, 1)
        idx = idx[0:-1:step]
    return idx.tolist()


def sky_reference(spatial_scale, inner_map_size):
    """:335-356 with C++'s types: int(1000 * float), 0.6f * float, log(double(1.1f) * M_PI * r * r / n) rounded to fp32."""
    f = np.float32
    n = int(f(1000) * f(spatial_scale))
    r = f(0.6) * f(inner_map_size)
    return n, float(r), float(f(math.log(np.float64(f(1.1)) * math.pi * np.float64(r) * np.float64(r) / np.float64(n))))


# ---- torch composition of the reference's code on this project's operators (GPU tests, tools/gs_init_bench.py) ----------------------
def rot6d_composition(a1, a2):
    """utils::rotation_6d_to_matrix + neural_gaussian.cpp:68-100 in torch, op for op."""
    import torch
    b1 = torch.nn.functional.normalize(a1, dim=-1)
    b2 = a2 - (b1 * a2).sum(-1, keepdim=True) * b1
    b2 = torch.nn.functional.normalize(b2, dim=-1)
    b3 = torch.cross(b1, b2, dim=-1)
    rot = torch.stack([b1, b2, b3], -1)
    rot = torch.stack([rot[..., 1], rot[..., 2], rot[..., 0]], -1)
    trace = rot[:, 0, 0] + rot[:, 1, 1] + rot[:, 2, 2]
    angle = torch.acos((trace.unsqueeze(-1) - 1.0) * 0.5)
    axis = torch.stack([rot[:, 2, 1] - rot[:, 1, 2], rot[:, 0, 2] - rot[:, 2, 0], rot[:, 1, 0] - rot[:, 0, 1]], -1) / (2.0 * torch.sin(angle))
    axis = torch.nn.functional.normalize(axis, dim=-1)
    q = torch.cat([torch.cos(angle * 0.5), torch.sin(angle * 0.5) * axis], -1).nan_to_num()
    return q, trace


def composition(net, xyz, delta):
    """init_gs_with_sdf(local_map, xyz, delta, true) with LocalMap::get_gradient's numerical branch, on SdfNet.get_sdf."""
    import torch
    with torch.no_grad():
        n = xyz.shape[0]
        offsets = torch.tensor([[[delta, 0.0, 0.0]], [[-delta, 0.0, 0.0]], [[0.0, delta, 0.0]], [[0.0, -delta, 0.0]], [[0.0, 0.0, delta]],
                                [[0.0, 0.0, -delta]]], dtype=torch.float32, device=xyz.device)
        points = xyz.unsqueeze(0) + offsets
        ps = net.get_sdf(points.view(-1, 3))[0].view(6, n, 1)
        inv_delta = 1.0 / delta
        grad = 0.5 * inv_delta * torch.cat([ps[0] - ps[1], ps[2] - ps[3], ps[4] - ps[5]], 1)
        sdf0 = net.get_sdf(xyz)[0]
        hess = inv_delta * inv_delta * (torch.cat([ps[0] + ps[1], ps[2] + ps[3], ps[4] + ps[5]], 1) - 2 * sdf0)
        q, trace = rot6d_composition(torch.nn.functional.normalize(grad, dim=-1), torch.nn.functional.normalize(hess, dim=-1))
        sdf, isigma = net.get_sdf(xyz)
        opacity = torch.exp(-sdf.square() * isigma).squeeze()
    return dict(grad=grad, curv_dom=hess, quaternion=q, opacity=opacity), trace
