"""The depth-to-normal frame of export_test_image (include/neural_mapping/neural_mapping.cpp:1288-1310), restated twice:

  restate(...)          numpy fp64, the contract of gssdf_render_depth_normal_u8 (include/gssdf_b200.h): world points without the camera
                        position, the 4-neighbour cross product, c / max(|c|, 1e-12), * alpha, * 0.5, + 0.5, trunc8;
  export_test_image(...) a line-by-line torch transcription of the reference's composition (sensor::get_image_coords_zdir,
                        depth_to_points, depth_point_to_normal, then tensor_to_cv_mat(depth2normal * alpha * 0.5f + 0.5f)) in any dtype:
                        fp64 as the arbiter, fp32 as what the reference computes.

Both return (bytes uint8 [C,H,W,3], q float64 [C,H,W,3]) with q = 255 * clamp(value, 0, 1) before the truncation."""
import numpy as np


def restate(depth, alpha, V, K):
    """depth, alpha [C,H,W]; V [C,4,4] world->camera; K [C,3,3] (any float arrays, evaluated in fp64)."""
    depth, alpha = np.asarray(depth, np.float64), np.asarray(alpha, np.float64)
    V, K = np.asarray(V, np.float64), np.asarray(K, np.float64)
    C, H, W = depth.shape
    n = np.zeros((C, H, W, 3))
    for c in range(C):
        xs, ys = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
        zx, zy = (xs + 0.5 - K[c, 0, 2]) / K[c, 0, 0], (ys + 0.5 - K[c, 1, 2]) / K[c, 1, 1]
        d = np.stack([V[c, 0, k] * zx + V[c, 1, k] * zy + V[c, 2, k] for k in range(3)], -1)  # rot @ zdir, rot = R^T
        P = d * depth[c][..., None]
        if H >= 3 and W >= 3:
            a = P[2:, 1:-1] - P[:-2, 1:-1]
            b = P[1:-1, 2:] - P[1:-1, :-2]
            cr = np.cross(a, b)
            n[c, 1:-1, 1:-1] = cr / np.maximum(np.linalg.norm(cr, axis=-1, keepdims=True), 1e-12)
    v = n * alpha[..., None] * 0.5 + 0.5
    with np.errstate(invalid="ignore"):
        q = np.clip(v, 0.0, 1.0) * 255.0
    out = np.where(np.isnan(q), 0, np.trunc(np.nan_to_num(q))).astype(np.uint8)
    return out, q


def export_test_image(depth, alpha, V, K, dtype):
    """The reference's composition in torch at `dtype`, with color_pose the camera->world pose whose view matrix is V."""
    import torch
    depth, alpha = torch.as_tensor(np.asarray(depth)), torch.as_tensor(np.asarray(alpha))
    V, K = np.asarray(V, np.float64), np.asarray(K, np.float64)
    C, H, W = depth.shape
    outs, qs = [], []
    for c in range(C):
        fx, fy, cx, cy = (float(np.asarray(K[c, i, j], np.float32 if dtype == torch.float32 else np.float64))
                          for i, j in ((0, 0), (1, 1), (0, 2), (1, 2)))
        # get_image_coords_zdir
        vu = torch.stack(torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij"), -1).to(dtype) + 0.5
        pt_x = (vu.select(2, 1) - cx) / fx
        pt_y = (vu.select(2, 0) - cy) / fy
        zdir = torch.stack([pt_x, pt_y, torch.ones_like(pt_x)], -1)
        # depth_to_points
        Rt = V[c, :3, :3].T  # color_pose = [R | t] with the view matrix [R^T, -R^T t] (NeuralGS::render): the rotation is V's transpose
        pose = torch.from_numpy(np.concatenate([Rt, -Rt @ V[c, :3, 3:4]], 1)).to(dtype)
        pos = pose[:, 3:4].squeeze()
        rot = pose[:, 0:3]
        d = depth[c].to(dtype).reshape(H, W, 1)
        render_points = zdir.matmul(rot.t()) * d + pos
        # depth_point_to_normal
        depth_normal = torch.zeros_like(render_points)
        if H >= 3 and W >= 3:
            dx = torch.cat([render_points[2:, 1:-1] - render_points[:-2, 1:-1]], 0)
            dy = torch.cat([render_points[1:-1, 2:] - render_points[1:-1, :-2]], 1)
            normal_map = torch.nn.functional.normalize(torch.cross(dx, dy, dim=-1), dim=-1)
            depth_normal[1:-1, 1:-1] = normal_map
        # export_test_image: depth2normal * alpha, then tensor_to_cv_mat(x * 0.5f + 0.5f)
        depth2normal = depth_normal * alpha[c].to(dtype).reshape(H, W, 1)
        x = depth2normal * 0.5 + 0.5
        y = x.clamp(0.0, 1.0) * 255
        outs.append(y.to(torch.uint8).numpy())
        qs.append(y.double().numpy())
    return np.stack(outs), np.stack(qs)
