"""f-6 splat initialisation from the trained SDF over the C ABI (DESIGN 7g).

`init_gs_with_sdf` is the reference's init_gs_with_sdf (include/neural_gaussian/neural_gaussian.cpp:19-127) as one gssdf_sdf_init_gs call;
`neural_gs_init` is the tensor part of NeuralGS::NeuralGS's `mesh_init && sdf_enable && geo_init` branch (:273-424): mesh the SDF, stride
the vertices down to the anchors, orient them from the SDF, append the sky sphere, draw the colours and drop NaN rows. The library never
syncs or allocates; `neural_gs_init` reads the mesh counts and the NaN count back once each, like the reference.

f-10 (DESIGN 7k): `dist_cuda2` is simple-knn's distCUDA2 as one gssdf_knn3_mean_dist2 call, and `neural_gs_init_points` is the
constructor's other branch, which starts from the depth cloud and sizes each splat by its three nearest neighbours."""
import ctypes as C
import math

import numpy as np
import torch

from . import cabi, mesh
from ._lib import check, lib, make_args

_f32 = np.float32


def _net_struct(net):
    with torch.no_grad():
        return net._net(net.params_, net.decoder_)


def sdf_init_gs(net_struct, x, delta, bce_isigma, quaternion, grad=None, curv_dom=None, opacity=None, n_live=None, ws=None):
    """Raw gssdf_sdf_init_gs on caller-allocated outputs (x [n,3], quaternion [n,4], grad / curv_dom [n,3], opacity [n])."""
    n = x.shape[0]
    ws = ws or cabi.Workspace(x.device)
    w = ws.get(lib().gssdf_sdf_init_gs_workspace_bytes(n))
    a = make_args("gssdf_sdf_init_gs_args", n=n, x=x, n_live=n_live, delta=float(delta), bce_isigma=float(bce_isigma), grad=grad,
                  curv_dom=curv_dom, quaternion=quaternion, opacity=opacity, workspace=w, workspace_bytes=w.numel())
    a.net = net_struct
    check(lib().gssdf_sdf_init_gs(C.byref(a), cabi._stream()))


def rot6d_to_quat(a1, a2, quaternion=None, n_live=None):
    """utils::rotation_6d_to_matrix(cat(a1, a2)) (include/utils/utils.cpp:693-719), columns [b2, b3, b1], then the reference's rotation ->
    quaternion with nan_to_num (neural_gaussian.cpp:367-392). a1, a2: CUDA float32 [n,3]. Returns quaternion [n,4] (w, x, y, z)."""
    a1 = cabi._req(a1, torch.float32, "a1")
    a2 = cabi._req(a2, torch.float32, "a2")
    if a1.shape != a2.shape or a1.dim() != 2 or a1.shape[1] != 3:
        raise ValueError(f"gssdf_b200: a1 and a2 must both be [n,3], got {tuple(a1.shape)} and {tuple(a2.shape)}")
    if quaternion is None:
        quaternion = torch.empty(a1.shape[0], 4, dtype=torch.float32, device=a1.device)
    a = make_args("gssdf_rot6d_to_quat_args", n=a1.shape[0], a1=a1, a2=a2, n_live=n_live, quaternion=quaternion)
    check(lib().gssdf_rot6d_to_quat(C.byref(a), cabi._stream()))
    return quaternion


def init_gs_with_sdf(net, xyzs, mesh_res, init_opa=True):
    """init_gs_with_sdf(local_map, xyzs, mesh_res, init_opa) (neural_gaussian.cpp:19-127). net: sdf.SdfNet (its bce_isigma is
    k_bce_isigma); xyzs: CUDA float32 [n,3] world points. Returns the reference's dict: quaternion [n,4], grad [n,3] (6-offset central
    difference with delta = mesh_res), curv_dom [n,3] (numerical Hessian diagonal) and, when init_opa, opacity [n] = exp(-sdf^2 isigma).
    The reference's k_vis_batch_pt_num batching does not change any value and is not repeated."""
    x = cabi._req(xyzs, torch.float32, "xyzs")
    if x.dim() != 2 or x.shape[1] != 3:
        raise ValueError(f"gssdf_b200: xyzs must be [n,3], got {tuple(x.shape)}")
    n, dev = x.shape[0], x.device
    out = {"quaternion": torch.empty(n, 4, dtype=torch.float32, device=dev),
           "grad": torch.empty(n, 3, dtype=torch.float32, device=dev),
           "curv_dom": torch.empty(n, 3, dtype=torch.float32, device=dev)}
    if init_opa:
        out["opacity"] = torch.empty(n, dtype=torch.float32, device=dev)
    sdf_init_gs(_net_struct(net), x, float(_f32(mesh_res)), float(_f32(net.bce_isigma)), out["quaternion"], out["grad"], out["curv_dom"],
                out.get("opacity"))
    return out


def anchor_indices(n_vertices, vis_batch_pt_num):
    """The reference's stride rule (neural_gaussian.cpp:302-306): with more than k_vis_batch_pt_num vertices, step = max(V //
    k_vis_batch_pt_num, 1) and slice(0, 0, -1, step) -- which stops before the LAST vertex. Returns a Python range."""
    if n_vertices > vis_batch_pt_num:
        step = max(n_vertices // vis_batch_pt_num, 1)
        return range(0, n_vertices - 1, step)
    return range(n_vertices)


def sky_count(spatial_scale):
    """int num_sky_points = 1000 * original_spatial_scale_ (:335-337): the product in fp32, truncated."""
    return int(_f32(_f32(1000) * _f32(spatial_scale)))


def sky_radius(inner_map_size):
    """sphere_radius = 0.6f * k_inner_map_size (:346), fp32."""
    return float(_f32(_f32(0.6) * _f32(inner_map_size)))


def sky_log_scale(inner_map_size, n_sky):
    """log(1.1f * M_PI * r * r / num_sky_points) (:353-356): double arithmetic from the fp32 factors, rounded to fp32 by torch::full."""
    r = sky_radius(inner_map_size)
    return float(_f32(math.log(float(_f32(1.1)) * math.pi * r * r / n_sky)))


def anchor_log_scale(mesh_res):
    """log(mesh_res) of torch::full({n, 3}, log(mesh_res)) (:309-311), as an fp32 value."""
    return float(_f32(math.log(float(_f32(mesh_res)))))


def neural_gs_init(tree, net, margin_box, leaf_size, *, vis_batch_pt_num, sh_degree, spatial_scale, inner_map_size, map_origin, sky=True,
                   generator=None, geo_init=True, cpu_generator=None):
    """The tensors NeuralGS::NeuralGS builds on its `k_mesh_init && sdf_enable && k_geo_init` branch (neural_gaussian.cpp:293-424), in the
    reference's order:
      1. mesh.meshing(tree, net, *margin_box, 0.5 * leaf_size) -- its vertices are already the unique(faces) set (DESIGN 7f);
      2. anchors = the vertices strided by `anchor_indices` (the last vertex is excluded when striding, as in the reference);
         scaling = log(mesh_res);
      3. quaternion / opacity from gssdf_sdf_init_gs (init_opa = true); with geo_init=False (k_geo_init = 0) random_quat on
         `cpu_generator` and opacity logit(0.1) instead;
      4. sky (k_sky_init): int(1000 * spatial_scale) points randn -> normalize(eps 1e-6) -> * 0.6 inner_map_size + map_origin, scale
         log(1.1 pi r^2 / n), quaternions from gssdf_rot6d_to_quat(samples, samples[:, (1, 2, 0)]), opacity logit(1) = +inf;
      5. offsets = 0, features_dc = rand [N,1,3], features_rest = 0 [N, (sh_degree+1)^2 - 1, 3];
      6. rows with a NaN in anchors / scaling / quaternion / opacity are dropped (isnan only: the +inf sky opacities stay).
    Random draws come from `generator` (on the net's device) in the reference's order: the sky randn, then the features_dc rand.
    As in the reference, `opacity` holds exp(-sdf^2 isigma) as the PRE-sigmoid parameter (get_opacity applies sigmoid, :471-478).
    Setting k_far (= 2 r) and saving the `gs_` mesh stay with the caller.
    Returns (dict of anchors, offsets, quaternion, scaling, opacity, features_dc, features_rest -- the order GsSdfTrainer.load takes --,
    number of dropped NaN rows)."""
    mesh_res = float(_f32(_f32(0.5) * _f32(leaf_size)))
    v, _, _ = mesh.meshing(tree, net, margin_box[0], margin_box[1], mesh_res)
    dev = v.device
    idx = anchor_indices(v.shape[0], vis_batch_pt_num)
    anchors = v[idx.start:idx.stop:idx.step].contiguous() if len(idx) else v[:0]
    scaling = torch.full((anchors.shape[0], 3), anchor_log_scale(mesh_res), dtype=torch.float32, device=dev)
    quaternion, opacity = _orientation(net if geo_init else None, anchors, mesh_res, cpu_generator)
    if sky:
        anchors, scaling, quaternion, opacity = append_sky(anchors, scaling, quaternion, opacity, spatial_scale, inner_map_size, map_origin,
                                                           generator)
    return finish_rows(anchors, scaling, quaternion, opacity, sh_degree, generator)


def _orientation(net, anchors, mesh_res, cpu_generator):
    """quaternion and opacity of NeuralGS::NeuralGS (neural_gaussian.cpp:321-333): from gssdf_sdf_init_gs with init_opa when the SDF is
    enabled and k_geo_init is set (net given), else random_quat on the CPU generator and logit(0.1f)."""
    if net is not None:
        r = init_gs_with_sdf(net, anchors, mesh_res, True)
        return r["quaternion"], r["opacity"]
    n, dev = anchors.shape[0], anchors.device
    return random_quat(n, cpu_generator).to(dev), torch.logit(0.1 * torch.ones(n, dtype=torch.float32, device=dev))


def append_sky(anchors, scaling, quaternion, opacity, spatial_scale, inner_map_size, map_origin, generator=None):
    """Step 4 of neural_gs_init (k_sky_init, neural_gaussian.cpp:335-401): int(1000 * spatial_scale) points randn (from `generator`) ->
    normalize(eps 1e-6) -> * 0.6 inner_map_size + map_origin, scale log(1.1 pi r^2 / n), quaternions from gssdf_rot6d_to_quat(samples,
    samples[:, (1, 2, 0)]), opacity logit(1) = +inf; appended after the given rows. Returns (anchors, scaling, quaternion, opacity)."""
    dev = anchors.device
    n_sky = sky_count(spatial_scale)
    radius = sky_radius(inner_map_size)
    samples = torch.randn(n_sky, 3, dtype=torch.float32, device=dev, generator=generator)
    samples = torch.nn.functional.normalize(samples, dim=-1, eps=1e-6)
    origin = torch.as_tensor(np.asarray(map_origin, np.float32).reshape(1, 3), device=dev)
    sky_anchor = samples * radius + origin
    sky_scale = torch.full((n_sky, 3), sky_log_scale(inner_map_size, n_sky), dtype=torch.float32, device=dev)
    sky_quat = rot6d_to_quat(samples, samples[:, [1, 2, 0]].contiguous())
    sky_opacity = torch.logit(torch.ones(n_sky, dtype=torch.float32, device=dev))
    return (torch.cat([anchors, sky_anchor], 0), torch.cat([scaling, sky_scale], 0), torch.cat([quaternion, sky_quat], 0),
            torch.cat([opacity, sky_opacity], 0))


def knn3_mean_dist2(points, out, ws=None):
    """Raw gssdf_knn3_mean_dist2 on a caller-allocated output (points CUDA float32 [n,3] contiguous, out float32 [n])."""
    n = points.shape[0]
    ws = ws or cabi.Workspace(points.device)
    w = ws.get(lib().gssdf_knn3_mean_dist2_workspace_bytes(n))
    a = make_args("gssdf_knn3_mean_dist2_args", n=n, points=points, out=out, workspace=w, workspace_bytes=w.numel())
    check(lib().gssdf_knn3_mean_dist2(C.byref(a), cabi._stream()))
    return out


def dist_cuda2(points, ws=None):
    """simple-knn's distCUDA2(points) (submodules/simple-knn/spatial.cu): for each point the mean of its three smallest squared distances
    to the other points, float32 [P] on the points' device (include/gssdf_b200.h f-10, DESIGN 7k). points: CUDA float32 [P,3], made
    contiguous as the reference does."""
    if not isinstance(points, torch.Tensor) or points.dim() != 2 or points.shape[1] != 3:
        raise ValueError(f"gssdf_b200: points must be a [P,3] tensor, got {tuple(getattr(points, 'shape', ()))}")
    x = cabi._req(points.contiguous(), torch.float32, "points")
    return knn3_mean_dist2(x, torch.empty(x.shape[0], dtype=torch.float32, device=x.device), ws)


def init_point_indices(n_points):
    """The reference's stride of the depth cloud before NeuralGS (neural_mapping.cpp:843-848): step = int(N / 1e6f) in fp32 (N rounded
    to fp32 first), at least 1, and slice(0, 0, -1, step) -- which always stops before the LAST point. Returns a Python range."""
    step = max(int(_f32(_f32(n_points) / _f32(1e6))), 1)
    return range(0, max(n_points - 1, 0), step)


def random_quat(n, cpu_generator=None):
    """random_quat_tensor(N) (include/neural_gaussian/gauss_utils.hpp:32-46): u, v, w = three torch.rand(N) draws from the CPU generator,
    q = (sqrt(1 - u) sin(2 pi v), sqrt(1 - u) cos(2 pi v), sqrt(u) sin(2 pi w), sqrt(u) cos(2 pi w)) in fp32 (2 pi rounded to fp32 by
    ATen's scalar multiply). Returns a CPU float32 [n,4] tensor; NeuralGS moves it to the device."""
    u = torch.rand(n, generator=cpu_generator)
    v = torch.rand(n, generator=cpu_generator)
    w = torch.rand(n, generator=cpu_generator)
    return torch.stack([torch.sqrt(1 - u) * torch.sin(2 * math.pi * v), torch.sqrt(1 - u) * torch.cos(2 * math.pi * v),
                        torch.sqrt(u) * torch.sin(2 * math.pi * w), torch.sqrt(u) * torch.cos(2 * math.pi * w)], -1)


def neural_gs_init_points(points, *, net=None, leaf_size, geo_init=True, sh_degree, spatial_scale, inner_map_size, map_origin, sky=True,
                          generator=None, cpu_generator=None):
    """The tensors NeuralGS::NeuralGS builds when it starts from points rather than from the SDF mesh (k_mesh_init = 0 or the SDF
    disabled; neural_gaussian.cpp:312-424), in the reference's order:
      1. anchors = points (the caller's depth cloud, strided by `init_point_indices` in the reference's trainer);
         scaling = log(sqrt(clamp_min(dist_cuda2(points), 1e-6))) repeated over the three axes;
      2. with an SDF (`net`) and geo_init: quaternion / opacity from gssdf_sdf_init_gs at delta 0.5 * leaf_size (init_opa = true);
         otherwise random_quat(n, cpu_generator) and opacity logit(0.1);
      3. the sky (k_sky_init), features and NaN-row filter exactly as neural_gs_init (append_sky, finish_rows).
    Random draws in the reference's order: the CPU u, v, w of random_quat, then `generator`'s sky randn and features_dc rand.
    Returns (dict, number of dropped NaN rows) like neural_gs_init."""
    anchors = cabi._req(points, torch.float32, "points")
    if anchors.dim() != 2 or anchors.shape[1] != 3:
        raise ValueError(f"gssdf_b200: points must be [n,3], got {tuple(anchors.shape)}")
    dist2 = torch.clamp_min(dist_cuda2(anchors), 1e-6)
    scaling = torch.log(torch.sqrt(dist2)).unsqueeze(-1).repeat(1, 3)
    mesh_res = float(_f32(_f32(0.5) * _f32(leaf_size)))
    quaternion, opacity = _orientation(net if geo_init else None, anchors, mesh_res, cpu_generator)
    if sky:
        anchors, scaling, quaternion, opacity = append_sky(anchors, scaling, quaternion, opacity, spatial_scale, inner_map_size, map_origin,
                                                           generator)
    return finish_rows(anchors, scaling, quaternion, opacity, sh_degree, generator)


def finish_rows(anchors, scaling, quaternion, opacity, sh_degree, generator=None):
    """Steps 5 and 6 of neural_gs_init (neural_gaussian.cpp:403-424): features_dc = rand [N,1,3] drawn for ALL rows, features_rest = 0,
    then the rows with a NaN in anchors / scaling / quaternion / opacity are dropped (isnan only). Returns (dict, number dropped)."""
    n, dev = anchors.shape[0], anchors.device
    features_dc = torch.rand(n, 1, 3, dtype=torch.float32, device=dev, generator=generator)
    features_rest = torch.zeros(n, (sh_degree + 1) ** 2 - 1, 3, dtype=torch.float32, device=dev)
    is_nan = anchors.isnan().any(-1) | scaling.isnan().any(-1) | quaternion.isnan().any(-1) | opacity.isnan()
    num_nan = int(is_nan.sum())
    if num_nan > 0:
        keep = (~is_nan).nonzero().squeeze(1)
        anchors, scaling, quaternion, opacity, features_dc, features_rest = (
            t.index_select(0, keep).contiguous() for t in (anchors, scaling, quaternion, opacity, features_dc, features_rest))
    # the reference leaves offsets_ at the unfiltered row count (:405, never index_selected); here it has the kept rows' size
    out = {"anchors": anchors, "offsets": torch.zeros(anchors.shape[0], 3, dtype=torch.float32, device=dev), "quaternion": quaternion,
           "scaling": scaling, "opacity": opacity, "features_dc": features_dc, "features_rest": features_rest}
    return out, num_nan
