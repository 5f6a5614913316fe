"""f-6 splat initialisation from the trained SDF over the C ABI (DESIGN 7g).

`init_gs_with_sdf` is the reference's init_gs_with_sdf (include/neural_gaussian/neural_gaussian.cpp:19-127) as one gssdf_sdf_init_gs call;
`neural_gs_init` is the tensor part of NeuralGS::NeuralGS's `mesh_init && sdf_enable && geo_init` branch (:273-424): mesh the SDF, stride
the vertices down to the anchors, orient them from the SDF, append the sky sphere, draw the colours and drop NaN rows. The library never
syncs or allocates; `neural_gs_init` reads the mesh counts and the NaN count back once each, like the reference."""
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
                   generator=None):
    """The tensors NeuralGS::NeuralGS builds on its `k_mesh_init && sdf_enable && k_geo_init` branch (neural_gaussian.cpp:293-424), in the
    reference's order:
      1. mesh.meshing(tree, net, *margin_box, 0.5 * leaf_size) -- its vertices are already the unique(faces) set (DESIGN 7f);
      2. anchors = the vertices strided by `anchor_indices` (the last vertex is excluded when striding, as in the reference);
         scaling = log(mesh_res);
      3. quaternion / opacity from gssdf_sdf_init_gs (init_opa = true);
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
    r = init_gs_with_sdf(net, anchors, mesh_res, True)
    quaternion, opacity = r["quaternion"], r["opacity"]
    if sky:
        n_sky = sky_count(spatial_scale)
        radius = sky_radius(inner_map_size)
        samples = torch.randn(n_sky, 3, dtype=torch.float32, device=dev, generator=generator)
        samples = torch.nn.functional.normalize(samples, dim=-1, eps=1e-6)
        origin = torch.as_tensor(np.asarray(map_origin, np.float32).reshape(1, 3), device=dev)
        sky_anchor = samples * radius + origin
        sky_scale = torch.full((n_sky, 3), sky_log_scale(inner_map_size, n_sky), dtype=torch.float32, device=dev)
        sky_quat = rot6d_to_quat(samples, samples[:, [1, 2, 0]].contiguous())
        sky_opacity = torch.logit(torch.ones(n_sky, dtype=torch.float32, device=dev))
        anchors = torch.cat([anchors, sky_anchor], 0)
        scaling = torch.cat([scaling, sky_scale], 0)
        quaternion = torch.cat([quaternion, sky_quat], 0)
        opacity = torch.cat([opacity, sky_opacity], 0)
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
