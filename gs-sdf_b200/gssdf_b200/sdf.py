"""Host-side mirror of the SDF operator surface (LocalMap / EncodingMap / TCNNEncoding) over the C ABI.

Reference (paths relative to /root/reference):
  TCNNEncoding(n_in, cfg, name, seed) / .forward(x) / .params_ / .get_out_dim()
                                          submodules/tcnn_binding/tcnn_binding/tcnn_binding.h:16-105
  LocalMap::get_sdf(xyz) -> {sdf, isigma}  include/neural_net/local_map.cpp:87-103
  LocalMap::get_gradient(xyz, delta, ..., numerical) include/neural_net/local_map.cpp:105-173 (numerical branch)
  NeuralSLAM::sdf_train_callback's outlier branch  include/neural_mapping/neural_mapping.cpp:559-592 (remove_outliers)
`params_` stays a flat fp32 [n_params] torch parameter (checkpoint layout of torch::save(local_map_ptr)).
All compute is in libgssdf_b200.so; autograd is plumbing.
"""
import ctypes
import ctypes.util
import math

import numpy as np
import torch

from . import cabi


class _SdfFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xyz, table, mlp, mod):
        n = xyz.shape[0]
        sdf = torch.empty(n, device=xyz.device)
        y1 = torch.empty(n, device=xyz.device)
        net = mod._net(table, mlp)
        cabi.sdf_fwd(net, xyz, sdf, y1)
        ctx.save_for_backward(xyz, table, mlp)
        ctx.mod = mod
        return sdf, y1

    @staticmethod
    def backward(ctx, v_sdf, v_y1):
        xyz, table, mlp = ctx.saved_tensors
        mod = ctx.mod
        n = xyz.shape[0]
        z = lambda t: torch.zeros(n, device=xyz.device) if t is None else t.contiguous()
        need_x, need_t, need_m = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        v_x = torch.empty(n, 3, device=xyz.device) if need_x else None
        tg = torch.zeros_like(table) if need_t else None
        mg = torch.zeros_like(mlp) if need_m else None
        cabi.sdf_bwd(mod._net(table, mlp), xyz, z(v_sdf), z(v_y1), tg, mg, v_x)
        return v_x, tg, mg, None


class SdfNet(torch.nn.Module):
    """EncodingMap (hash grid, tcnn fp16 semantics) + LocalMap decoder (Linear/ReLU) evaluated by the fused kernels."""

    def __init__(self, device, n_levels=16, n_features=2, log2_hashmap_size=19, base_resolution=32, per_level_scale=2.0,
                 hidden_dim=64, geo_num_layer=3, origin=(0.0, 0.0, 0.0), map_size=0.0, bce_isigma=1.0, seed=1337, mlp_mode=None):
        super().__init__()
        self.cfg = dict(n_levels=n_levels, n_features=n_features, log2_hashmap_size=log2_hashmap_size, base_resolution=base_resolution,
                        per_level_scale=per_level_scale, hidden_dim=hidden_dim, n_hidden=geo_num_layer)
        self.origin, self.inv_size = tuple(float(o) for o in origin), (1.0 / map_size if map_size else 0.0)
        self.bce_isigma = bce_isigma
        probe = cabi.sdf_net(torch.zeros(1, device=device), torch.zeros(1, device=device), **self.cfg)
        n_table, n_mlp = cabi.sdf_table_params(probe), cabi.sdf_mlp_params(probe)
        g = torch.Generator(device="cpu").manual_seed(seed)
        # tcnn grid init U(-1e-4, 1e-4) (grid.h:1059-1062); torch::nn::Linear default (kaiming_uniform(a=sqrt(5)))
        self.params_ = torch.nn.Parameter(((torch.rand(n_table, generator=g) * 2 - 1) * 1e-4).to(device))
        chunks = []
        in_dim = n_levels * n_features
        dims = [in_dim] + [hidden_dim] * (1 + geo_num_layer) + [2]
        for k, o in zip(dims[:-1], dims[1:]):
            bound = 1.0 / math.sqrt(k)
            chunks += [(torch.rand(o * k, generator=g) * 2 - 1) * bound, (torch.rand(o, generator=g) * 2 - 1) * bound]
        self.decoder_ = torch.nn.Parameter(torch.cat(chunks).to(device))
        assert self.decoder_.numel() == n_mlp
        self._half = torch.empty(n_table, dtype=torch.float16, device=device)
        self._half_version = None
        # decoder arithmetic: wgmma tensor cores where supported (hidden 64, <= 3 hidden->hidden layers), else fp32 CUDA cores
        self.mlp_mode = (1 if hidden_dim == 64 and geo_num_layer <= 3 else 0) if mlp_mode is None else int(mlp_mode)
        self._packed = torch.empty(cabi.sdf_mlp_packed_bytes(probe), dtype=torch.uint8, device=device) if self.mlp_mode == 1 else None
        self._packed_version = None

    def get_out_dim(self):
        return self.cfg["n_levels"] * self.cfg["n_features"]

    def refresh_half(self):
        """fp32 master -> fp16 shadow; call after every optimiser step (the reference re-casts on every forward)."""
        cabi.sdf_table_to_half(self.params_.detach(), self._half)
        self._half_version = self.params_._version

    def _net(self, table, mlp):
        if self._half_version != self.params_._version:
            self.refresh_half()
        if self.mlp_mode == 1 and self._packed_version != self.decoder_._version:
            cabi.sdf_mlp_pack(cabi.sdf_net(self._half, mlp.detach(), **self.cfg), self._packed)
            self._packed_version = self.decoder_._version
        return cabi.sdf_net(self._half, mlp.detach(), origin=self.origin, inv_size=self.inv_size, mlp_mode=self.mlp_mode,
                            mlp_packed=self._packed, **self.cfg)

    def get_sdf(self, xyz):
        sdf, y1 = _SdfFunction.apply(xyz.contiguous(), self.params_, self.decoder_, self)
        isigma = 1 + torch.nn.functional.softplus(y1, beta=100) * self.bce_isigma
        return sdf.unsqueeze(-1), isigma.unsqueeze(-1)

    def get_gradient_numerical(self, xyz, delta):
        """LocalMap::get_gradient(_numerical_grad = true), local_map.cpp:110-147 (without the Hessian)."""
        offs = torch.tensor([[delta, 0, 0], [-delta, 0, 0], [0, delta, 0], [0, -delta, 0], [0, 0, delta], [0, 0, -delta]],
                            device=xyz.device, dtype=xyz.dtype).unsqueeze(1)
        pts = (xyz.unsqueeze(0) + offs).view(-1, 3)
        s = self.get_sdf(pts)[0].view(6, xyz.shape[0], 1)
        return 0.5 / delta * torch.cat([s[0] - s[1], s[2] - s[3], s[4] - s[5]], 1)


_libm = None


def _m():
    """The host's libm: the threshold is computed with the same logf / log / exp the reference's C++ calls."""
    global _libm
    if _libm is None:
        L = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
        L.logf.restype, L.logf.argtypes = ctypes.c_float, [ctypes.c_float]
        for fn in (L.log, L.exp):
            fn.restype, fn.argtypes = ctypes.c_double, [ctypes.c_double]
        _libm = L
    return _libm


def outlier_threshold(it, total_it, truncated_dis, outlier_dist):
    """The fp32 threshold of sdf_train_callback's outlier removal (neural_mapping.cpp:542,565-566), one rounding at a time:
    iter_ratio = (float)it / total_it in fp32; exp(logf(truncated_dis) * (1 - iter_ratio) + log(outlier_dist) * iter_ratio) with the first
    product in fp32 (k_truncated_dis is a float) and the rest in double; then rounded once to fp32, which is what `tensor < double` compares
    against."""
    f, m = np.float32, _m()
    ratio = f(it) / f(total_it)
    a = f(m.logf(float(f(truncated_dis)))) * (f(1) - ratio)
    return float(f(m.exp(float(a) + m.log(float(outlier_dist)) * float(ratio))))


def outlier_rows(N, vis_batch_pt_num=1_638_400):
    """How many leading rows of an N-row pack the reference's chunk loop can keep. It evaluates rows [i, min(i + B, N - 1)) for
    i = 0, B, 2B, ..., so never the last row. A chunk of exactly one row (B == 1, or the last chunk when (N - 1) % B == 1) keeps nothing:
    `.squeeze()` makes its mask 0-d, and nonzero() of a 0-d True squeezes to an empty index (of a 0-d False to a [0,0] one, which makes
    the reference throw)."""
    n, b = max(N - 1, 0), vis_batch_pt_num
    if b == 1:
        return 0
    return n - 1 if n % b == 1 else n


def remove_outliers(net, pack, it, total_it, *, truncated_dis, outlier_dist, interval, vis_batch_pt_num=1_638_400, ws=None):
    """sdf_train_callback's outlier branch (neural_mapping.cpp:559-592) on a depth pack: a dict of [N, k] tensors with the points under
    "xyz" (e.g. origin, direction, depth, xyz). At it > 0 with it % interval == 0, keeps the rows r < outlier_rows(N, vis_batch_pt_num)
    with |net.get_sdf(xyz[r])| < outlier_threshold(...) in every field, in order: the last row is never evaluated, as in the reference.
    Other iterations return the pack unchanged. Returns (pack, number of rows); the count is read back once.
    A CUDA pack is compacted on the device by gssdf_sdf_outlier_filter (the fields are views of the first rows of new N-row buffers). A CPU
    pack (where the reference keeps it) sends xyz to the device once and index_selects every field on the host with the kept rows.
    Where the reference throws (N == 0, a chunk with exactly one kept row among several), the pack is empty, or the row kept."""
    N = pack["xyz"].shape[0]
    if not (it > 0 and it % interval == 0):
        return pack, N
    thr = outlier_threshold(it, total_it, truncated_dis, outlier_dist)
    n = outlier_rows(N, vis_batch_pt_num)
    dev = net.params_.device
    ws = cabi.Workspace(dev) if ws is None else ws
    n_kept = torch.empty(1, dtype=torch.int64, device=dev)
    ns = net._net(net.params_, net.decoder_)
    xyz = pack["xyz"].reshape(N, 3)
    if xyz.is_cuda:
        out = {k: torch.empty_like(v, memory_format=torch.contiguous_format) for k, v in pack.items()}
        cols = [(v.contiguous(), out[k]) for k, v in pack.items()]
        cabi.sdf_outlier_filter(ns, xyz.contiguous(), thr, cols, n_kept, ws, n=n)
        kept = int(n_kept.item())
        return {k: v[:kept] for k, v in out.items()}, kept
    index = torch.empty(n, dtype=torch.int64, device=dev)
    cabi.sdf_outlier_filter(ns, xyz[:n].to(dev, torch.float32).contiguous(), thr, [], n_kept, ws, index=index, n=n)
    kept = int(n_kept.item())
    idx = index[:kept].cpu()
    return {k: v.index_select(0, idx) for k, v in pack.items()}, kept
