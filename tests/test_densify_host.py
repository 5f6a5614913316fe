"""CPU checks of the densification arbiter (tests/densify_oracle.py) and its scenes (tests/densify_scenes.py).

- The arbiter agrees with a float64 torch transcription of the reference's strategy functions (neural_gaussian.cpp: update_state,
  grow_gs = duplicate + split, prune_gs, prune_invisible_gs, prune_nan_gs, reset_opacity, with optimizer_utils.cpp's moment handling).
- Every scene populates every flag bit and every decision clears its threshold by MARGIN.
- Sensitivity: each one-line kernel mistake of densify_oracle.MUTATIONS moves some output of the GPU tests' scenes beyond the GPU bar."""
import numpy as np
import pytest

import densify_oracle as A
import densify_scenes as S

torch = pytest.importorskip("torch")
f64 = torch.float64


def _quat_to_rotmat(q):  # utils::normalized_quat_to_rotmat
    w, x, y, z = q.unbind(-1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                        2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                        2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1).view(-1, 3, 3)


class RefGS:
    """The reference's parameter tensors, Adam moments and state in float64 torch, surgery as neural_gaussian.cpp writes it."""
    SEG = dict(offsets=(0, 3), quaternion=(3, 7), scaling=(7, 10), opacity=(10, 11), features_dc=(11, 14), features_rest=(14, None))

    def __init__(self, snap):
        t = lambda a: torch.tensor(np.asarray(a), dtype=f64)
        self.P = {k: t(snap["P"][:, a:b]) for k, (a, b) in self.SEG.items()}
        self.M = {k: t(snap["M"][:, a:b]) for k, (a, b) in self.SEG.items()}
        self.V = {k: t(snap["V"][:, a:b]) for k, (a, b) in self.SEG.items()}
        self.anchors, self.state = t(snap["anchors"]), {k: t(v) for k, v in snap["state"].items()}

    def rows(self, d):
        return torch.cat([d[k] for k in self.SEG], 1).numpy()

    def _sel(self, idx, ext=None):  # prune_optimizer / prune_cat_tensors_to_optimizer: zeros appended to both moments
        for k in self.SEG:
            e = ext[k] if ext else self.P[k][:0]
            self.P[k] = torch.cat([self.P[k][idx], e])
            self.M[k] = torch.cat([self.M[k][idx], torch.zeros_like(e)])
            self.V[k] = torch.cat([self.V[k][idx], torch.zeros_like(e)])

    def update_state(self, gid, v, vis, radii, W, H, n_cameras):
        grads = torch.tensor(v, dtype=f64).clone()
        gid = torch.tensor(gid)
        grads[:, 0] = grads[:, 0] * W * 0.5 * n_cameras
        grads[:, 1] = grads[:, 1] * H * 0.5 * n_cameras
        st = self.state
        st["grad2d"].index_add_(0, gid, grads.norm(2, -1))
        st["count"].index_add_(0, gid, torch.ones(len(gid), dtype=f64))
        r = torch.tensor(radii, dtype=f64).max(-1).values / float(max(W, H))
        vis = torch.tensor(vis, dtype=f64)
        # the reference's index_put_(maximum(index_select)) keeps one unspecified write per id that several cameras saw; the kernel's
        # atomic max keeps the largest, which is the running maximum written out here
        for i in range(len(gid)):
            st["vis"][gid[i]] = torch.maximum(st["vis"][gid[i]], vis[i])
            st["radii"][gid[i]] = torch.maximum(st["radii"][gid[i]], r[i])

    def grow(self, c, it, randn):
        st = self.state
        grads = st["grad2d"] / st["count"].clamp_min(1)
        high = grads > c["grow_grad2d"]
        scale = torch.exp(self.P["scaling"])[:, :2]
        small = scale.max(-1).values <= c["grow_scale3d"] * c["spatial_scale"]
        is_dupli, is_split = high & small, high & ~small
        if it < c["scale2d_stop"]:
            is_split |= st["radii"] > c["grow_scale2d"]
        di = is_dupli.nonzero().flatten()
        if len(di):  # duplicate
            self.anchors = torch.cat([self.anchors, self.anchors[di]])
            self._sel(torch.arange(len(is_dupli)), {k: self.P[k][di] for k in self.SEG})
            for k in st:
                st[k] = torch.cat([st[k], st[k][di]])
        is_split = torch.cat([is_split, torch.zeros(len(di), dtype=torch.bool)])
        sel, rest = is_split.nonzero().flatten(), (~is_split).nonzero().flatten()
        ns, K = len(sel), 2
        if ns:  # split
            scales = torch.exp(self.P["scaling"][sel])
            scales = torch.cat([scales[:, :2], torch.zeros(ns, 1, dtype=f64)], 1)
            sample_scales = scales.unsqueeze(0) * torch.tensor(randn, dtype=f64).view(K, ns, 3)
            quats = torch.nn.functional.normalize(self.P["quaternion"][sel], dim=-1)
            off = (torch.einsum("nij,nj,bnj->bni", _quat_to_rotmat(quats), scales, sample_scales) + self.P["offsets"][sel].unsqueeze(0)).reshape(-1, 3)
            ext = {k: self.P[k][sel].repeat(K, 1) for k in self.SEG}
            ext["offsets"], ext["scaling"] = off, torch.log(scales / float(np.float32(1.6))).repeat(K, 1)
            self.anchors = torch.cat([self.anchors[rest], self.anchors[sel].repeat(K, 1)])
            self._sel(rest, ext)
            for k in st:
                st[k] = torch.cat([st[k][rest], st[k][sel].repeat(K)])
        return len(di), ns

    def prune(self, is_prune):
        valid = (~is_prune).nonzero().flatten()
        self.anchors = self.anchors[valid]
        self._sel(valid)
        for k in self.state:
            self.state[k] = self.state[k][valid]

    def prune_gs(self, c, it, reset_every):
        scale = torch.exp(self.P["scaling"])[:, :2]
        is_prune = (torch.sigmoid(self.P["opacity"][:, 0]) < c["prune_opa"]) | (scale.min(-1).values < float(np.float32(1e-4)))
        if it > reset_every:
            is_prune |= scale.max(-1).values > c["prune_scale3d"] * c["spatial_scale"]
        self.prune(is_prune)

    def prune_nan_gs(self):
        self.prune(self.P["offsets"].isnan().any(-1) | self.P["scaling"].isnan().any(-1) | self.P["quaternion"].isnan().any(-1))

    def prune_invisible_gs(self, it, num_train_data):
        if it > 0 and it % num_train_data == 0:
            is_prune = self.state["vis"] < float(np.float32(1e-4))
            self.state["vis"].zero_()
            self.prune(is_prune)

    def reset_opacity(self, prune_opa):
        cap = float(np.float32(np.log(2 * prune_opa / (1 - 2 * prune_opa))))
        self.P["opacity"] = self.P["opacity"].clamp_max(cap)
        self.M["opacity"].zero_()
        self.V["opacity"].zero_()


def _f32cfg(it_stop=4000):
    c = {k: float(np.float32(v)) for k, v in S.CFG.items()}
    c["scale2d_stop"] = it_stop
    return c


def _assert_snap(got, ref, tag):
    for key, d in (("P", ref.P), ("M", ref.M), ("V", ref.V)):
        np.testing.assert_allclose(got[key], ref.rows(d), rtol=1e-12, atol=1e-14, err_msg=f"{tag} {key}")
    np.testing.assert_array_equal(got["anchors"], ref.anchors.numpy(), err_msg=tag)
    for k in A.STATE_NAMES:
        np.testing.assert_array_equal(got["state"][k], ref.state[k].numpy(), err_msg=f"{tag} state {k}")


@pytest.mark.parametrize("K", [1, 16])
def test_arbiter_matches_reference_transcription(K):
    """update_state with three cameras, then the Densifier's event order: prune_nan_gs, grow_gs, prune_gs past reset_every,
    prune_invisible_gs, reset_opacity."""
    sc = S.flag_scene(600, K, seed=K)
    N, rng = 600, np.random.default_rng(K)
    st = {k: np.zeros(N) for k in A.STATE_NAMES}
    inp = S.render_inputs(N, 3, 1200, 680, seed=K)
    want, _ = A.update_state(st, inp["gid"], inp["v"], inp["vis"], inp["radii"], 1200, 680, 3)
    snap = A.snapshot(sc["rows"], rng.normal(size=sc["rows"].shape), rng.uniform(size=sc["rows"].shape), rng.normal(size=(N, 3)), st)
    ref = RefGS(snap)
    ref.update_state(inp["gid"], inp["v"], inp["vis"], inp["radii"], 1200, 680, 3)
    for k in A.STATE_NAMES:  # the arbiter's radii are the kernel's correctly rounded fp32 quotient
        np.testing.assert_allclose(want[k], ref.state[k].numpy(), rtol=A.U if k == "radii" else 1e-13, atol=0, err_msg=k)
    # the designed statistics drive the events (their margins are nudged; the random render inputs' are not)
    snap["state"] = {k: np.asarray(sc[k], np.float64) for k in A.STATE_NAMES}
    ref = RefGS(snap)
    c, it = _f32cfg(), 3100
    snap = A.prune_nan_gs(snap, A.event_flags(snap, c, it, False)[0])
    ref.prune_nan_gs()
    _assert_snap(snap, ref, "prune_nan_gs")
    f = A.event_flags(snap, c, it, True)[0]
    ns = int(((f & A.SPLIT) != 0).sum())
    randn = rng.normal(size=(2 * ns, 3))
    snap, nd, ns2 = A.grow_gs(snap, f, randn)
    assert ref.grow(c, it, randn) == (nd, ns2) and nd > 10 and ns2 > 10
    _assert_snap(snap, ref, "grow_gs")
    snap = A.prune_gs(snap, A.event_flags(snap, c, it, False)[0], it, 3000)
    ref.prune_gs(c, it, 3000)
    _assert_snap(snap, ref, "prune_gs")
    snap = A.prune_invisible_gs(snap, A.event_flags(snap, c, it, False)[0], it, 50)
    ref.prune_invisible_gs(it, 50)
    _assert_snap(snap, ref, "prune_invisible_gs")
    snap = A.reset_opacity(snap, c["prune_opa"])
    ref.reset_opacity(c["prune_opa"])
    _assert_snap(snap, ref, "reset_opacity")


@pytest.mark.parametrize("K", S.KS)
@pytest.mark.parametrize("N", S.NS)
def test_scenes_populate_every_flag_and_clear_margins(N, K):
    sc = S.flag_scene(N, K, seed=N + 3)
    c = S.CFG
    f, m = A.flags(sc["rows"], sc["grad2d"], sc["count"], sc["vis"], sc["radii"], c["grow_grad2d"], c["grow_scale3d"], c["grow_scale2d"], True,
                   c["prune_opa"], c["prune_scale3d"])
    assert all(float(v.min()) >= S.MARGIN for v in m.values())
    if N >= len(S.CLASSES):
        assert int(np.bitwise_or.reduce(f)) == 127
        for j in range(10):  # each NaN column on its own
            assert (f[sc["cls"] == f"nan_{j}"] & A.P_NAN).all()
        assert ((f[sc["cls"] == "split_2d"] & A.SPLIT) != 0).all()
        assert (f[sc["cls"] == "split_prune"] & (A.SPLIT | A.P_OPA) == (A.SPLIT | A.P_OPA)).all()


def test_trainer_scenes_clear_margins():
    for deg in (0, 3):
        sc = S.trainer_scene(3000, (deg + 1) ** 2, 160, 96, seed=deg + 5)
        assert set(sc["cls"]) == set(S.CLASSES)


def _outputs(mut):
    """every output the GPU tests compare, with its scale, on a few of their cases"""
    out = []
    for N, C in ((257, 3),):
        inp = S.render_inputs(N, C, 1200, 680, seed=N + 10 * C)
        st0 = {k: np.zeros(N, np.float32) for k in A.STATE_NAMES}
        w, s = A.update_state(st0, inp["gid"], inp["v"], inp["vis"], inp["radii"], 1200, 680, C, mut)
        out += [(w[k], s[k]) for k in A.STATE_NAMES]
    sc = S.flag_scene(257, 1, seed=260)
    c = S.CFG
    for grow, use2d in ((True, True), (True, False), (False, False)):
        f, _ = A.flags(sc["rows"], sc["grad2d"] if grow else None, sc["count"] if grow else None, sc["vis"], sc["radii"], c["grow_grad2d"],
                       c["grow_scale3d"], c["grow_scale2d"], use2d, c["prune_opa"], c["prune_scale3d"], mut)
        out.append((f, 0.0))
    for K, N, so, sn, n_new, n_state in ((1, 255, 255, 300, 300, 1), (4, 255, 255, 300, 300, 1), (16, 257, 300, 520, 514, 3)):
        case = S.remap_case(S.flag_scene(N, K, seed=K * 100 + N), so, sn, n_new, n_state, seed=N + K)
        w, s = A.remap(K, so, sn, n_new, case["src"], case["mode"], case["randn_row"], case["randn"], case["old"], case["new"],
                       case["states_old"], case["states_new"], mut)
        out += [(w["params"], s), (w["exp_avg"], 0.0), (w["exp_avg_sq"], 0.0), (w["anchors"], 0.0)] + [(x, 0.0) for x in w["states"]]
    return out


def test_every_mutation_moves_an_output_beyond_the_gpu_bar():
    base = _outputs(())
    for mut in A.MUTATIONS:
        moved = sum(int(A.off_bar(m[0], b[0], b[1]).sum()) for m, b in zip(_outputs(mut), base))
        assert moved > 0, f"{mut[0]} moves no output beyond the GPU bar"
