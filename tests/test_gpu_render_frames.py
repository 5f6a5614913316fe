"""The render path on the GPU (DESIGN 7p): gssdf_render_frames_u8 byte for byte against the numpy restatement
(render_frames_oracle.py), views.render_views over a camera spec of mixed resolutions and intrinsics against one-view SplatRenderer
renders, through the intersection-capacity regrowth, against GsTrainer.render after a short box-room run (bck_color 0 and 1), and for a
splat set written to PLY and read back."""
import numpy as np
import pytest
import torch

import render_frames_oracle as O
from gssdf_b200 import io as IO
from gssdf_b200 import render as RD
from gssdf_b200 import scene as S
from gssdf_b200 import views as VW

pytestmark = pytest.mark.gpu


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _outputs(C, W, H, seed):
    """out_colors / out_normals of C views: colours spanning [-0.2, 1.2], depths in (0, 80) m with a share of zero, negative and
    tie-valued depths, and the last view of a batch (of more than one) without any positive depth."""
    rng = np.random.default_rng(seed)
    oc = rng.uniform(-0.2, 1.2, (C, H, W, 4)).astype(np.float32)
    d = rng.uniform(0.01, 12.0, (C, H, W)).astype(np.float32)
    d[rng.random((C, H, W)) < 0.1] = 0.0
    d[rng.random((C, H, W)) < 0.05] *= -1
    far = rng.random((C, H, W)) < 0.02
    d[far] = rng.uniform(60, 80, far.sum())
    tie = rng.random((C, H, W)) < 0.05
    d[tie] = (rng.integers(1, 9000, tie.sum()) + 0.5).astype(np.float32) / np.float32(1000)
    if C > 1:
        d[-1] = np.where(rng.random((H, W)) < 0.5, 0.0, -1.0)
    oc[..., 3] = d
    on = rng.uniform(-1.1, 1.1, (C, H, W, 3)).astype(np.float32)
    return oc, on


@pytest.mark.parametrize("W,H", [(1200, 680), (1920, 1080), (33, 17)])
@pytest.mark.parametrize("C", [1, 8])
def test_frames_kernel_matches_the_oracle(W, H, C):
    dev = _dev()
    oc, on = _outputs(C, W, H, seed=W + C)
    got = VW.render_frames(torch.from_numpy(oc).to(dev), torch.from_numpy(on).to(dev))
    want = O.render_frames(oc, on)
    for name, g, w in zip(("color", "depth", "normal"), got, want):
        g = g.cpu().numpy()
        assert np.array_equal(g, w), f"{name}: {(g != w).any(-1).sum()} pixels differ"
    if C > 1:  # one call of C views equals C calls of one view
        for c in (0, C - 1):
            one = VW.render_frames(torch.from_numpy(oc[c:c + 1]).to(dev), torch.from_numpy(on[c:c + 1]).to(dev))
            for g, o in zip(got, one):
                assert torch.equal(g[c:c + 1], o)


def test_frames_kernel_rejects_bad_arguments():
    dev = _dev()
    oc = torch.zeros(1, 4, 4, 4, device=dev)
    with pytest.raises(ValueError):
        VW.render_frames(oc, torch.zeros(1, 4, 4, 4, device=dev))
    with pytest.raises(ValueError):
        VW.render_frames(oc.double(), torch.zeros(1, 4, 4, 3, device=dev))


def test_frames_workspace_one_byte_short_is_rejected():
    import ctypes as C
    from gssdf_b200._lib import lib, make_args
    dev = _dev()
    oc, on = torch.zeros(2, 17, 33, 4, device=dev), torch.zeros(2, 17, 33, 3, device=dev)
    out = [torch.empty(2, 17, 33, 3, dtype=torch.uint8, device=dev) for _ in range(3)]
    need = lib().gssdf_render_frames_workspace_bytes(2, 33, 17)
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    for nbytes, rc in ((need - 1, -1), (need, 0)):
        a = make_args("gssdf_render_frames_args", C=2, W=33, H=17, out_colors=oc, out_normals=on, color=out[0], depth=out[1],
                      normal=out[2], workspace=ws, workspace_bytes=nbytes)
        assert lib().gssdf_render_frames_u8(C.byref(a), None) == rc
        if rc:
            assert "workspace" in lib().gssdf_last_error().decode()
    assert lib().gssdf_render_frames_workspace_bytes(2, 0, 17) == 0 and lib().gssdf_render_frames_workspace_bytes(-1, 33, 17) == 0


# ---- render_views --------------------------------------------------------------------------------------------------------------------
DEG = 3


def _raw_splats(N, dev, seed=0):
    sc = S.box_scene(N, DEG, seed=seed, scale_mult=6.0)
    op = np.clip(sc["opacities"], 1e-6, 1 - 1e-6)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)
    return dict(anchors=t(sc["means"]), offsets=torch.zeros(N, 3, device=dev), quaternion=t(sc["quats"]), scaling=t(np.log(sc["scales"])),
                opacity=t(np.log(op / (1 - op))), features_dc=t(sc["sh"][:, :1]), features_rest=t(sc["sh"][:, 1:]))


def _spec_cameras(tmp_path, n):
    """A camera spec of n frames in runs of three resolutions (one run longer than a batch), each frame with its own intrinsics."""
    sizes = [(160, 96)] * 5 + [(97, 61)] * 2 + [(200, 120)] * 3 + [(160, 96)] * (n - 10)
    lines = ["# render camera spec, one line per frame"]
    for i, (w, h) in enumerate(sizes[:n]):
        f = 0.55 * w * (1 + 0.03 * i)
        lines.append(f"{w} {h} {f:.3f} {f * 1.01:.3f} {w / 2 - 0.5 + 0.2 * i:.3f} {h / 2 - 0.5 - 0.1 * i:.3f}  # frame {i}")
    p = tmp_path / "spec.txt"
    p.write_text("\n".join(lines) + "\n")
    return VW.load_camera_spec(str(p), n)


def _poses(n):
    V, _ = S.cameras(list(range(n)), 160, 96)
    return torch.linalg.inv(torch.from_numpy(V).double()).float()


def _one_view(sp, pose, cam, bck_color=0):
    """One-view SplatRenderer.forward at the camera, then the oracle."""
    dev = sp["anchors"].device
    W, H, K = cam
    N = sp["anchors"].shape[0]
    R = RD.SplatRenderer(N, (DEG + 1) ** 2, 1, W, H, dev, 64 * N, sh_degree=DEG)
    R.forward(sp["anchors"], sp["quaternion"], sp["scaling"], sp["opacity"], sp["features_dc"], VW.world_to_camera(pose)[None].to(dev),
              K[None].to(dev), raw=dict(offsets=sp["offsets"], sh_rest=sp["features_rest"]), bck_color=bck_color)
    assert R.read_counts()["isect_overflow"] == 0
    return O.render_frames(R.out_colors.cpu().numpy(), R.out_normals.cpu().numpy())


def _check_views(got, sp, poses, cams):
    assert len(got) == len(cams)
    for i, fr in enumerate(got):
        c, d, n = _one_view(sp, poses[i], cams[i])
        W, H, _ = cams[i]
        assert tuple(fr["color"].shape) == (H, W, 3) and fr["color"].dtype == torch.uint8 and not fr["color"].is_cuda
        for name, w in (("color", c[0]), ("depth", d[0]), ("normal", n[0])):
            assert np.array_equal(fr[name].numpy(), w), f"frame {i} ({W}x{H}) {name}"


def test_render_views_over_a_mixed_camera_spec(tmp_path):
    dev = _dev()
    sp = _raw_splats(3000, dev)
    n = 13
    cams, poses = _spec_cameras(tmp_path, n), _poses(n)
    got = list(VW.render_views(sp, poses, cams, sh_degree=DEG, batch=4))
    _check_views(got, sp, poses, cams)


def test_render_views_regrows_the_intersection_capacity(tmp_path, monkeypatch):
    dev = _dev()
    sp = _raw_splats(3000, dev, seed=1)
    n = 10
    cams, poses = _spec_cameras(tmp_path, n), _poses(n)
    monkeypatch.setattr(VW, "ISECT_PER_SPLAT", 0)  # every new renderer starts with a capacity of one intersection
    got = list(VW.render_views(sp, poses, cams, sh_degree=DEG, batch=8))
    _check_views(got, sp, poses, cams)


# ---- after training ----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def trained():
    """Short GsTrainer runs on the box room with bck_color 0 and 1 (the helpers of test_gpu_backgrounds_masks)."""
    _dev()
    import test_gpu_backgrounds_masks as BM
    room = BM._room(False)
    c2w = BM._poses(12, seed=3)
    frames = (c2w, BM._images(c2w))
    S_ = BM._sdf_trainer(room, 200, seed=5)
    out = {}
    for bck in (0, 1):
        G = BM._gs_trainer(room, S_, frames, 40, bck_color=bck)
        G.run()
        out[bck] = G
    return out, c2w, BM._K(), BM.W, BM.H


@pytest.mark.parametrize("bck_color", [0, 1])
def test_render_views_equals_the_trainers_render(trained, bck_color):
    Gs, c2w, K, W, H = trained
    G = Gs[bck_color]
    st = G.state()
    deg = G.T.R.sh_degree
    idx = [0, 5, 11]
    got = list(VW.render_views(st["splats"], c2w[idx], (W, H, K), sh_degree=deg, bck_color=bck_color))
    for k, i in enumerate(idx):
        img = st["render"](VW.world_to_camera(c2w[i]))
        assert np.array_equal(got[k]["color"].numpy(), O.trunc8(img.cpu().numpy())), f"view {i}"


def test_a_ply_round_trip_renders_the_same_frames(trained, tmp_path):
    """io.export_gs_to_ply stores anchors + offsets summed in fp32 and the third log-scale as log(1e-6); the projection forms the same
    fp32 sum from anchors and offsets, and a 2D splat reads only its first two scales, so the frames are identical."""
    Gs, c2w, K, W, H = trained
    G = Gs[0]
    sp = G.state()["splats"]
    deg_max = int(round(((sp["features_rest"].shape[1] + 1) ** 0.5))) - 1
    path = str(tmp_path / "gs.ply")
    IO.export_gs_to_ply(path, **sp)
    back = {k: v.to(sp["anchors"].device) for k, v in IO.load_ply_to_gs(path, deg_max).items()}
    deg = G.T.R.sh_degree
    live = list(VW.render_views(sp, c2w, (W, H, K), sh_degree=deg))
    read = list(VW.render_views(back, c2w, (W, H, K), sh_degree=deg))
    for i, (a, b) in enumerate(zip(live, read)):
        for k in ("color", "depth", "normal"):
            assert torch.equal(a[k], b[k]), f"view {i} {k}"


def test_render_path_writes_the_reference_layout(tmp_path):
    cv2 = pytest.importorskip("cv2")
    dev = _dev()
    sp = _raw_splats(2000, dev, seed=2)
    poses, cam = _poses(3), (160, 96, torch.tensor([[90.0, 0, 79.5], [0, 90.0, 47.5], [0, 0, 1]]))
    frames = list(VW.render_views(sp, poses, cam, sh_degree=DEG))
    assert VW.render_path(sp, poses, cam, str(tmp_path / "path"), sh_degree=DEG) == 3
    names = ["a.png", "b.png", "c.png"]
    VW.render_path(sp, poses, cam, str(tmp_path / "eval"), names=names, sh_degree=DEG)
    for i in range(3):
        rgb = cv2.imread(str(tmp_path / "path" / "color" / "renders" / f"{i}.png"))[..., ::-1]
        assert np.array_equal(rgb, frames[i]["color"].numpy())
        dep = cv2.imread(str(tmp_path / "path" / "depth" / "renders" / f"{i}.png"))[..., ::-1]
        assert np.array_equal(dep, frames[i]["depth"].numpy())
        nrm = cv2.imread(str(tmp_path / "eval" / "normal" / names[i]))[..., ::-1]
        assert np.array_equal(nrm, frames[i]["normal"].numpy())
    assert not (tmp_path / "path" / "normal").exists()


def test_the_shim_twin_writes_the_same_bytes():
    dev = _dev()
    import gssdf_shim as shim
    oc, on = _outputs(3, 97, 61, seed=11)
    a = VW.render_frames(torch.from_numpy(oc).to(dev), torch.from_numpy(on).to(dev))
    b = shim.gssdf_render_frames(torch.from_numpy(oc).to(dev), torch.from_numpy(on).to(dev))
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    one = shim.gssdf_render_frames(torch.from_numpy(oc[1]).to(dev), torch.from_numpy(on[1]).to(dev))
    assert all(torch.equal(x[1:2], y) for x, y in zip(a, one))
