"""No-GPU checks of training on frames of several cameras (DESIGN 7q): io.load_colmap_cameras against a g++ restatement of
DataParser::load_cameras (include/data_loader/data_parsers/base_parser.cpp:429-496), GsTrainer's argument errors for camera tables and
frame lists (raised before any device work), FramesU8's layout, and the new C entry points (exported, ABI revision unchanged)."""
import subprocess
import types

import numpy as np
import pytest
import torch

from gssdf_b200 import gstrain as GT
from gssdf_b200 import io as IO

# load_cameras' loop with sensor::Cameras reduced to the fields it writes; `scale` is sensor_.camera.scale (a float)
LOAD_CAMERAS_CPP = r"""
#include <cstdio>
#include <fstream>
#include <map>
#include <sstream>
#include <stdexcept>
#include <string>
struct Cameras { int width, height, model; float fx, fy, cx, cy; };
int main(int argc, char **argv) {
  float scale = std::stof(argv[2]);
  std::ifstream file(argv[1]);
  std::string line;
  std::map<int, Cameras> cameras;
  try {
    while (std::getline(file, line)) {
      std::istringstream iss(line);
      if (line[0] == '#') continue;
      int cam_id; std::string model_type; int width, height;
      iss >> cam_id >> model_type >> width >> height;
      Cameras camera; camera.width = width; camera.height = height;
      if ((model_type == "OPENCV") || (model_type == "PINHOLE")) {
        camera.model = 0; float fx, fy, cx, cy; iss >> fx >> fy >> cx >> cy;
        camera.fx = fx; camera.fy = fy; camera.cx = cx; camera.cy = cy;
      } else if (model_type == "OPENCV_FISHEYE") {
        camera.model = 1; float fx, fy, cx, cy, k1, k2, k3, k4; iss >> fx >> fy >> cx >> cy >> k1 >> k2 >> k3 >> k4;
        camera.fx = fx; camera.fy = fy; camera.cx = cx; camera.cy = cy;
      } else {
        throw std::runtime_error("Unsupported camera model: " + model_type);
      }
      camera.width = scale * camera.width; camera.height = scale * camera.height;
      camera.fx = scale * camera.fx; camera.fy = scale * camera.fy; camera.cx = scale * camera.cx; camera.cy = scale * camera.cy;
      cameras[cam_id] = camera;
    }
  } catch (const std::exception &e) { std::printf("error %s\n", e.what()); return 0; }
  for (auto &kv : cameras) {
    const Cameras &c = kv.second;
    std::printf("%d %d %d %d %a %a %a %a\n", kv.first, c.model, c.width, c.height, c.fx, c.fy, c.cx, c.cy);
  }
  return 0;
}
"""

FILES = {
    "colmap": "# Camera list with one line of data per camera:\n#   CAMERA_ID, MODEL, WIDTH, HEIGHT, PARAMS[]\n# Number of cameras: 3\n"
              "1 PINHOLE 1920 1080 1371.7 1371.7 960 540\n2 OPENCV 1279 719 903.3333 901.15 639.7 359.1 -0.05 0.01 0.001 -0.0002\n"
              "7 PINHOLE 641 479 512.25 510.75 320.5 239.5",
    "repeat": "3 PINHOLE 100 80 50 50 50 40\n#3 PINHOLE 1 1 1 1 1 1\n3 OPENCV 333 111 77.7 66.6 166.5 55.5 0 0 0 0\n",
    "fisheye": "1 PINHOLE 100 80 50 50 50 40\n2 OPENCV_FISHEYE 640 480 300 300 320 240 0.1 0.01 0 0\n",
    "unknown": "1 SIMPLE_RADIAL 640 480 300 320 240 0.1\n",
}


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    d = tmp_path_factory.mktemp("load_cameras")
    src, exe = d / "load_cameras.cpp", d / "load_cameras"
    src.write_text(LOAD_CAMERAS_CPP)
    subprocess.check_call(["/usr/bin/g++", "-O3", str(src), "-o", str(exe)])
    return exe


def _reference(exe, path, scale):
    out = subprocess.run([str(exe), str(path), repr(float(np.float32(scale)))], capture_output=True, text=True, check=True).stdout
    if out.startswith("error"):
        return out.strip()
    cams = {}
    for line in out.splitlines():
        t = line.split()
        cams[int(t[0])] = (int(t[1]), int(t[2]), int(t[3])) + tuple(np.float32(float.fromhex(v)) for v in t[4:])
    return cams


@pytest.mark.parametrize("scale", [1.0, 0.5, 0.3, 0.37, 1.7])
@pytest.mark.parametrize("name", ["colmap", "repeat"])
def test_parser_equals_load_cameras(exe, tmp_path, name, scale):
    """Comments, a repeated id (the last line wins), OPENCV's ignored distortion, the truncated fp32 product of the sizes and the fp32
    products of the intrinsics, bit for bit."""
    p = tmp_path / "cameras.txt"
    p.write_text(FILES[name])
    want = _reference(exe, p, scale)
    got = IO.load_colmap_cameras(str(p), scale=scale)
    assert sorted(got) == sorted(want)
    for cid, (W, H, K) in got.items():
        model, w, h, fx, fy, cx, cy = want[cid]
        assert model == 0 and (W, H) == (w, h), (cid, W, H, w, h)
        k = K.numpy()
        assert K.dtype == torch.float32 and k.shape == (3, 3)
        assert [k[0, 0], k[1, 1], k[0, 2], k[1, 2]] == [fx, fy, cx, cy], cid
        assert k[0, 1] == k[1, 0] == k[2, 0] == k[2, 1] == 0 and k[2, 2] == 1
    if name == "colmap" and scale == 0.3:
        assert got[2][:2] == (383, 215)  # 0.3f * 1279 = 383.7, 0.3f * 719 = 215.7: truncated


def test_parser_rejects_fisheye_and_unknown_models(exe, tmp_path):
    p = tmp_path / "cameras.txt"
    p.write_text(FILES["fisheye"])
    assert isinstance(_reference(exe, p, 1.0), dict)  # the reference reads it (and undistorts later)
    with pytest.raises(ValueError, match="OPENCV_FISHEYE"):
        IO.load_colmap_cameras(str(p))
    p.write_text(FILES["unknown"])
    assert _reference(exe, p, 1.0) == "error Unsupported camera model: SIMPLE_RADIAL"
    with pytest.raises(ValueError, match="Unsupported camera model: SIMPLE_RADIAL"):
        IO.load_colmap_cameras(str(p))
    with pytest.raises(ValueError, match="does not exist"):
        IO.load_colmap_cameras(str(tmp_path / "missing.txt"))
    p.write_text("1 PINHOLE 640 480 300 300\n")
    with pytest.raises(ValueError, match="cannot parse"):
        IO.load_colmap_cameras(str(p))
    p.write_text("\n1 PINHOLE 64 48 30 30 32 24\n\n")  # blank lines: skipped here (the reference fails on them)
    assert list(IO.load_colmap_cameras(str(p))) == [1]


# ---- GsTrainer's argument errors ----------------------------------------------------------------------------------------------------
def _trainer(images, K, n=None, **kw):
    sdf = types.SimpleNamespace(dev=torch.device("cuda:0"))  # nothing past the argument checks is reached
    n = len(images) if n is None else n
    return GT.GsTrainer(sdf, {}, torch.eye(4).repeat(n, 1, 1), K, images, capacity=10, spatial_scale=1.0, **kw)


def test_gs_trainer_argument_errors():
    two = [torch.zeros(12, 20, 3), torch.zeros(8, 16, 3)]
    with pytest.raises(ValueError, match="empty"):
        _trainer([], torch.eye(3), n=1)
    with pytest.raises(ValueError, match=r"K must be \[3,3\] or \[T,3,3\] with T = 2"):
        _trainer(two, torch.eye(3).repeat(3, 1, 1))
    with pytest.raises(ValueError, match=r"K must be"):
        _trainer(two, torch.eye(4))
    with pytest.raises(ValueError, match=r"K must be"):
        _trainer(torch.zeros(2, 12, 20, 3), torch.eye(3).repeat(1, 1, 1))
    with pytest.raises(ValueError, match="several sizes"):
        _trainer(two, torch.eye(3), mask=torch.ones(12, 20, dtype=torch.bool))
    with pytest.raises(ValueError, match=r"float32 tensor \[H,W,3\]"):
        _trainer([torch.zeros(12, 20, 3), torch.zeros(12, 20, 4)], torch.eye(3))
    with pytest.raises(ValueError, match=r"float32 tensor \[H,W,3\]"):
        _trainer([torch.zeros(12, 20, 3, dtype=torch.float64)], torch.eye(3))
    st = GT.FramesU8.pack([np.zeros((12, 20, 3), np.uint8), np.zeros((8, 16, 3), np.uint8)])
    with pytest.raises(ValueError, match="several sizes"):
        _trainer(st, torch.eye(3).repeat(2, 1, 1), n=2, mask=torch.ones(12, 20, dtype=torch.bool))
    with pytest.raises(ValueError, match=r"K must be"):
        _trainer(st, torch.eye(3).repeat(3, 1, 1), n=2)
    # one size: the mask's own checks apply (a CPU mask is refused as before)
    with pytest.raises(ValueError, match="on cuda"):
        _trainer([torch.zeros(12, 20, 3)] * 2, torch.eye(3), mask=torch.ones(12, 20, dtype=torch.bool))
    with pytest.raises(ValueError, match=r"\[H,W\]"):
        _trainer([torch.zeros(12, 20, 3)] * 2, torch.eye(3), mask=torch.ones(8, 16, dtype=torch.bool))


def test_frames_u8_layout():
    rng = np.random.default_rng(3)
    frames = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for w, h in ((5, 3), (1, 1), (7, 2))]
    st = GT.FramesU8.pack(frames)
    assert st.sizes == [(5, 3), (1, 1), (7, 2)] and st.offsets == [0, 45, 48, 90] and not st.is_cuda
    for i, f in enumerate(frames):
        assert np.array_equal(st.frame(i).numpy(), f)
    assert GT.parse_frames(st) == ("u8", [(5, 3), (1, 1), (7, 2)])
    assert GT.parse_frames(torch.zeros(4, 3, 5, 3)) == ("stack", [(5, 3)] * 4)
    with pytest.raises(ValueError, match="uint8"):
        GT.FramesU8.pack([np.zeros((3, 5, 3), np.float32)])
    with pytest.raises(ValueError, match="bytes"):
        GT.FramesU8(torch.zeros(44, dtype=torch.uint8), [(5, 3)])
    with pytest.raises(ValueError, match="at least one frame"):
        GT.FramesU8(torch.zeros(0, dtype=torch.uint8), [])


# ---- the C entry points -------------------------------------------------------------------------------------------------------------
def test_entry_points_are_declared_exported_and_abi_unchanged():
    import ctypes
    from gssdf_b200 import _lib
    L = _lib.lib()
    for name in ("gssdf_densify_update_state_sized", "gssdf_frames_u8_expand", "gssdf_densify_update_state"):
        assert name in _lib.FUNCS and hasattr(L, name), name
    assert L.gssdf_abi_revision() == 18
    fake = 0x1000  # never dereferenced: every check runs before the launch
    for kw, msg in ((dict(W=0, H=4, store=fake, gt=fake), b"bad frame"), (dict(W=4, H=4, offset=-1, store=fake, gt=fake), b"negative offset"),
                    (dict(W=4, H=4, store=None, gt=fake), b"null pointer"), (dict(W=4, H=4, store=fake, gt=fake + 4), b"16-byte")):
        a = _lib.make_args("gssdf_frames_u8_expand_args", **kw)
        assert L.gssdf_frames_u8_expand(ctypes.byref(a), None) == -1, kw
        assert msg in L.gssdf_last_error(), (kw, L.gssdf_last_error())
    d = _lib.make_args("gssdf_densify_update_args", N=4, cap=4, counts=fake, gaussian_ids=fake, v_densify=fake, visibilities=fake, radii=fake,
                       width=8, height=8, n_cameras=1, grad2d=fake, count=fake, vis=fake, radii_state=fake)
    for s in (0.0, -1.0, float("nan")):
        assert L.gssdf_densify_update_state_sized(ctypes.byref(d), ctypes.c_float(s), None) == -1
        assert b"image_size must be positive" in L.gssdf_last_error()
    assert L.gssdf_densify_update_state_sized(None, ctypes.c_float(1.0), None) == -1
