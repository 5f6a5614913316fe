"""f-4: the reference's on-disk formats, so that `view` / `render` of a reference build can load what this path trained and vice versa.

  gs.ply                  NeuralGS::export_gs_to_ply / load_ply_to_gs (include/neural_gaussian/neural_gaussian.cpp:928-1188): binary
                          little-endian PLY, one `vertex` element, float32 properties in this order:
                          x y z | f_dc_0..2 | f_rest_0..3(K-1)-1 (channel-major: features_rest.transpose(1,2).flatten(1)) | opacity (logit) |
                          scale_0 scale_1 scale_2 (log; scale_2 = log(1e-6) "to make it compatible with 3DGS") | rot_0..3 (w,x,y,z, raw)
                          x y z = anchors + offsets; loading puts everything into anchors and zeroes the offsets (:1137-1143).
  as_occ_prior.ply        point cloud the occupancy octree is rebuilt from (neural_mapping.cpp:1366-1374; property names x y z)
  pt.yaml                 write_pt_params / read_pt_params (include/params/params.cpp:443-481): OpenCV-FileStorage YAML with map_origin,
                          inner_map_size, package_path; the octree level / map size are re-derived from leaf_size on load
  local_map_checkpoint.pt torch::save(local_map_ptr) (neural_mapping.cpp:1331-1342): a libtorch module archive with the flat tcnn parameter
                          `encoder_local_map` and `decoder.{0,2,4,..}.{weight,bias}`; written / read through the libtorch shim
                          (gssdf_shim.LocalMapReplay.save / .load), because only libtorch can produce its own archive format.
  mesh_*.ply              NeuralSLAM::save_mesh -> mc::save_mesh_as_ply (include/mesher/cumcubes/src/cumcubes.cpp:30-80): binary PLY with
                          float x y z + uchar red green blue per vertex and `list int int vertex_index` triangles
Host-side file I/O only: numpy + torch tensors, no device code."""
import math
import os
import re

import numpy as np
import torch


def _ply_header(n, props, element="vertex"):
    lines = ["ply", "format binary_little_endian 1.0", f"element {element} {n}"] + [f"property float {p}" for p in props] + ["end_header"]
    return ("\n".join(lines) + "\n").encode("ascii")


def gs_ply_properties(n_sh_bases):
    props = ["x", "y", "z"] + [f"f_dc_{i}" for i in range(3)]
    props += [f"f_rest_{i}" for i in range((n_sh_bases - 1) * 3)]
    return props + ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]


def export_gs_to_ply(path, anchors, offsets, features_dc, features_rest, opacity, scaling, quaternion):
    """All arguments are the RAW NeuralGS parameters ([N,3] [N,3] [N,1,3] [N,K-1,3] [N] [N,3] [N,4])."""
    c = lambda t: t.detach().float().cpu()
    xyz = c(anchors) + c(offsets)
    n = xyz.shape[0]
    f_dc = c(features_dc).transpose(1, 2).flatten(1)
    cols = [xyz, f_dc]
    K = 1
    if features_rest is not None and features_rest.numel() > 0:
        K = 1 + features_rest.shape[1]
        cols.append(c(features_rest).transpose(1, 2).flatten(1))
    sc = c(scaling)
    sc = torch.cat([sc[:, :2], torch.full((n, 1), math.log(1e-6))], -1)
    cols += [c(opacity).view(n, 1), sc, c(quaternion)]
    data = torch.cat(cols, 1).contiguous().numpy().astype("<f4")
    props = gs_ply_properties(K)
    assert data.shape[1] == len(props)
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "wb") as f:
        f.write(_ply_header(n, props))
        f.write(data.tobytes())
    return n


def _read_ply(path):
    with open(path, "rb") as f:
        raw = f.read()
    end = raw.index(b"end_header\n") + len(b"end_header\n")
    header = raw[:end].decode("ascii").splitlines()
    if header[0] != "ply" or "binary_little_endian" not in header[1]:
        raise ValueError(f"{path}: only binary little-endian PLY is supported (the reference writes binary, neural_gaussian.cpp:1030)")
    n, props, in_vertex = 0, [], False
    types = {"float": "<f4", "float32": "<f4", "double": "<f8", "float64": "<f8", "uchar": "u1", "uint8": "u1", "int": "<i4", "int32": "<i4",
             "short": "<i2", "ushort": "<u2", "uint": "<u4"}
    for ln in header:
        t = ln.split()
        if t[:1] == ["element"]:
            in_vertex = t[1] == "vertex"
            if in_vertex:
                n = int(t[2])
        elif t[:1] == ["property"] and in_vertex:
            if t[1] == "list":
                raise ValueError("list properties are not part of the GS-SDF formats")
            props.append((t[2], types[t[1]]))
    arr = np.frombuffer(raw, dtype=np.dtype(props), count=n, offset=end)
    return arr


def load_ply_to_gs(path, sh_degree, device="cpu"):
    """NeuralGS::load_ply_to_gs: returns dict(anchors, offsets (zeros), features_dc [N,1,3], features_rest [N,K-1,3], opacity, scaling,
    quaternion); properties are looked up BY NAME like tinyply does, so 3DGS-written files load too."""
    a = _read_ply(path)
    K = (sh_degree + 1) ** 2
    col = lambda names: torch.from_numpy(np.stack([a[k].astype(np.float32) for k in names], 1)).to(device)
    anchors = col(["x", "y", "z"])
    out = dict(anchors=anchors, offsets=torch.zeros_like(anchors))
    out["features_dc"] = col([f"f_dc_{i}" for i in range(3)]).view(-1, 3, 1).transpose(1, 2).contiguous()
    if sh_degree > 0:
        out["features_rest"] = col([f"f_rest_{i}" for i in range((K - 1) * 3)]).view(-1, 3, K - 1).transpose(1, 2).contiguous()
    else:
        out["features_rest"] = torch.zeros(anchors.shape[0], 0, 3, device=device)
    out["opacity"] = col(["opacity"]).view(-1)
    out["scaling"] = col(["scale_0", "scale_1", "scale_2"])
    out["quaternion"] = col(["rot_0", "rot_1", "rot_2", "rot_3"])
    return out


def write_points_ply(path, xyz):
    """as_occ_prior.ply: x y z float32."""
    d = xyz.detach().float().cpu().contiguous().numpy().astype("<f4")
    with open(path, "wb") as f:
        f.write(_ply_header(d.shape[0], ["x", "y", "z"]))
        f.write(d.tobytes())


def read_points_ply(path, device="cpu"):
    a = _read_ply(path)
    return torch.from_numpy(np.stack([a["x"], a["y"], a["z"]], 1).astype(np.float32)).to(device)


def write_pt_params(path, map_origin, inner_map_size, package_path=""):
    """write_pt_params (params.cpp:443-453); cv::Mat's operator<< prints a 1x3 float row as [a, b, c]."""
    o = [float(v) for v in np.asarray(map_origin, np.float32).reshape(3)]
    fmt = lambda v: repr(np.float32(v).item()) if v != int(v) else str(int(v))
    with open(path, "w") as f:
        f.write("%YAML:1.0\n")
        f.write("map_origin: !!opencv-matrix\n   rows: 1\n   cols: 3\n   dt: f\n   data: [" + ", ".join(fmt(v) for v in o) + "]\n")
        f.write(f"inner_map_size: {inner_map_size:g}\n")
        f.write(f"package_path: {package_path}\n")


def read_pt_params(path, leaf_size):
    """read_pt_params (params.cpp:455-481): values + the quantities the reference re-derives from them."""
    txt = open(path).read()
    m = re.search(r"map_origin:.*?data:\s*\[([^\]]*)\]", txt, flags=re.S)
    origin = np.array([float(v) for v in m.group(1).split(",")], np.float32)
    inner = float(re.search(r"inner_map_size:\s*([-+0-9.eE]+)", txt).group(1))
    pkg = re.search(r"package_path:\s*(.*)", txt)
    level = int(math.ceil(math.log2((inner + 2 * leaf_size) / leaf_size)))
    res = 2 ** level
    return dict(map_origin=origin, inner_map_size=inner, package_path=pkg.group(1).strip() if pkg else "", x_max=0.5 * inner, x_min=-0.5 * inner,
                octree_level=level, map_resolution=res, map_size=res * leaf_size, map_size_inv=1.0 / (res * leaf_size))


def save_mesh_as_ply(path, vertices, faces, colors):
    """mc::save_mesh_as_ply (include/mesher/cumcubes/src/cumcubes.cpp:30-80): binary little-endian PLY; per vertex `float x y z` +
    `uchar red green blue` (15 bytes, unpadded), per face `property list int int vertex_index` (the count 3 as int32, then three int32).
    vertices [V,3] float32, faces [F,3] int32, colors [V,3] uint8 (torch tensors on any device, or numpy arrays)."""
    c = lambda t: t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)
    v, f, col = c(vertices).astype("<f4").reshape(-1, 3), c(faces).astype("<i4").reshape(-1, 3), c(colors).astype("u1").reshape(-1, 3)
    if len(col) != len(v):
        raise ValueError(f"save_mesh_as_ply: {len(v)} vertices but {len(col)} colours")
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {len(v)}", "property float x", "property float y", "property float z",
            "property uchar red", "property uchar green", "property uchar blue", f"element face {len(f)}",
            "property list int int vertex_index", "end_header"]
    rec = np.empty(len(v), np.dtype([("xyz", "<f4", 3), ("rgb", "u1", 3)]))
    rec["xyz"], rec["rgb"] = v, col
    fr = np.empty((len(f), 4), "<i4")
    fr[:, 0], fr[:, 1:] = 3, f
    with open(path, "wb") as fh:
        fh.write(("\n".join(head) + "\n").encode("ascii"))
        fh.write(rec.tobytes())
        fh.write(fr.tobytes())


def read_mesh_ply(path):
    """Reads what save_mesh_as_ply (or the reference's writer) wrote: (vertices [V,3] float32, faces [F,3] int32, colors [V,3] uint8) as
    numpy arrays. Only that layout is accepted: triangles, `list int int`, x y z float + red green blue uchar."""
    with open(path, "rb") as fh:
        raw = fh.read()
    end = raw.index(b"end_header\n") + len(b"end_header\n")
    head = raw[:end].decode("ascii").splitlines()
    m_v = re.search(r"element vertex (\d+)", "\n".join(head))
    m_f = re.search(r"element face (\d+)", "\n".join(head))
    want = ["property float x", "property float y", "property float z", "property uchar red", "property uchar green",
            "property uchar blue", "property list int int vertex_index"]
    if head[:2] != ["ply", "format binary_little_endian 1.0"] or not m_v or not m_f or [h for h in head if h.startswith("property")] != want:
        raise ValueError(f"{path}: not a mesh PLY in the layout of mc::save_mesh_as_ply")
    nv, nf = int(m_v.group(1)), int(m_f.group(1))
    rec = np.frombuffer(raw, np.dtype([("xyz", "<f4", 3), ("rgb", "u1", 3)]), count=nv, offset=end)
    fr = np.frombuffer(raw, "<i4", count=4 * nf, offset=end + 15 * nv).reshape(nf, 4)
    if nf and not (fr[:, 0] == 3).all():
        raise ValueError(f"{path}: only triangle faces are supported")
    return rec["xyz"].astype(np.float32), fr[:, 1:].astype(np.int32), rec["rgb"].astype(np.uint8)


def load_colmap_cameras(path, scale=1.0):
    """COLMAP's cameras.txt as DataParser::load_cameras reads it (include/data_loader/data_parsers/base_parser.cpp:429-496): the camera
    table {camera_id: (W, H, K)} with K a float32 [3,3] pinhole, in the form views.render_views and gstrain.GsTrainer take. A line whose
    first character is `#` is a comment; every other line is `camera_id model width height params...`. PINHOLE and OPENCV are read as
    pinhole `fx fy cx cy` (OPENCV's distortion parameters are ignored, as the reference does). `scale` is the sensor's fp32 image scale:
    width / height become (int)(scale * w) (fp32 product, truncated) and fx, fy, cx, cy the fp32 products with scale. A repeated id
    keeps its last line. OPENCV_FISHEYE raises ValueError (undistortion is out of scope here), as does any other model, a missing file or
    a line that does not parse. One departure: blank lines are skipped (the reference reads them as a camera and fails)."""
    if not os.path.exists(path):
        raise ValueError(f"Camera file does not exist: {path}")
    s = np.float32(scale)
    cams = {}
    with open(path, "r", encoding="latin-1") as f:
        for line in f.read().split("\n"):
            if line.startswith("#") or not line.strip():
                continue
            tok = line.split()
            model = tok[1] if len(tok) > 1 else ""
            if model == "OPENCV_FISHEYE":
                raise ValueError(f"load_colmap_cameras: OPENCV_FISHEYE needs undistortion, which is not supported: {line!r}")
            if model not in ("PINHOLE", "OPENCV"):
                raise ValueError(f"Unsupported camera model: {model}")
            try:
                cam_id, w, h = int(tok[0]), int(tok[2]), int(tok[3])
                fx, fy, cx, cy = (np.float32(float(v)) for v in tok[4:8])
                if len(tok) < 8:
                    raise IndexError
            except (ValueError, IndexError):
                raise ValueError(f"load_colmap_cameras: cannot parse {line!r}") from None
            W, H = int(s * np.float32(w)), int(s * np.float32(h))
            fx, fy, cx, cy = (s * v for v in (fx, fy, cx, cy))
            cams[cam_id] = (W, H, torch.tensor([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]], dtype=torch.float32))
    return cams
