"""On-disk formats either side of the render / fusion path, without ``plyfile``:

* Gaussian PLY — the 3DGS vertex layout the reference writes and reads with plyfile
  (model/gaussian_model.py:250-281 save_ply, :288-344 load_ply): binary little-endian, one ``vertex`` element,
  float32 properties  x y z nx ny nz f_dc_0..2 f_rest_0..(3*((D+1)^2-1)-1) opacity scale_0..2 rot_0..3, with the
  SH coefficients stored channel-major (``transpose(1, 2).flatten``).
* fused-feature ``.pt`` — ``{"feat": float16 (n, C), "mask_full": bool (P,)}`` (fusion.py:234-257), consumed at
  eval_segmentation.py:211-219, view_viser.py:61-75, dataset/feature_dataset.py:63-64.
* dynamic ``params.npz`` (model/gaussian_model.py:346-378).
* labelled scan vertices — the ``vertex`` properties of a binary little-endian mesh PLY such as ScanNet's
  ``*_vh_clean_2.labels.ply`` (``load_ply_vertices``), the ground truth of a 3D point evaluation."""
from __future__ import annotations

import os
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2",
              "ushort": "u2", "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4",
              "float": "f4", "float32": "f4", "double": "f8", "float64": "f8"}
C0 = 0.28209479177387814  # utils/sh_utils.py:24


def gaussian_attribute_names(n_dc: int, n_rest: int, n_scale: int = 3, n_rot: int = 4) -> List[str]:
    """model/gaussian_model.py:250-263 construct_list_of_attributes."""
    names = ["x", "y", "z", "nx", "ny", "nz"]
    names += [f"f_dc_{i}" for i in range(n_dc)]
    names += [f"f_rest_{i}" for i in range(n_rest)]
    names.append("opacity")
    names += [f"scale_{i}" for i in range(n_scale)]
    names += [f"rot_{i}" for i in range(n_rot)]
    return names


def write_vertex_ply(path: str, names: List[str], table: np.ndarray) -> None:
    """Binary little-endian PLY with one float32 ``vertex`` element (what PlyData([el]).write produces)."""
    table = np.ascontiguousarray(table, dtype="<f4")
    if table.ndim != 2 or table.shape[1] != len(names):
        raise ValueError("table must be (N, len(names))")
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    header = "ply\nformat binary_little_endian 1.0\n" + f"element vertex {table.shape[0]}\n"
    header += "".join(f"property float {n}\n" for n in names) + "end_header\n"
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(table.tobytes())


def _first_element_header(f, path: str):
    """Read a PLY header up to end_header: (format, first element's name, its count, [(property, dtype code)])."""
    if f.readline().strip() != b"ply":
        raise ValueError(f"{path}: not a PLY file")
    fmt, name, count, props, in_first, seen_elem = None, None, 0, [], False, 0
    while True:
        line = f.readline()
        if not line:
            raise ValueError(f"{path}: truncated PLY header")
        tok = line.decode("ascii", "replace").split()
        if not tok or tok[0] in ("comment", "obj_info"):
            continue
        if tok[0] == "format":
            fmt = tok[1]
        elif tok[0] == "element":
            seen_elem += 1
            in_first = seen_elem == 1
            if in_first:
                name, count = tok[1], int(tok[2])
        elif tok[0] == "property" and in_first:
            if tok[1] == "list":
                raise ValueError(f"{path}: list properties are not supported")
            if tok[1] not in _PLY_TYPES:
                raise ValueError(f"{path}: unknown property type {tok[1]}")
            props.append((tok[2], _PLY_TYPES[tok[1]]))
        elif tok[0] == "end_header":
            return fmt, name, count, props


def read_vertex_ply(path: str) -> Dict[str, np.ndarray]:
    """First element of a PLY file as {property: 1-D array}.  binary_little_endian, binary_big_endian and
    ascii are accepted; list properties are not (the Gaussian layout has none)."""
    with open(path, "rb") as f:
        fmt, _, count, props = _first_element_header(f, path)
        if fmt == "ascii":
            rows = np.loadtxt(f, dtype=np.float64, max_rows=count, ndmin=2)
            if rows.shape != (count, len(props)):
                raise ValueError(f"{path}: ascii body does not match the header")
            return {n: rows[:, i].astype(t) for i, (n, t) in enumerate(props)}
        if fmt not in ("binary_little_endian", "binary_big_endian"):
            raise ValueError(f"{path}: unsupported PLY format {fmt}")
        order = "<" if fmt == "binary_little_endian" else ">"
        dt = np.dtype([(n, order + t) for n, t in props])
        data = np.frombuffer(f.read(dt.itemsize * count), dtype=dt, count=count)
        return {n: np.ascontiguousarray(data[n]).astype(t) for n, t in props}


def load_ply_vertices(path: str, names: Sequence[str]) -> Dict[str, np.ndarray]:
    """The named properties of the ``vertex`` element of a binary little-endian PLY, {name: 1-D array} in each
    property's own type (``float`` -> float32, ``ushort`` -> uint16, ...).  ``vertex`` must be the first element and
    hold scalar properties only; the elements after it (faces, edges) are not read.  Enough for the ``x, y, z, label``
    of a ScanNet ``*_vh_clean_2.labels.ply``; the raw-label -> class mapping is the caller's.  ASCII and big-endian
    files, a missing property and a truncated body raise ``ValueError``."""
    with open(path, "rb") as f:
        fmt, element, count, props = _first_element_header(f, path)
        if fmt != "binary_little_endian":
            raise ValueError(f"{path}: PLY format {fmt} is not supported (binary_little_endian only)")
        if element != "vertex":
            raise ValueError(f"{path}: the first element is {element!r}, not 'vertex'")
        have = dict(props)
        missing = [n for n in names if n not in have]
        if missing:
            raise ValueError(f"{path}: vertex element has no properties {missing} (it has {list(have)})")
        dt = np.dtype([(n, "<" + t) for n, t in props])
        body = f.read(dt.itemsize * count)
        if len(body) != dt.itemsize * count:
            raise ValueError(f"{path}: truncated vertex data ({len(body)} of {dt.itemsize * count} bytes)")
        data = np.frombuffer(body, dtype=dt, count=count)
        return {n: np.ascontiguousarray(data[n]).astype(have[n]) for n in names}


def save_gaussian_ply(path: str, model) -> None:
    """model/gaussian_model.py:265-281 for any object with the reference's raw parameter tensors."""
    npy = lambda t: t.detach().cpu().numpy()
    xyz = npy(model._xyz)
    f_dc = npy(model._features_dc.detach().transpose(1, 2).flatten(start_dim=1).contiguous())
    f_rest = npy(model._features_rest.detach().transpose(1, 2).flatten(start_dim=1).contiguous())
    opac, scale, rot = npy(model._opacity), npy(model._scaling), npy(model._rotation)
    names = gaussian_attribute_names(f_dc.shape[1], f_rest.shape[1], scale.shape[1], rot.shape[1])
    table = np.concatenate((xyz, np.zeros_like(xyz), f_dc, f_rest, opac, scale, rot), axis=1)
    write_vertex_ply(path, names, table)


def load_gaussian_ply(path: str, model, device="cuda"):
    """model/gaussian_model.py:288-344: fills the raw parameter tensors of ``model`` (float32 on ``device``)."""
    el = read_vertex_ply(path)
    n = el["x"].shape[0]
    by_index = lambda prefix: sorted((k for k in el if k.startswith(prefix)), key=lambda k: int(k.split("_")[-1]))
    xyz = np.stack((el["x"], el["y"], el["z"]), axis=1)
    f_dc = np.stack((el["f_dc_0"], el["f_dc_1"], el["f_dc_2"]), axis=1).reshape(n, 3, 1)
    rest_names = by_index("f_rest_")
    coeffs = (model.max_sh_degree + 1) ** 2 - 1
    if len(rest_names) != 3 * coeffs:
        raise ValueError(f"{path}: {len(rest_names)} f_rest_* properties, expected {3 * coeffs} for SH degree "
                         f"{model.max_sh_degree}")
    f_rest = (np.stack([el[k] for k in rest_names], axis=1) if rest_names else np.zeros((n, 0))).reshape(n, 3, coeffs)
    scales = np.stack([el[k] for k in by_index("scale_")], axis=1)
    rots = np.stack([el[k] for k in by_index("rot")], axis=1)
    t = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float32, device=device)
    model._xyz = t(xyz)
    model._features_dc = t(f_dc).transpose(1, 2).contiguous()
    model._features_rest = t(f_rest).transpose(1, 2).contiguous()
    model._opacity = t(el["opacity"][:, None])
    model._scaling = t(scales)
    model._rotation = t(rots)
    model.active_sh_degree = model.max_sh_degree
    return model


def save_fused_features(path: str, features: torch.Tensor, mask_full: torch.Tensor) -> None:
    """fusion.py:234-257: ``features`` are the rows of the Gaussians selected by ``mask_full`` (P,) bool."""
    if mask_full.dtype != torch.bool or mask_full.ndim != 1 or int(mask_full.sum()) != features.shape[0]:
        raise ValueError("mask_full must be a (P,) bool mask selecting exactly features.shape[0] Gaussians")
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    torch.save({"feat": features.detach().cpu().half(), "mask_full": mask_full.detach().cpu()}, path)


def load_fused_features(path: str, num_gaussians: int = None, device="cpu") -> Tuple[torch.Tensor, torch.Tensor]:
    """-> (feat float16 (n, C), mask_full bool (P,)); eval_segmentation.py:211-219 scatters them back with
    ``features[mask_full] = feat``."""
    blob = torch.load(path, map_location="cpu")
    feat, mask = blob["feat"], blob["mask_full"]
    if mask.dtype != torch.bool or int(mask.sum()) != feat.shape[0]:
        raise ValueError(f"{path}: mask_full does not select feat.shape[0] rows")
    if num_gaussians is not None and mask.shape[0] != num_gaussians:
        raise ValueError(f"{path}: mask_full has {mask.shape[0]} entries, scene has {num_gaussians} Gaussians")
    return feat.to(device), mask.to(device)


def scatter_fused_features(feat: torch.Tensor, mask_full: torch.Tensor, device="cuda") -> torch.Tensor:
    """(P, C) float32 table with the stored rows at ``mask_full`` and zeros elsewhere."""
    out = torch.zeros((mask_full.shape[0], feat.shape[1]), dtype=torch.float32, device=device)
    out[mask_full.to(device)] = feat.to(device=device, dtype=torch.float32)
    return out


def load_dynamic_npz(path: str, t: int, model, device="cuda", cache: dict = None):
    """model/gaussian_model.py:346-378: time step ``t`` of a Dynamic-3D-Gaussians ``params.npz``."""
    if cache is None or "params" not in cache:
        params = {k: np.array(v).astype(np.float32) for k, v in dict(np.load(path)).items()}
        if cache is not None:
            cache["params"] = params
    else:
        params = cache["params"]
    tt = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float32, device=device)
    n = params["logit_opacities"].shape[0]
    model.is_fg = params["seg_colors"][:, 0] > 0.5
    model._features_rest = torch.zeros((n, (model.max_sh_degree + 1) ** 2 - 1, 3), dtype=torch.float32, device=device)
    model._opacity = tt(params["logit_opacities"])
    model._scaling = tt(params["log_scales"])
    model.active_sh_degree = model.max_sh_degree
    model._xyz = tt(params["means3D"][t])
    model._features_dc = tt(((params["rgb_colors"][t] - 0.5) / C0)[:, :, None]).transpose(1, 2).contiguous()  # RGB2SH
    model._rotation = tt(params["unnorm_rotations"][t])
    return model
