"""The nearest-point query without a GPU: sgb_nearest is bound and refuses bad arguments before it touches the ctx or
enqueues anything; the fp32 brute-force oracle the GPU tests compare against is the numpy expression bit for bit and
agrees with a float64 k-d tree wherever fp32 rounding cannot tie the two nearest rows; load_ply_vertices reads the
vertex properties of binary little-endian PLY files and refuses other formats; time_nearest.py starts and refuses to
run without a GPU."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from nearest_ref import d2_numpy, nearest_oracle  # noqa: E402

from semantic_gaussians_b200 import _lib  # noqa: E402

E_INVALID = -1   # SGB_E_INVALID, include/sgb200.h
INF = float("inf")


def test_symbol_is_bound():
    lib = _lib.load()
    assert "sgb_nearest" in _lib.EXPORTS and hasattr(lib, "sgb_nearest")
    assert lib.sgb_nearest.argtypes is not None


def _call(ctx=1, P=10, ref=1, M=10, query=1, max_dist2=INF, index=1, dist2=1):
    # ctx 1 and the pointers 1 are dummies: a refused call must fail before any of them is dereferenced or launched on
    return _lib.load().sgb_nearest(ctx, P, ref, M, query, max_dist2, index, dist2, None)


@pytest.mark.parametrize("kw,msg", [
    (dict(ctx=None), b"null ctx"),
    (dict(P=-1), b"[0, 2^31 - 1]"),
    (dict(P=2**31), b"[0, 2^31 - 1]"),
    (dict(M=-1), b"[0, 2^31 - 1]"),
    (dict(M=2**31), b"[0, 2^31 - 1]"),
    (dict(max_dist2=math.nan), b"NaN"),
    (dict(ref=None), b"null argument"),
    (dict(query=None), b"null argument"),
    (dict(index=None), b"null argument"),
    (dict(dist2=None), b"null argument"),
])
def test_bad_arguments_are_refused_before_the_ctx_is_used(kw, msg):
    assert _call(**kw) == E_INVALID
    assert msg in _lib.load().sgb_last_error()


def test_empty_sets_may_pass_null_pointers():
    assert _call(M=0, query=None, index=None, dist2=None) == 0                     # M == 0 launches nothing
    assert _call(P=0, ref=None, M=0, query=None, index=None, dist2=None) == 0
    assert _call(P=2**31 - 1, M=0, query=None, index=None, dist2=None, max_dist2=-1.0) == 0


def test_python_api_refuses_non_cuda_inputs():
    from semantic_gaussians_b200.metric import nearest_points, transfer_labels
    z = torch.zeros((4, 3))
    with pytest.raises(ValueError, match="CUDA tensor"):
        nearest_points(z, z)
    with pytest.raises(ValueError, match="CUDA tensor"):
        nearest_points(np.zeros((4, 3), np.float32), z)
    with pytest.raises(ValueError, match="integer tensor"):
        transfer_labels(z, z, torch.zeros(4))
    with pytest.raises(ValueError, match="integer tensor"):
        transfer_labels(z, z, torch.zeros(5, dtype=torch.int64))


def _cloud(n, seed):
    rng = np.random.default_rng(seed)
    return rng.uniform(-2, 2, (n, 3)).astype(np.float32)


def test_oracle_is_the_numpy_float32_expression():
    rng = np.random.default_rng(1)
    q = np.concatenate([_cloud(300, 2), rng.normal(0, 50, (20, 3)).astype(np.float32)])
    r = _cloud(700, 3)
    d = d2_numpy(q, r)
    assert d.dtype == np.float32
    index, dist2 = nearest_oracle(torch.from_numpy(q), torch.from_numpy(r))
    want = d.argmin(1)                                   # first minimum: the smallest row
    assert np.array_equal(index.numpy(), want)
    assert np.array_equal(dist2.numpy().view(np.int32), d[np.arange(len(q)), want].view(np.int32))


@pytest.mark.parametrize("kind", ["uniform", "clustered", "surface"])
def test_oracle_matches_a_float64_kdtree_away_from_fp32_ties(kind):
    from scipy.spatial import cKDTree

    from semantic_gaussians_b200.scene_synth import surface_points
    rng = np.random.default_rng(7)
    if kind == "uniform":
        r, q = _cloud(5000, 8), _cloud(3000, 9) * 1.2
    elif kind == "clustered":
        c = rng.uniform(-4, 4, (10, 3))
        r = (c[rng.integers(0, 10, 5000)] + rng.normal(0, 0.05, (5000, 3))).astype(np.float32)
        q = (c[rng.integers(0, 10, 3000)] + rng.normal(0, 0.1, (3000, 3))).astype(np.float32)
    else:
        r, q = surface_points(5000, 10), surface_points(3000, 11)
    index, dist2 = nearest_oracle(torch.from_numpy(q), torch.from_numpy(r))
    d, j = cKDTree(r.astype(np.float64)).query(q.astype(np.float64), k=2)
    untied = d[:, 1] ** 2 - d[:, 0] ** 2 > 1e-5 * d[:, 1] ** 2 + 1e-30
    assert untied.mean() > 0.99
    assert np.array_equal(index.numpy()[untied], j[untied, 0])
    assert np.allclose(dist2.numpy(), d[:, 0] ** 2, rtol=1e-5, atol=1e-12)


def test_oracle_edge_cases():
    r = torch.tensor([[1.0, 0, 0], [0, 0, 0], [1.0, 0, 0], [math.nan, 0, 0], [-1.0, 0, 0], [math.inf, 0, 0]])
    q = torch.tensor([[1.0, 0, 0], [0.5, 0, 0], [0, 0, 0], [math.inf, 0, 0], [-100.0, 0, 0]])
    index, dist2 = nearest_oracle(q, r)
    assert index.tolist() == [0, 0, 1, -1, 4]                    # duplicates and equidistant rows: the smallest wins
    assert dist2.tolist() == [0.0, 0.25, 0.0, INF, 99.0 ** 2]
    index, dist2 = nearest_oracle(q, r, max_dist2=0.25)           # d2 == max_dist2 matches
    assert index.tolist() == [0, 0, 1, -1, -1] and dist2[3:].tolist() == [INF, INF]
    index, _ = nearest_oracle(q, r[:0])
    assert index.tolist() == [-1] * 5


# ---- load_ply_vertices

def _write_ply(path, fmt, vertex_props, rows, tail=b"", extra_header=""):
    header = f"ply\nformat {fmt} 1.0\ncomment synthetic\nelement vertex {len(rows)}\n"
    header += "".join(f"property {t} {n}\n" for n, t, _ in vertex_props)
    header += extra_header + "end_header\n"
    order = ">" if fmt == "binary_big_endian" else "<"
    dt = np.dtype([(n, order + code) for n, _, code in vertex_props])
    body = np.array([tuple(r) for r in rows], dtype=dt).tobytes()
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(body)
        f.write(tail)


_PROPS = [("x", "float", "f4"), ("y", "float", "f4"), ("z", "float", "f4"), ("red", "uchar", "u1"),
          ("green", "uchar", "u1"), ("blue", "uchar", "u1"), ("alpha", "uchar", "u1"), ("label", "ushort", "u2"),
          ("quality", "double", "f8"), ("flags", "int", "i4"), ("tag", "char", "i1"), ("w", "short", "i2")]
_FACES = "element face 2\nproperty list uchar int vertex_indices\n"
_FACE_BODY = bytes([3]) + np.array([0, 1, 2], "<i4").tobytes() + bytes([3]) + np.array([2, 1, 0], "<i4").tobytes()


def _rows(n, seed):
    rng = np.random.default_rng(seed)
    return [(*rng.normal(size=3).astype(np.float32), *rng.integers(0, 256, 4), int(rng.integers(0, 65536)),
             float(rng.normal()), int(rng.integers(-2**31, 2**31)), int(rng.integers(-128, 128)),
             int(rng.integers(-32768, 32768))) for _ in range(n)]


def test_load_ply_vertices_reads_mixed_types_and_skips_faces(tmp_path):
    from semantic_gaussians_b200.io_formats import load_ply_vertices
    rows = _rows(37, 1)
    path = str(tmp_path / "scene_vh_clean_2.labels.ply")
    _write_ply(path, "binary_little_endian", _PROPS, rows, tail=_FACE_BODY, extra_header=_FACES)
    got = load_ply_vertices(path, ["x", "y", "z", "label"])
    assert list(got) == ["x", "y", "z", "label"]
    assert got["label"].dtype == np.uint16 and got["x"].dtype == np.float32
    assert np.array_equal(got["label"], np.array([r[7] for r in rows], np.uint16))
    assert np.array_equal(np.stack([got["x"], got["y"], got["z"]], 1), np.array([r[:3] for r in rows], np.float32))
    every = load_ply_vertices(path, [n for n, _, _ in _PROPS])
    for i, (n, _, code) in enumerate(_PROPS):
        assert every[n].dtype == np.dtype(code)
        assert np.array_equal(every[n], np.array([r[i] for r in rows], dtype=code)), n


def test_load_ply_vertices_refuses_other_formats_and_bad_files(tmp_path):
    from semantic_gaussians_b200.io_formats import load_ply_vertices
    rows = _rows(5, 2)
    be = str(tmp_path / "be.ply")
    _write_ply(be, "binary_big_endian", _PROPS, rows)
    with pytest.raises(ValueError, match="binary_big_endian"):
        load_ply_vertices(be, ["x"])
    asc = str(tmp_path / "ascii.ply")
    with open(asc, "w") as f:
        f.write("ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\nend_header\n1.0\n")
    with pytest.raises(ValueError, match="ascii"):
        load_ply_vertices(asc, ["x"])
    le = str(tmp_path / "le.ply")
    _write_ply(le, "binary_little_endian", _PROPS, rows)
    with pytest.raises(ValueError, match="no properties"):
        load_ply_vertices(le, ["x", "label_raw"])
    with open(le, "rb") as f:
        data = f.read()
    short = str(tmp_path / "short.ply")
    with open(short, "wb") as f:
        f.write(data[:-3])
    with pytest.raises(ValueError, match="truncated"):
        load_ply_vertices(short, ["x"])
    faces_first = str(tmp_path / "faces_first.ply")
    with open(faces_first, "wb") as f:
        f.write(b"ply\nformat binary_little_endian 1.0\nelement face 0\nproperty uchar n\nelement vertex 0\n"
                b"property float x\nend_header\n")
    with pytest.raises(ValueError, match="not 'vertex'"):
        load_ply_vertices(faces_first, ["x"])


# ---- tools/time_nearest.py

def _run_tool(*args):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    return subprocess.run([sys.executable, os.path.join(ROOT, "tools", "time_nearest.py"), *args], capture_output=True,
                          text=True, timeout=300, env=env, cwd=ROOT)


def test_time_nearest_starts_and_refuses_to_run_without_a_gpu():
    p = _run_tool("--help")
    assert p.returncode == 0 and "usage:" in p.stdout, p.stderr[-2000:]
    p = _run_tool()
    assert p.returncode != 0
    assert p.stderr.strip().splitlines()[-1] == "time_nearest.py needs a GPU", p.stderr[-2000:]
