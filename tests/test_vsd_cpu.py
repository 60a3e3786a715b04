"""CPU: the T-LESS evaluation without a device -- the rasterizer / VSD oracle against the unmodified reference's
`vsd_obj` (tests/golden/vsd.npz), read_ply, the ABI's refusals, and eval_vsd's batch checks."""
import ctypes as C
import os
import struct

import numpy as np
import pytest
import torch

from oracle import render_oracle as ro


# ------------------------------------------------------------------ oracle against the reference
@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "vsd.npz")))


def _frame(g, i):
    name = ("box", "sphere")[int(g["mesh_of_frame"][i])]
    v, f = g[f"{name}_vertices"], g[f"{name}_faces"]
    H, W = g["depth_raw"].shape[1:]
    d_gt = ro.render(v, f, g["gt_poses"][i], g["K"], (H, W))[0].numpy()
    d_est = ro.render(v, f, g["pred_poses"][i], g["K"], (H, W)).numpy()
    return g["depth_raw"][i] / 10.0, d_gt, d_est


def test_oracle_reproduces_the_reference(golden):
    """bitwise for "step" (integer counts, one correctly rounded division), 1e-12 for "tlinear" (summation order)"""
    F = len(golden["depth_raw"])
    for s, (delta, tau) in enumerate(golden["settings"]):
        delta, tau = int(delta), int(tau)
        for i in range(F):
            dt, dg, de = _frame(golden, i)
            step = ro.vsd(dt, dg, de, golden["K"], delta, tau, "step")
            assert np.array_equal(step, golden["vsd_step"][s, i]), (s, i, step, golden["vsd_step"][s, i])
            tl = ro.vsd(dt, dg, de, golden["K"], delta, tau, "tlinear")
            assert np.allclose(tl, golden["vsd_tlinear"][s, i], rtol=1e-12, atol=0), (s, i)
    # the errors span the range: a perfect pose, occlusion and a far-off rotation
    assert golden["vsd_step"].min() == 0.0 and golden["vsd_step"].max() > 0.5


def test_oracle_distance_images_and_masks(golden):
    dt, dg, de = _frame(golden, 0)
    K = golden["K"]
    assert np.array_equal(ro.dist_image(dt, K), golden["dist_test0"])
    assert np.array_equal(ro.dist_image(de[2], K), golden["dist_est0"])
    gt, est = ro.visib_masks(ro.dist_image(dt, K), ro.dist_image(dg, K), ro.dist_image(de[2], K), 15)
    assert np.array_equal(gt, golden["visib_gt0"]) and np.array_equal(est, golden["visib_est0"])
    assert golden["visib_gt0"].sum() > 50 and (dt == 0).any()


def test_oracle_conventions():
    """the sample point of pixel (r, c) is (c + 1/2, r + 1/2); canonical vertex order; top-left rule"""
    K = (100.0, 100.0, 0.0, 0.0)
    # a small triangle around image point (3.5, 2.5) at Z = 100: only pixel (2, 3)
    Z = 100.0
    pts = np.array([[3.3, 2.3], [3.8, 2.4], [3.5, 2.8]])
    v = np.concatenate([pts * Z / 100.0, np.full((3, 1), Z)], axis=1).astype(np.float32)
    d = ro.render(v, np.array([[0, 1, 2]]), np.eye(4), K, (6, 8))[0]
    assert d.nonzero().tolist() == [[2, 3]] and d[2, 3] == 100.0
    f = torch.tensor([[5, 3, 4], [3, 4, 5], [4, 5, 3], [5, 4, 3]])
    assert ro.canonical_faces(f).tolist() == [[3, 4, 5], [3, 4, 5], [3, 4, 5], [3, 5, 4]]
    assert ro._top_left(1, 0) and ro._top_left(0, -1) and not ro._top_left(-1, 0) and not ro._top_left(0, 1)


# ------------------------------------------------------------------ read_ply
def _write_ascii(path, v, f, extra=True, key="vertex_indices"):
    with open(path, "w") as fh:
        fh.write("ply\nformat ascii 1.0\ncomment test\n")
        fh.write(f"element vertex {len(v)}\nproperty float x\nproperty float y\nproperty float z\n")
        if extra:
            fh.write("property float nx\nproperty uchar red\n")
        fh.write(f"element face {len(f)}\nproperty list uchar int {key}\nend_header\n")
        for p in v:
            fh.write(" ".join(repr(float(x)) for x in p) + (" 0.5 7" if extra else "") + "\n")
        for q in f:
            fh.write(f"{len(q)} " + " ".join(str(int(i)) for i in q) + "\n")


def _write_binary(path, v, f, vtype="double", ctype="uchar", itype="uint"):
    fmt = {"double": "d", "float": "f"}[vtype]
    cf = {"uchar": "B", "int": "i", "ushort": "H"}[ctype]
    idf = {"uint": "I", "int": "i", "ushort": "H"}[itype]
    with open(path, "wb") as fh:
        fh.write(f"ply\nformat binary_little_endian 1.0\nelement vertex {len(v)}\nproperty {vtype} x\n"
                 f"property {vtype} y\nproperty {vtype} z\nproperty uchar alpha\nproperty float s\n"
                 f"element face {len(f)}\nproperty list {ctype} {itype} vertex_index\n"
                 f"element edge 1\nproperty int vertex1\nproperty int vertex2\nend_header\n".encode())
        for p in v:
            fh.write(struct.pack("<" + fmt * 3 + "Bf", *[float(x) for x in p], 9, 1.5))
        for q in f:
            fh.write(struct.pack("<" + cf + idf * len(q), len(q), *[int(i) for i in q]))
        fh.write(struct.pack("<ii", 0, 1))


@pytest.mark.parametrize("kind", ["ascii", "ascii_plain", "bin_double", "bin_float_int"])
def test_read_ply(tmp_path, kind):
    from nope_b200.vsd import read_ply
    v, f = ro.sphere(30.0, 1)
    path = str(tmp_path / "m.ply")
    if kind == "ascii":
        _write_ascii(path, v, f)
    elif kind == "ascii_plain":
        _write_ascii(path, v, f, extra=False, key="vertex_index")
    elif kind == "bin_double":
        _write_binary(path, v, f)
    else:
        _write_binary(path, v, f, vtype="float", ctype="int", itype="int")
    vv, ff = read_ply(path)
    assert vv.dtype == np.float32 and ff.dtype == np.int32
    assert np.array_equal(vv, v) and np.array_equal(ff, f)


def test_read_ply_refusals(tmp_path):
    from nope_b200.vsd import read_ply
    v, f = ro.box()
    p = str(tmp_path / "quad.ply")
    _write_ascii(p, v, [[0, 1, 3, 2]] + f.tolist())
    with pytest.raises(ValueError, match="triangle"):
        read_ply(p)
    p = str(tmp_path / "quad.bin.ply")
    _write_binary(p, v, f.tolist() + [[0, 1, 3, 2]])
    with pytest.raises(ValueError, match="triangle"):
        read_ply(p)
    p = str(tmp_path / "quad_mid.bin.ply")                # the one-read path sees a count of 4 and parses row by row
    _write_binary(p, v, f.tolist()[:5] + [[0, 1, 3, 2]] + f.tolist()[5:], ctype="int", itype="ushort")
    with pytest.raises(ValueError, match="triangle"):
        read_ply(p)
    p = str(tmp_path / "range.ply")
    _write_ascii(p, v, f.tolist() + [[0, 1, 8]])
    with pytest.raises(ValueError, match="outside"):
        read_ply(p)
    p = str(tmp_path / "neg.ply")
    _write_binary(p, v, f.tolist() + [[0, -1, 2]], ctype="uchar", itype="int")
    with pytest.raises(ValueError, match="outside"):
        read_ply(p)
    p = str(tmp_path / "big.ply")
    with open(p, "wb") as fh:
        fh.write(b"ply\nformat binary_big_endian 1.0\nelement vertex 0\nend_header\n")
    with pytest.raises(ValueError, match="format"):
        read_ply(p)
    from nope_b200.vsd import Mesh
    with pytest.raises(ValueError, match="outside"):
        Mesh(v, np.array([[0, 1, 8]]), device="cpu")


# ------------------------------------------------------------------ ABI
P = C.c_void_p(256)
_R = dict(v=P, V=8, f=P, F=12, p=P, P=2, fx=500.0, fy=500.0, cx=320.0, cy=240.0, zn=0.05, H=48, W=64, o=P)


@pytest.mark.parametrize("bad,needle", [
    (dict(v=None), "null"), (dict(f=None), "null"), (dict(p=None), "null"), (dict(o=None), "null"),
    (dict(V=0), "V, F"), (dict(F=0), "V, F"), (dict(P=0), "V, F"), (dict(P=65536), "P"),
    (dict(H=0), "H and W"), (dict(W=0), "H and W"), (dict(H=8193), "H and W"), (dict(W=8193), "H and W"),
    (dict(zn=0.0), "znear"), (dict(zn=-1.0), "znear"), (dict(fx=float("inf")), "finite"),
    (dict(cy=float("nan")), "finite")])
def test_render_refusals(bad, needle):
    from nope_b200 import _lib
    lib = _lib.load()
    a = {**_R, **bad}
    assert lib.nope_render_depth(a["v"], a["V"], a["f"], a["F"], a["p"], a["P"], a["fx"], a["fy"], a["cx"], a["cy"],
                                 a["zn"], a["H"], a["W"], a["o"], None) != 0
    assert needle in lib.nope_last_error().decode()


_S = dict(t=P, g=P, e=P, F=2, P=5, H=48, W=64, K=P, d=15.0, tau=20.0, c=0, o=P)


@pytest.mark.parametrize("bad,needle", [
    (dict(t=None), "null"), (dict(g=None), "null"), (dict(e=None), "null"), (dict(K=None), "null"),
    (dict(o=None), "null"), (dict(F=0), "F and P"), (dict(P=0), "F and P"), (dict(H=0), "H and W"),
    (dict(W=9000), "H and W"), (dict(c=2), "cost_type"), (dict(c=-1), "cost_type"), (dict(d=-0.5), "delta"),
    (dict(d=float("nan")), "delta"), (dict(tau=0.0), "tau"), (dict(tau=-1.0), "tau"), (dict(tau=float("inf")), "tau")])
def test_vsd_refusals(bad, needle):
    from nope_b200 import _lib
    lib = _lib.load()
    a = {**_S, **bad}
    assert lib.nope_vsd_error(a["t"], a["g"], a["e"], a["F"], a["P"], a["H"], a["W"], a["K"], a["d"], a["tau"], a["c"],
                              a["o"], None) != 0
    assert needle in lib.nope_last_error().decode()


def test_python_argument_errors():
    from nope_b200.vsd import vsd_errors
    z3, z4 = torch.zeros(1, 8, 8), torch.zeros(1, 2, 8, 8)
    K = torch.eye(3)[None]
    for kw in (dict(cost_type="linear"), dict(delta=-1), dict(tau=0)):
        with pytest.raises(ValueError):
            vsd_errors(z3, z3, z4, K, **kw)
    with pytest.raises(ValueError):
        vsd_errors(z3, z3, torch.zeros(1, 2, 8, 9), K)


# ------------------------------------------------------------------ eval_vsd batch checks
def _cpu_model():
    from nope_b200.encoder import FeatureExtractor
    from nope_b200.model import PoseConditional

    class _NoDevice:
        device = torch.device("cpu")
        encoder = FeatureExtractor(descriptor_size=8)

        def __getattr__(self, name):
            raise AssertionError("device work before the argument check")

    m = PoseConditional(_NoDevice())
    m.tless_cad = {1: object()}
    return m


def _batch(B=2, N=6):
    return {"query": torch.zeros(B, 3, 256, 256), "reference": torch.zeros(B, 3, 256, 256),
            "gt_relativeR": torch.zeros(B, 6), "all_relativeR": torch.zeros(B, N, 6),
            "template_poses": torch.zeros(B, N, 3, 3), "query_pose": torch.zeros(B, 3, 3),
            "query_translation": torch.zeros(B, 3, 1), "intrinsic": torch.zeros(B, 3, 3),
            "depth_path": ["a.png"] * B, "obj_id": torch.ones(B, dtype=torch.int64)}


def test_eval_vsd_refuses_malformed_batches():
    model = _cpu_model()
    for key in _batch():
        b = _batch()
        del b[key]
        with pytest.raises(KeyError):
            model.eval_vsd(b, "obj01")
    for key, val in [("reference", torch.zeros(3, 3, 256, 256)), ("template_poses", torch.zeros(2, 6, 4, 4)),
                     ("template_poses", torch.zeros(1, 6, 3, 3)), ("all_relativeR", torch.zeros(2, 5, 6)),
                     ("query_pose", torch.zeros(2, 4, 4)), ("query_translation", torch.zeros(2, 3)),
                     ("intrinsic", torch.zeros(2, 4)), ("depth_path", ["a.png"]), ("obj_id", torch.ones(3)),
                     ("obj_id", torch.tensor([1, 2]))]:
        with pytest.raises(ValueError):
            model.eval_vsd({**_batch(), key: val}, "obj01")
    with pytest.raises(ValueError):
        model.test_step({"tless_obj01": {**_batch(), "obj_id": torch.tensor([7, 1])}}, 0)
