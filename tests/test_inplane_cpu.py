"""CPU: the in-plane rotation search without a device -- the angle table, the pose rule against the reference's own
in-plane helpers (tests/golden/inplane.npz), the pinhole identity behind it, the oracle's exact cases, the ABI's
refusals, and the Python argument errors."""
import ctypes as C
import math
import os
import types

import numpy as np
import pytest
import torch

from oracle import inplane_oracle as orc


# ------------------------------------------------------------------ convention
@pytest.mark.parametrize("A", [1, 2, 3, 4, 7, 12, 36, 72, 360])
def test_angle_table(A):
    from nope_b200.inplane import inplane_angles, inplane_rotations, inplane_table
    ang = inplane_angles(A)
    assert ang.dtype == torch.float64 and ang.shape == (A,)
    assert torch.equal(ang, torch.arange(A, dtype=torch.float64) * 360.0 / A)
    cs = inplane_table(A)
    assert cs.dtype == torch.float32 and cs.shape == (A, 2)
    for a in range(A):
        if (4 * a) % A == 0:                                  # quarter turns: exactly 0 and +-1
            q = (4 * a) // A
            assert cs[a].tolist() == [[1.0, 0.0], [0.0, 1.0], [-1.0, 0.0], [0.0, -1.0]][q]
        else:
            t = 2.0 * math.pi * a / A
            assert cs[a, 0].item() == float(np.float32(math.cos(t))) and cs[a, 1].item() == float(np.float32(math.sin(t)))
    Rz = inplane_rotations(A)
    assert Rz.dtype == torch.float64 and Rz.shape == (A, 3, 3)
    assert torch.allclose(Rz @ Rz.transpose(1, 2), torch.eye(3, dtype=torch.float64).expand(A, 3, 3), atol=1e-15)
    assert torch.equal(Rz[:, 2], torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64).expand(A, 3))
    assert torch.allclose(Rz[:, 0, 0], torch.cos(torch.deg2rad(ang)), atol=1e-15)
    assert torch.allclose(Rz[:, 1, 0], torch.sin(torch.deg2rad(ang)), atol=1e-15)
    assert torch.equal(Rz[:, 0, 1], -Rz[:, 1, 0]) and torch.equal(Rz[:, 1, 1], Rz[:, 0, 0])
    assert torch.equal(Rz[:, :2, :2].reshape(A, 4)[:, [0, 2]].float(), cs)


def test_compose_against_the_reference_helpers(golden_dir):
    """R = Rz(alpha) T is the reference's adding_inplane_to_pose(T, inplane=-alpha), and its compute_inplane(R, T)
    returns -alpha"""
    from nope_b200.inplane import compose
    g = np.load(os.path.join(golden_dir, "inplane.npz"))
    T = torch.from_numpy(g["template_R"])
    assert len(T) >= 16 and len(set(g["A"].tolist())) >= 3
    for i in range(len(T)):
        A, a = int(g["A"][i]), int(g["angle_idx"][i])
        assert g["alpha_deg"][i] == a * 360.0 / A
        R = compose(T, torch.tensor([i]), torch.tensor([a]), A)[0]
        assert R.dtype == torch.float64
        assert np.allclose(R.numpy(), g["query_R"][i], rtol=0, atol=1e-12), i
        d = (g["inplane"][i] + g["alpha_deg"][i]) % 360.0              # compute_inplane = -alpha (mod 360)
        assert min(d, 360.0 - d) < 1e-9, (i, g["inplane"][i], g["alpha_deg"][i])
    # batched indices and the [1, N, 3, 3] template form
    idx = torch.arange(len(T)).view(4, -1)
    R = compose(T[None], idx, torch.zeros_like(idx), 7)
    assert R.shape == idx.shape + (3, 3) and torch.equal(R, T[idx])


def test_pinhole_identity():
    """projecting Rz(alpha) T X equals c + R2(alpha) (projection of T X - c): rolling the camera rotates its image
    about the principal point"""
    g = torch.Generator().manual_seed(0)
    f, c = 300.0, (127.5, 127.5)
    cc = torch.tensor(c, dtype=torch.float64)
    for _ in range(20):
        q = torch.randn(4, generator=g, dtype=torch.float64)
        w, x, y, z = (q / q.norm()).tolist()
        T = torch.tensor([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                          [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                          [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], dtype=torch.float64)
        t = torch.tensor([0.1, -0.2, 4.0], dtype=torch.float64) + 0.1 * torch.randn(3, generator=g, dtype=torch.float64)
        X = torch.randn(50, 3, generator=g, dtype=torch.float64)
        al = float(torch.rand(1, generator=g)) * 2 * math.pi
        ca, sa = math.cos(al), math.sin(al)
        Rz = torch.tensor([[ca, -sa, 0.0], [sa, ca, 0.0], [0.0, 0.0, 1.0]], dtype=torch.float64)
        R2 = Rz[:2, :2]
        p = orc.project(T, t, X, f, c)
        p_roll = orc.project(Rz @ T, Rz @ t, X, f, c)
        assert (p_roll - (cc + (p - cc) @ R2.T)).abs().max() < 1e-9


# ------------------------------------------------------------------ oracle
@pytest.mark.parametrize("H,W", [(16, 16), (9, 9), (7, 12)])
def test_oracle_exact_cases(H, W):
    from nope_b200.inplane import inplane_table
    g = torch.Generator().manual_seed(1)
    img = torch.rand(2, 3, H, W, generator=g) * 2 - 1
    out = orc.rotate(img, inplane_table(8))
    assert out.shape == (2, 8, 3, H, W)
    assert torch.equal(out[:, 0], img)                                 # bin 0: the input, bit for bit
    if H == W:
        for q in (1, 2, 3):                                            # quarter turns: torch.rot90
            assert torch.equal(out[:, 2 * q], torch.rot90(img, q, dims=(-2, -1))), q
    # taps outside the image read -1: the corners of a 45-degree copy lie outside
    assert (out[:, 1, :, 0, 0] == -1).all() and (out[:, 1, :, -1, -1] == -1).all()


def test_oracle_bilinear_and_joint_topk():
    from nope_b200.inplane import inplane_table
    img = torch.arange(25, dtype=torch.float32).view(1, 1, 5, 5).expand(1, 3, 5, 5).contiguous()
    out = orc.rotate(img, inplane_table(8))[0, 1, 0]                   # 45 degrees: centre fixed
    assert out[2, 2] == img[0, 0, 2, 2]
    # (x, y) = (3, 2): source (2 + cos45, 2 + sin45); bilinear of a linear ramp I = 5 y + x is the ramp itself
    s = math.sqrt(0.5)
    assert abs(float(out[2, 3]) - (5 * (2 + s) + (2 + s))) < 1e-5
    sim = torch.tensor([[[0.0, 3.0, 1.0], [3.0, -1.0, 2.0]]])          # [1, A=2, N=3]: a tie at flat 1 and 3
    n, a = orc.joint_topk(sim, 4)
    assert n.tolist() == [[1, 0, 2, 2]] and a.tolist() == [[0, 1, 1, 0]]


# ------------------------------------------------------------------ ABI
P = C.c_void_p(256)


@pytest.mark.parametrize("args,needle", [
    ((None, 1, 8, 8, P, 4, P), "null"), ((P, 1, 8, 8, None, 4, P), "null"), ((P, 1, 8, 8, P, 4, None), "null"),
    ((P, 0, 8, 8, P, 4, P), "B"), ((P, 1, 0, 8, P, 4, P), "H"), ((P, 1, 8, 0, P, 4, P), "W"),
    ((P, 1, 8, 8, P, 0, P), "A"), ((P, 1, 8, 8, P, 361, P), "A")])
def test_rotate_refusals(args, needle):
    from nope_b200 import _lib
    lib = _lib.load()
    assert lib.nope_inplane_rotate(*args, None) != 0
    assert needle in lib.nope_last_error().decode()


@pytest.mark.parametrize("args,needle", [
    ((P, None, 1, P, 4, P), "null"), ((P, P, 1, None, 4, P), "null"), ((P, P, 1, P, 4, None), "null"),
    ((P, P, 0, P, 4, P), "B"), ((P, P, 1, P, 0, P), "A"), ((P, P, 1, P, 361, P), "A"),
    ((None, P, 1, P, 4, P), "encoder")])
def test_encode_inplane_refusals(args, needle):
    from nope_b200 import _lib
    lib = _lib.load()
    assert lib.nope_encoder_encode_inplane(*args, None) != 0
    assert needle in lib.nope_last_error().decode()


# ------------------------------------------------------------------ Python argument errors
def _cpu_model():
    from nope_b200.encoder import FeatureExtractor
    from nope_b200.model import PoseConditional

    class _NoDevice:
        device = torch.device("cpu")
        encoder = FeatureExtractor(descriptor_size=8)

        def sweep(self, *a, **kw):
            raise AssertionError("device work before the argument check")

        def set_metric(self, *a, **kw):
            raise AssertionError("device work before the argument check")

    return PoseConditional(_NoDevice())


def test_python_argument_errors_without_a_device():
    from nope_b200.inplane import check_inplane_args, inplane_table
    model = _cpu_model()
    img, rel = torch.zeros(1, 3, 256, 256), torch.zeros(1, 42, 6)
    bad = [dict(angles=0), dict(angles=361), dict(angles=2.0), dict(angles=True), dict(k=0), dict(k=65),
           dict(angles=1, k=43),                                                     # k > A * N
           dict(all_relativeR=torch.zeros(2, 42, 6)), dict(all_relativeR=torch.zeros(1, 42, 9)),
           dict(all_relativeR=torch.zeros(42, 6)), dict(query=torch.zeros(2, 3, 256, 256),
                                                        reference=torch.zeros(3, 3, 256, 256),
                                                        all_relativeR=torch.zeros(3, 42, 6))]
    for kw in bad:
        kw = {"query": img, "reference": img, "all_relativeR": rel, **kw}
        with pytest.raises(ValueError):
            model.predict_pose_inplane(**kw)
    tf = torch.zeros(1, 42, 8, 32, 32)
    for q, t, kw in [(img, tf, dict(angles=0)), (img, tf, dict(k=0)), (img, tf[:, :2], dict(angles=4, k=9)),
                     (img[0], tf, {}), (img, tf[0], {}), (img, torch.zeros(1, 42, 4, 32, 32), {}),
                     (torch.zeros(2, 3, 256, 256), torch.zeros(3, 42, 8, 32, 32), {})]:
        with pytest.raises(ValueError):
            model.retrieval_inplane(q, t, **kw)
    for args in [(0, 5, 10), (361, 5, 10), (4, 0, 10), (4, 65, 10), (2, 5, 2), (3, 1, 0)]:
        with pytest.raises(ValueError):
            check_inplane_args(*args)
    assert check_inplane_args(2, 4, 2) == (2, 4)
    with pytest.raises(ValueError):
        inplane_table(0)


def test_torch_backend_has_no_inplane_path():
    from nope_b200 import _lib
    from nope_b200.encoder import FeatureExtractor
    from nope_b200.inplane import rotate_images
    enc = FeatureExtractor(descriptor_size=8, backend="torch")
    with pytest.raises(_lib.NopeError):
        enc.encode_image_inplane(torch.zeros(1, 3, 256, 256), 4)
    with pytest.raises(_lib.NopeError):
        rotate_images(torch.zeros(1, 3, 8, 8), 4)


def test_sharded_model_is_refused():
    from nope_b200.model import PoseConditional
    model = PoseConditional(types.SimpleNamespace(device=torch.device("cpu")))
    model.dist = object()
    img = torch.zeros(1, 3, 256, 256)
    with pytest.raises(NotImplementedError, match="shard"):
        model.predict_pose_inplane(img, img, torch.zeros(1, 42, 6))
