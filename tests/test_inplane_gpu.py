"""GPU: the in-plane rotation search.  inplane_rotate_kernel against the torch oracle bit for bit (and its exact
cases); the sign of the convention on rendered points; the encoder's chunked loop against encode_image of the
materialised rotated batch; predict_pose_inplane against separate predict_pose calls on rotated queries, its joint
ranking and poses, its query forms and A = 1; recovery of quarter-turned images through retrieval_inplane; and no host
synchronisation.  The weights are seeded: nothing here says how well a trained model recovers a roll."""
import math

import pytest
import torch

from _util import no_host_sync
from oracle import inplane_oracle as orc

pytestmark = pytest.mark.gpu

B, Q, K = 2, 3, 5


def max_rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float(((a - b).abs() / b.abs().clamp_min(1e-30)).max())


# ------------------------------------------------------------------ kernel
@pytest.mark.parametrize("A", [1, 4, 7, 36])
@pytest.mark.parametrize("H,W", [(256, 256), (33, 33), (23, 17)])
def test_rotate_kernel_matches_oracle(A, H, W):
    from nope_b200.inplane import inplane_table, rotate_images
    g = torch.Generator().manual_seed(A * 1000 + H)
    img = torch.rand(2, 3, H, W, generator=g) * 2 - 1
    img[0, 1, 3, 4] = -0.0
    out = rotate_images(img.cuda(), A).cpu()
    assert out.shape == (2, A, 3, H, W)
    assert torch.equal(out, orc.rotate(img, inplane_table(A)))
    assert torch.equal(out.view(torch.int32), orc.rotate(img, inplane_table(A)).view(torch.int32))   # bits, signs of 0
    assert torch.equal(out[:, 0], img)
    if H == W and A % 4 == 0:
        for q in (1, 2, 3):
            assert torch.equal(out[:, q * A // 4], torch.rot90(img, q, dims=(-2, -1))), q


def _render(pts, H, W, sigma=3.0):
    """Gaussian blobs at pixel positions pts [n, 2] on the -1 background, three equal channels"""
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    d2 = (xs[None] - pts[:, 0, None, None]) ** 2 + (ys[None] - pts[:, 1, None, None]) ** 2
    img = -1 + 2 * torch.exp(-d2 / (2 * sigma * sigma)).sum(0)
    return img.float().expand(3, H, W)


def test_geometry_sign_on_device():
    """Render points under T and under Rz(alpha) T.  Rotating the second image by alpha (the kernel's copy at bin a)
    gives the first back, within bilinear error; rotating it by -alpha does not."""
    from nope_b200.inplane import inplane_rotations, rotate_images
    H = W = 128
    f, c = 150.0, ((W - 1) / 2, (H - 1) / 2)
    g = torch.Generator().manual_seed(3)
    qv = torch.randn(4, generator=g, dtype=torch.float64)
    w, x, y, z = (qv / qv.norm()).tolist()
    T = torch.tensor([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                      [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                      [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], dtype=torch.float64)
    t = torch.tensor([0.0, 0.0, 4.0], dtype=torch.float64)
    X = torch.randn(6, 3, generator=g, dtype=torch.float64) * 0.4
    A, a = 36, 5                                                     # alpha = 50 degrees
    Rz = inplane_rotations(A)[a]
    p = orc.project(T, t, X, f, c)
    p_roll = orc.project(Rz @ T, Rz @ t, X, f, c)
    assert ((p - torch.tensor(c)).norm(dim=1) < 0.4 * W).all()       # every blob stays inside after any rotation
    img, img_roll = _render(p, H, W), _render(p_roll, H, W)
    rot = rotate_images(img_roll[None].cuda(), A)[0].cpu()
    err_plus = float((rot[a] - img).abs().max())
    err_minus = float((rot[A - a] - img).abs().max())
    assert err_plus < 0.1, err_plus                                  # 0.060 (the oracle computes the same bits)
    assert err_minus > 1.0, err_minus                                # 3.13


# ------------------------------------------------------------------ encoder loop
def test_encoder_loop_equals_encode_of_the_rotated_batch(gpu_model):
    """3 images x 12 angles = 36 pairs: one full chunk of 32 and one of 4"""
    from nope_b200.inplane import rotate_images
    enc = gpu_model.u_net.encoder
    g = torch.Generator().manual_seed(7)
    img = (torch.rand(3, 3, 256, 256, generator=g) * 2 - 1).cuda()
    feat = enc.encode_image_inplane(img, 12)
    assert feat.shape == (3, 12, enc.latent_dim, 32, 32)
    ref = enc.encode_image(rotate_images(img, 12).view(36, 3, 256, 256)).view(3, 12, enc.latent_dim, 32, 32)
    assert torch.equal(feat, ref)
    assert torch.equal(enc.encode_image_inplane(img[:1], 1)[:, 0], enc.encode_image(img[:1]))


# ------------------------------------------------------------------ search
@pytest.fixture(scope="module")
def scene():
    from nope_b200.poses import icosphere_object_rotations, synthetic_pose_batch
    from oracle import inputs
    rel = synthetic_pose_batch(642, B)[0].cuda()
    tp = torch.from_numpy(icosphere_object_rotations(2))
    g = torch.Generator().manual_seed(21)
    q = torch.rand(B, Q, 3, 256, 256, generator=g) * 2 - 1
    _, r = inputs.make_images(seed=9, batch=B)
    return {"rel": rel, "tp": tp, "q": q.cuda(), "r": r.cuda()}


def test_search_matches_separate_calls_ranking_and_poses(gpu_model, scene):
    from nope_b200.inplane import compose, inplane_rotations, rotate_images
    A = 7
    q, r, rel, tp = scene["q"], scene["r"], scene["rel"], scene["tp"]
    R, n, a, sim = gpu_model.predict_pose_inplane(q, r, rel, tp, k=K, angles=A)
    assert sim.shape == (B, Q, A, 642) and n.shape == a.shape == (B, Q, K) and R.shape == (B, Q, K, 3, 3)
    assert n.dtype == a.dtype == torch.int64 and R.dtype == torch.float64
    rot = rotate_images(q.reshape(B * Q, 3, 256, 256), A)
    for ai in range(A):
        sep = gpu_model.predict_pose(rot[:, ai].reshape(B, Q, 3, 256, 256), r, rel, k=K)[2]
        assert max_rel(sim[:, :, ai], sep) < 1e-6, ai
    n_o, a_o = orc.joint_topk(sim, K)
    assert torch.equal(n.cpu(), n_o) and torch.equal(a.cpu(), a_o)
    flat = sim.reshape(B, Q, A * 642).cpu()
    assert torch.equal(flat.gather(-1, (a * 642 + n).cpu()), flat.sort(dim=-1, descending=True).values[..., :K])
    assert torch.allclose(R.cpu(), compose(tp, n.cpu(), a.cpu(), A), rtol=0, atol=1e-14)
    assert torch.allclose(R.cpu(), inplane_rotations(A)[a.cpu()] @ tp[n.cpu()], rtol=0, atol=1e-14)


def test_query_forms_and_one_angle(gpu_model, scene):
    q, r, rel, tp = scene["q"], scene["r"], scene["rel"], scene["tp"]
    A = 4
    for qq, rr, rl, lead in ((q[:, 0], r, rel, (B,)), (q[0], r[:1], rel[:1], (Q,)), (q, r, rel, (B, Q))):
        R, n, a, sim = gpu_model.predict_pose_inplane(qq, rr, rl, tp, k=K, angles=A)
        assert R.shape == lead + (K, 3, 3) and n.shape == a.shape == lead + (K,) and sim.shape == lead + (A, 642)
        assert ((a >= 0) & (a < A)).all() and ((n >= 0) & (n < 642)).all()
        # angles = 1 is predict_pose with angle_idx all 0
        R1, n1, a1, sim1 = gpu_model.predict_pose_inplane(qq, rr, rl, tp, k=K, angles=1)
        Rp, np_, simp = gpu_model.predict_pose(qq, rr, rl, tp, k=K)
        assert torch.equal(n1, np_) and (a1 == 0).all() and torch.equal(R1.cpu(), Rp.double().cpu())
        assert max_rel(sim1[..., 0, :], simp) < 1e-6
    assert gpu_model.predict_pose_inplane(q[:, 0], r, rel, None, k=K, angles=2)[0] is None


@pytest.mark.parametrize("A", [4, 36])
def test_retrieval_recovers_quarter_turns(gpu_model, A):
    """templates: the features of M images; queries: those images turned by j quarter turns.  The best (angle, pose)
    is the bin that undoes the turn and the image's own template."""
    enc = gpu_model.u_net.encoder
    M = 6
    g = torch.Generator().manual_seed(A)
    img = (torch.rand(M, 3, 256, 256, generator=g) * 2 - 1).cuda()
    tf = enc.encode_image(img)[None]                                  # [1, M, C, 32, 32]: generated once
    turns = [j % 4 for j in range(M)]
    qry = torch.stack([torch.rot90(img[j], turns[j], dims=(-2, -1)) for j in range(M)])
    sim, n, a = gpu_model.retrieval_inplane(qry, tf, k=2, angles=A)
    assert sim.shape == (M, A, M) and n.shape == a.shape == (M, 2)
    assert n[:, 0].tolist() == list(range(M))
    assert a[:, 0].tolist() == [((4 - j) % 4) * A // 4 for j in turns]
    n_o, a_o = orc.joint_topk(sim, 2)
    assert torch.equal(n.cpu(), n_o) and torch.equal(a.cpu(), a_o)
    # one query against per-query template sets (template batch M, query batch 1)
    sim1, n1, a1 = gpu_model.retrieval_inplane(qry[1:2], tf.expand(M, -1, -1, -1, -1), k=1, angles=A)
    assert sim1.shape == (M, A, M) and (n1[:, 0] == 1).all() and (a1[:, 0] == 3 * A // 4).all()
    assert torch.equal(sim1[0], sim[1])


def test_search_does_not_synchronise(gpu_model, scene):
    """predict_pose_inplane on device inputs, after one warm-up call (which allocates the staging buffer and uploads
    the angle tables), under torch's sync debug mode.  That mode sees synchronisation on the Python / torch side
    only: a synchronising call inside the library would not be caught here."""
    q, r, rel = scene["q"], scene["r"], scene["rel"]
    tp = scene["tp"].cuda()
    first = gpu_model.predict_pose_inplane(q, r, rel, tp, k=K, angles=6)
    with no_host_sync():
        out = gpu_model.predict_pose_inplane(q, r, rel, tp, k=K, angles=6)
    torch.cuda.synchronize()
    for x, y in zip(out, first):
        assert torch.equal(x, y)
