"""GPU: the joint roll and viewpoint refinement.  inplane_rotate_pairs_kernel, pose_refine_inplane_propose and
pose_refine_inplane_select against the torch oracle bit for bit; the encoder's pair loop against encode_image of the
materialised pairs; whole refinements replayed step by step through the oracle, every returned score against a
separate sweep of its (pose, latent); R against an independent composition; the query forms of predict_pose and the
edge cases; no host synchronisation; and roll recovery through a stub engine whose templates do not depend on the
pose.  The weights are seeded: nothing here says how well a trained model recovers a roll."""
import math

import numpy as np
import pytest
import torch

from _util import no_host_sync
from oracle import inplane_oracle
from oracle import inplane_refine_oracle as orc

pytestmark = pytest.mark.gpu

B, Q, KEEP, K = 2, 3, 2, 5


def _equal(a, b):
    return torch.equal(a.cpu(), b.cpu())


def random_rotations(n, g):
    q = torch.randn((n, 4), generator=g, dtype=torch.float64)
    w, x, y, z = (q / q.norm(dim=1, keepdim=True)).unbind(1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                        2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                        2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], dim=1).reshape(n, 3, 3)


def random_cossin(shape, g):
    t = torch.rand(shape, generator=g, dtype=torch.float64) * 2 * math.pi
    return torch.stack([t.cos(), t.sin()], dim=-1).float()


# ------------------------------------------------------------------ rotate pairs
@pytest.mark.parametrize("H,W", [(256, 256), (33, 33), (23, 17)])
def test_rotate_pairs_kernel_matches_oracle(H, W):
    from nope_b200.inplane import inplane_table, rotate_images
    from nope_b200.inplane_refine import rotate_pairs
    g = torch.Generator().manual_seed(H * 31 + W)
    img = torch.rand(3, 3, H, W, generator=g) * 2 - 1
    img[1, 2, 5, 6] = -0.0
    P = 11
    idx = torch.tensor([0, 2, 1, -1, 1, 3, 0, 2, 100, 1, 0], dtype=torch.int32)
    cs = random_cossin((P,), g)
    cs[4] = torch.tensor([0.9, 0.3])                                                # not a unit vector
    out = rotate_pairs(img.cuda(), idx.cuda(), cs.cuda()).cpu()
    want = orc.rotate_pairs(img, idx, cs)
    assert torch.equal(out.view(torch.int32), want.view(torch.int32))              # bits, signs of zero
    for p in (3, 5, 8):                                                             # out of range: all -1
        assert (out[p] == -1).all()
    for p in (2, 4, 6):                                                             # their neighbours unchanged
        assert torch.equal(out[p], inplane_oracle.rotate(img[int(idx[p]):int(idx[p]) + 1], cs[p:p + 1])[0, 0])
    # at table entries, rotate_pairs is rotate_images' copy a
    A = 36
    table = inplane_table(A)
    a = torch.tensor([0, 5, 9, 17, 35, 3], dtype=torch.int64)
    bi = torch.tensor([0, 1, 2, 2, 0, 1], dtype=torch.int32)
    pairs = rotate_pairs(img.cuda(), bi.cuda(), table[a].cuda()).cpu()
    full = rotate_images(img.cuda(), A).cpu()
    assert torch.equal(pairs, full[bi.long(), a])


def test_encode_rotated_equals_encode_of_the_pairs(gpu_model):
    """P = 36 pairs: one chunk of 32 and one of 4.  Also states whether a latent depends on the chunk it was
    encoded in (the native encoder's batch invariance)."""
    from nope_b200.inplane_refine import rotate_pairs
    enc = gpu_model.u_net.encoder
    g = torch.Generator().manual_seed(7)
    img = (torch.rand(3, 3, 256, 256, generator=g) * 2 - 1).cuda()
    P = 36
    idx = torch.randint(-1, 4, (P,), generator=g, dtype=torch.int32).cuda()
    cs = random_cossin((P,), g).cuda()
    feat = enc.encode_image_rotated(img, idx, cs)
    assert feat.shape == (P, enc.latent_dim, 32, 32)
    assert torch.equal(feat, enc.encode_image(rotate_pairs(img, idx, cs)))
    alone = torch.cat([enc.encode_image_rotated(img, idx[p:p + 1], cs[p:p + 1]) for p in range(3)])
    print(f"encoder batch invariance: a pair encoded alone equals its latent in a chunk of 32: "
          f"{torch.equal(alone, feat[:3])} (max abs difference {float((alone - feat[:3]).abs().max()):.3g})")


# ------------------------------------------------------------------ propose / select kernels
@pytest.fixture(scope="module")
def grids():
    from nope_b200.inplane_refine import InplaneRefiner
    from nope_b200.poses import icosphere_object_rotations, synthetic_pose_batch
    R2 = icosphere_object_rotations(2)
    rel = synthetic_pose_batch(642, B)[0].cuda()
    return {"R": R2, "rel": rel, "ref": InplaneRefiner(R2, angles=36, steps=3)}


@pytest.mark.parametrize("keep", [1, 2, 16])
def test_propose_and_select_kernels_match_oracle(grids, keep):
    from nope_b200.inplane_refine import propose, select
    ref = grids["ref"]
    g = torch.Generator().manual_seed(keep)
    N, R = 642, B * Q
    D = random_rotations(R * keep, g).float().reshape(R, keep, 9)
    D[1] = torch.randn(keep, 9, generator=g)                                        # not rotations
    seed = torch.randint(-3, N + 3, (R, keep), generator=g, dtype=torch.int32)
    seed[0, 0] = 7
    cs = random_cossin((R, keep), g)
    cs[2] = torch.randn(keep, 2, generator=g)                                       # not unit rolls
    if keep > 1:
        seed[4] = torch.tensor([-1] + [12] * (keep - 1), dtype=torch.int32)         # padding centre first
        D[0, 1], seed[0, 1], cs[0, 1] = D[0, 0], seed[0, 0], cs[0, 0]               # an exact duplicate centre
    seed[5] = -1                                                                    # no valid centre at all
    poses = grids["rel"]
    for s in (0, 2):
        cand = propose(D.cuda(), seed.cuda(), cs.cuda(), poses, ref.stencils[s].cuda(), ref.rolls[s], Q)
        cand_o = orc.propose(D, seed, cs, poses.cpu(), ref.stencils[s], ref.rolls[s], Q)
        for name in ("D", "seed", "rel", "poses", "cossin"):
            assert _equal(cand[name], cand_o[name]), (s, name)
        assert (cand_o["seed"][5] == -1).all()
        sim = torch.randint(-4, 1, (R, keep * 3, keep * 9), generator=g).float()   # exact ties everywhere
        for k in (1, 10, 64):
            if k > 27 * keep * keep:
                continue
            out = select(sim.cuda(), cand, ref.thresholds[s], k)
            out_o = orc.select(sim, cand_o, ref.thresholds[s], k)
            for name in ("D", "seed", "cossin", "aslot", "score", "rel"):
                assert _equal(out[name], out_o[name]), (s, k, name)
            assert (out_o["seed"][5] == -1).all() and torch.isneginf(out_o["score"][5]).all()


# ------------------------------------------------------------------ whole refinements
def _search(model, q, r, rel, A, keep):
    """the in-plane search restated: -> (reference latents, [rows, A] query latents, best score per row,
    seeds, seed latents) with rows = B * Q"""
    from nope_b200.model import topk
    enc, u = model.u_net.encoder, model.u_net
    u.set_metric("l2")
    Bq = r.shape[0]
    rows = q.reshape(-1, 3, 256, 256)
    rf = enc.encode_image(r)
    qf = enc.encode_image_inplane(rows, A)                                          # [rows, A, C, 32, 32]
    N = rel.shape[1]
    sim = u.sweep(rf, rel, query_feat=qf.view(Bq, -1, *qf.shape[2:]), want_emb=False, want_sim=True)["sim"]
    top_v, flat = topk(sim.view(rows.shape[0], A * N), keep)
    n, a = flat % N, flat // N
    lat = qf[torch.arange(rows.shape[0], device=qf.device)[:, None], a]
    return rf, qf, top_v[:, 0], (n, a), lat


@pytest.fixture(scope="module")
def scene():
    from oracle import inputs
    g = torch.Generator().manual_seed(21)
    q = (torch.rand(B, Q, 3, 256, 256, generator=g) * 2 - 1).cuda()
    _, r = inputs.make_images(seed=9, batch=B)
    return {"q": q, "r": r.cuda()}


def test_refine_replays_through_the_oracle(gpu_model, grids, scene):
    from nope_b200.inplane_refine import propose, refine_inplane, select
    u, ref, rel = gpu_model.u_net, grids["ref"], grids["rel"]
    enc = u.encoder
    q, r = scene["q"], scene["r"]
    rf, _, best0, (n, a), lat0 = _search(gpu_model, q, r, rel, ref.angles, KEEP)
    rows = B * Q
    out = refine_inplane(u, enc, rf, q, rel, (n.view(B, Q, KEEP), a.view(B, Q, KEEP)),
                         lat0.view(B, Q, KEEP, *lat0.shape[2:]), ref, k=K)
    assert out["D"].shape == (B, Q, K, 3, 3) and out["cossin"].shape == (B, Q, K, 2)
    assert out["hypotheses"] == ref.steps * KEEP * 9 and out["crops"] == ref.steps * KEEP * 2
    ref_rows = rf[:, None].expand(B, Q, *rf.shape[1:]).reshape(rows, *rf.shape[1:])
    imgs = q.reshape(rows, 3, 256, 256)
    _, _, table = ref._on(rf.device)
    cur = {"D": torch.eye(3).reshape(1, 1, 9).expand(rows, KEEP, 9).contiguous().cuda(),
           "seed": n.to(torch.int32), "cossin": table[a].contiguous()}
    lat = lat0
    best = [best0.cpu()]
    for s in range(ref.steps):
        cand = propose(cur["D"], cur["seed"], cur["cossin"], rel, ref.stencils[s].cuda(), ref.rolls[s], Q)
        cand_o = orc.propose(cur["D"], cur["seed"], cur["cossin"], rel.cpu(), ref.stencils[s], ref.rolls[s], Q)
        for name in ("D", "seed", "rel", "poses", "cossin"):
            assert _equal(cand[name], cand_o[name]), (s, name)
        cs = cand["cossin"].view(rows, KEEP, 3, 2)
        idx = torch.arange(rows, device=rf.device, dtype=torch.int32)[:, None].expand(rows, KEEP * 2).reshape(-1)
        fresh = enc.encode_image_rotated(imgs, idx, cs[:, :, 1:].reshape(-1, 2)).view(rows, KEEP, 2, *rf.shape[1:])
        qf = torch.cat([lat[:, :, None], fresh], dim=2).view(rows, KEEP * 3, *rf.shape[1:])
        sim = u.sweep(ref_rows, cand["poses"], query_feat=qf, want_emb=False, want_sim=True)["sim"]
        n_out = K if s == ref.steps - 1 else KEEP
        cur = select(sim, cand, ref.thresholds[s], n_out)
        cur_o = orc.select(sim, cand_o, ref.thresholds[s], n_out)
        for name in ("D", "seed", "cossin", "aslot", "score", "rel"):
            assert _equal(cur[name], cur_o[name]), (s, name)
        lat = qf[torch.arange(rows, device=qf.device)[:, None], cur["aslot"].long().clamp_min(0)]
        best.append(cur["score"][:, 0].cpu())
        if s == 0:
            # the centre pair re-scores the search's best (angle, pose) to the same bits
            assert torch.equal(sim[:, 0, 0].cpu(), best0.cpu())
    for b0, b1 in zip(best, best[1:]):
        assert (b1 >= b0).all(), (b0, b1)
    assert _equal(out["score"].reshape(rows, K), cur["score"])
    assert _equal(out["D"].reshape(rows, K, 9), cur["D"]) and _equal(out["cossin"].reshape(rows, K, 2), cur["cossin"])
    assert torch.equal(out["latent"].reshape(rows, K, *rf.shape[1:]), lat)
    # every returned score is exactly a separate sweep of its (rel6d, latent)
    sc = torch.stack([u.sweep(ref_rows, out["rel6d"].reshape(rows, K, 6)[:, t:t + 1],
                              query_feat=out["latent"].reshape(rows, K, *rf.shape[1:])[:, t], want_emb=False,
                              want_sim=True)["sim"][:, 0] for t in range(K)], dim=1)
    assert torch.equal(sc, out["score"].reshape(rows, K))
    assert (out["score"][..., :-1] >= out["score"][..., 1:]).all()
    # is the returned latent the latent of that rolled crop encoded alone?
    alone = enc.encode_image_rotated(imgs, torch.arange(rows, device=rf.device, dtype=torch.int32),
                                     out["cossin"].reshape(rows, K, 2)[:, 0])
    print(f"returned latents equal encode_image_rotated of the crop alone: "
          f"{torch.equal(alone, out['latent'].reshape(rows, K, *rf.shape[1:])[:, 0])}")


def test_R_is_roll_times_D_times_the_seed_template(gpu_model, grids, scene):
    ref, rel, tp = grids["ref"], grids["rel"], torch.from_numpy(grids["R"])
    q, r = scene["q"], scene["r"]
    from nope_b200.inplane_refine import refine_inplane
    u = gpu_model.u_net
    rf, _, _, (n, a), lat = _search(gpu_model, q, r, rel, ref.angles, KEEP)
    out = refine_inplane(u, u.encoder, rf, q, rel, (n.view(B, Q, KEEP), a.view(B, Q, KEEP)),
                         lat.view(B, Q, KEEP, *lat.shape[2:]), ref, k=K)
    Rm, seed, alpha, score = gpu_model.predict_pose_inplane_refined(q, r, rel, ref, k=K, keep=KEEP)
    assert torch.equal(score, out["score"]) and torch.equal(seed, out["seed"])
    cs = out["cossin"].cpu().double()
    c, s = cs[..., 0].numpy(), cs[..., 1].numpy()
    Rz = np.zeros(c.shape + (3, 3))
    Rz[..., 0, 0], Rz[..., 0, 1], Rz[..., 1, 0], Rz[..., 1, 1], Rz[..., 2, 2] = c, -s, s, c, 1.0
    want = Rz @ out["D"].cpu().double().numpy() @ tp.numpy()[seed.cpu().numpy()]
    assert Rm.dtype == torch.float64 and np.allclose(Rm.cpu().numpy(), want, rtol=0, atol=1e-12)
    assert torch.allclose(alpha.cpu(), torch.rad2deg(torch.atan2(cs[..., 1], cs[..., 0])), rtol=0, atol=1e-12)


def test_query_forms_and_edge_cases(gpu_model, grids, scene):
    from nope_b200.inplane_refine import InplaneRefiner
    q, r, rel = scene["q"], scene["r"], grids["rel"]
    ref = grids["ref"]
    for qq, rr, rl, lead in ((q[:, 0], r, rel, (B,)), (q[0], r[:1], rel[:1], (Q,)), (q, r, rel, (B, Q))):
        R, seed, alpha, score = gpu_model.predict_pose_inplane_refined(qq, rr, rl, ref, k=K, keep=KEEP)
        assert R.shape == lead + (K, 3, 3) and seed.shape == alpha.shape == score.shape == lead + (K,)
        assert seed.dtype == torch.int64 and alpha.dtype == torch.float64 and R.dtype == torch.float64
        assert ((seed >= 0) & (seed < 642)).all() and torch.isfinite(score).all()
        assert (score[..., :-1] >= score[..., 1:]).all()
        Rc = R.cpu()
        assert torch.allclose(Rc @ Rc.transpose(-1, -2), torch.eye(3, dtype=torch.float64).expand_as(Rc), atol=1e-5)
        sim = gpu_model.predict_pose_inplane(qq, rr, rl, None, k=1, angles=ref.angles)[3]
        assert (score[..., 0] >= sim.flatten(-2).max(dim=-1).values).all()      # never below the search's best
    # A = 1 and keep = 1
    one = InplaneRefiner(grids["R"], angles=1, steps=2)
    R, seed, alpha, score = gpu_model.predict_pose_inplane_refined(q[:, 0], r, rel, one, k=3, keep=1)
    assert R.shape == (B, 3, 3, 3) and torch.isfinite(score).all()
    sim = gpu_model.predict_pose(q[:, 0], r, rel, k=1)[2]
    assert (score[:, 0] >= sim.max(dim=-1).values).all()


def test_does_not_synchronise(gpu_model, grids, scene):
    """predict_pose_inplane_refined on device inputs after one warm-up call, under torch's sync debug mode.  That
    mode sees synchronisation on the Python / torch side only: a synchronising call inside the library would not be
    caught here."""
    q, r, rel, ref = scene["q"], scene["r"], grids["rel"], grids["ref"]
    first = gpu_model.predict_pose_inplane_refined(q, r, rel, ref, k=K, keep=KEEP)
    with no_host_sync():
        out = gpu_model.predict_pose_inplane_refined(q, r, rel, ref, k=K, keep=KEEP)
    torch.cuda.synchronize()
    for x, y in zip(out, first):
        assert torch.equal(x, y)


# ------------------------------------------------------------------ roll recovery
class StubEngine:
    """sweep() scores every pose against one template, the encoder latent of image I: a score that depends on the
    roll of the query latent only (minus the mean squared difference)"""

    def __init__(self, template):
        self.t = template
        self.device = template.device

    def sweep(self, ref_feat, poses, query_feat=None, want_emb=False, want_sim=True, k=0):
        qf = query_feat if query_feat.dim() == 5 else query_feat[:, None]
        s = -((qf - self.t) ** 2).mean(dim=(-3, -2, -1))                               # [R, rows]
        sim = s[..., None].expand(*s.shape, poses.shape[1]).contiguous()
        return {"sim": sim if query_feat.dim() == 5 else sim[:, 0], "emb": None, "topv": None, "topi": None}


def _disc_image(g, size=256):
    """smooth asymmetric content inside the inscribed circle, -1 outside: rotations about the centre lose nothing"""
    ys, xs = torch.meshgrid(torch.arange(size, dtype=torch.float64), torch.arange(size, dtype=torch.float64),
                            indexing="ij")
    c = (size - 1) / 2
    img = torch.zeros(3, size, size, dtype=torch.float64)
    for ch in range(3):
        for _ in range(6):
            px, py = (torch.rand(2, generator=g, dtype=torch.float64) * 0.9 - 0.45) * size + c
            sig = float(torch.rand(1, generator=g, dtype=torch.float64)) * 18 + 8
            img[ch] += torch.exp(-((xs - px) ** 2 + (ys - py) ** 2) / (2 * sig * sig))
    img = img / img.amax(dim=(1, 2), keepdim=True) * 1.8 - 0.9
    inside = (xs - c) ** 2 + (ys - c) ** 2 <= (c - 2) ** 2
    return torch.where(inside, img, torch.tensor(-1.0, dtype=torch.float64)).float()


def test_roll_recovery_with_a_stub_engine(gpu_model, grids):
    """Queries: I rotated by seeded off-bin angles -beta; the stub's templates ignore the pose, so the search can
    only get the roll right.  The refined |alpha - beta| against the bin search's.  Measured on an H100 80GB HBM3:
    bin search median 2.002 degrees (max 4.949), refined median 0.166 (max 0.316); the gates leave about twice
    that."""
    from nope_b200.inplane_refine import InplaneRefiner, refine_inplane, roll_degrees, rotate_pairs
    enc = gpu_model.u_net.encoder
    g = torch.Generator().manual_seed(5)
    I = _disc_image(g).cuda()[None]
    stub = StubEngine(enc.encode_image(I))
    A, n_q, keep = 36, 24, 2
    ref = InplaneRefiner(grids["R"], angles=A, steps=4)
    beta = torch.rand(n_q, generator=g, dtype=torch.float64) * 360 - 180
    cs = torch.stack([torch.cos(torch.deg2rad(-beta)), torch.sin(torch.deg2rad(-beta))], dim=-1).float()
    qimg = rotate_pairs(I, torch.zeros(n_q, dtype=torch.int32).cuda(), cs.cuda())      # [n_q, 3, 256, 256]
    rel = grids["rel"][:1]
    qf = enc.encode_image_inplane(qimg, A)                                              # [n_q, A, C, 32, 32]
    rf = torch.zeros(1, enc.latent_dim, 32, 32, device=qf.device)
    sim = stub.sweep(rf, rel, qf.view(1, n_q * A, *qf.shape[2:]))["sim"].view(n_q, A * 642)
    flat = torch.sort(-sim, dim=1, stable=True).indices[:, :keep]
    n, a = flat % 642, flat // 642
    lat = qf[torch.arange(n_q, device=qf.device)[:, None], a]
    out = refine_inplane(stub, enc, rf, qimg[None], rel, (n[None], a[None]), lat[None], ref, k=1)
    alpha_bin = a[:, 0].double().cpu() * 360.0 / A
    alpha_ref = roll_degrees(out["cossin"][0, :, 0]).cpu()

    def err(x):
        return ((x - beta + 180) % 360 - 180).abs()

    e_bin, e_ref = err(alpha_bin), err(alpha_ref)
    print(f"roll recovery over {n_q} queries, A = {A}, keep = {keep}, {ref.steps} steps: bin search median "
          f"{float(e_bin.median()):.3f} deg (max {float(e_bin.max()):.3f}), refined median "
          f"{float(e_ref.median()):.3f} deg (max {float(e_ref.max()):.3f})")
    assert float(e_ref.median()) < 0.25 * float(e_bin.median())
    assert float(e_ref.median()) < 0.35 and float(e_ref.max()) < 0.7
