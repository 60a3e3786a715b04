"""GPU: the T-LESS evaluation.  depth_raster_kernel against the torch oracle bit for bit, geometry that does not need
the oracle (exact plane depths, sample positions, watertight shared edges, order and winding independence, batching),
vsd_kernel against the unmodified reference's values (tests/golden/vsd.npz) and the oracle, and eval_vsd / test_step
end to end on a synthetic tless_obj01 batch.  The weights are seeded: the VSD numbers say nothing about a trained
model."""
import os

import numpy as np
import pytest
import torch

from _scenes import K3, tless_batch
from _util import no_host_sync, same_bits
from oracle import render_oracle as ro

pytestmark = pytest.mark.gpu

def _render(v, f, poses, K, size, znear=0.05):
    from nope_b200.vsd import Mesh, render_depth
    return render_depth(Mesh(v, f), torch.as_tensor(np.asarray(poses)), K, size, znear=znear).cpu()


# ------------------------------------------------------------------ kernel vs oracle
_K_SMALL = (120.0, 118.0, 40.3, 29.8)
_POSES = np.stack([ro.look_pose(0.3, -0.4, 0.2, t=(0, 0, 300)),
                   ro.look_pose(1.1, 0.2, -0.7, t=(60, -20, 250)),       # across the image border
                   ro.look_pose(0.0, 0.0, 0.0, t=(2000, 0, 300)),        # fully off-screen
                   ro.look_pose(0.2, 0.1, 0.0, t=(0, 0, 45)),            # covers the whole image, some vertices
                   ro.look_pose(2.0, 1.0, 0.5, t=(-5, 4, 200))])         # another view (znear and the 2^20 px
                                                                          # bound: their own tests below)


@pytest.mark.parametrize("mesh", ["box", "sphere", "soup", "plane"])
def test_render_matches_oracle(mesh):
    v, f = {"box": ro.box, "sphere": lambda: ro.sphere(40.0, 2), "soup": lambda: ro.soup(96, seed=3),
            "plane": lambda: ro.plane(7, 5)}[mesh]()
    out = _render(v, f, _POSES, _K_SMALL, (60, 80))
    ref = ro.render(v, f, _POSES, _K_SMALL, (60, 80))
    assert out.shape == (len(_POSES), 60, 80)
    assert same_bits(out, ref)
    assert (out[0] > 0).any() and (out[2] == 0).all()


def test_render_full_cover_edges_through_samples_and_ties():
    """a quad larger than the image; triangles whose edges run through sample centres (integer + 1/2 in every
    coordinate at Z = f); two coplanar overlapping triangles (exact depth ties)"""
    Z, fpx = 100.0, 100.0
    K = (fpx, fpx, 0.0, 0.0)
    big = np.array([[-50, -50, Z], [500, -50, Z], [500, 500, Z], [-50, 500, Z]], dtype=np.float32)
    edges = np.array([[1.5, 1.5, Z], [9.5, 1.5, Z], [1.5, 7.5, Z], [9.5, 7.5, Z], [5.5, 4.5, Z]], dtype=np.float32)
    v = np.concatenate([big, edges, edges + np.array([0, 0, 0], np.float32)])
    f = np.array([[0, 1, 2], [0, 2, 3], [4, 5, 6], [5, 7, 6], [4, 5, 8], [9, 10, 11], [10, 12, 11]], dtype=np.int32)
    pose = np.eye(4, dtype=np.float32)
    for faces in (f[:2], f[2:4], f[4:], f):
        out = _render(v, faces, pose[None], K, (12, 16))
        assert same_bits(out, ro.render(v, faces, pose, K, (12, 16)))
    assert (_render(v, f[:2], pose[None], K, (12, 16)) == 100.0).all()


def test_render_tless_size_matches_oracle():
    v, f = ro.sphere(45.0, 2)
    poses = np.stack([ro.look_pose(0.3, 0.2, 0.1, t=(10, -15, 600)), ro.look_pose(-0.5, 0.9, 0.0, t=(-250, 120, 500))])
    out = _render(v, f, poses, K3, (540, 720))
    assert same_bits(out, ro.render(v, f, poses, K3, (540, 720)))
    assert (out > 0).sum() > 1000


# ------------------------------------------------------------------ geometry without the oracle
def test_plane_depths():
    """a fronto-parallel plane renders its Z exactly; a tilted plane matches the ray-plane depth within 1e-6"""
    v, f = ro.plane(6, 4, 400.0, 300.0)
    K = (150.0, 150.0, 32.0, 24.0)
    out = _render(v, f, ro.look_pose(t=(0, 0, 321.25))[None], K, (48, 64))[0]
    assert (out == 321.25).all()
    # snapping a vertex by up to 1/512 px moves the depth by (1/512) tan(tilt) / f of itself: 1e-7 here
    K, (H, W) = (1075.0, 1073.0, 360.0, 270.0), (540, 720)
    pose = ro.look_pose(0.2, -0.1, 0.0, t=(0, 0, 300))
    out = _render(v, f, pose[None], K, (H, W))[0].double()
    R, t = pose[:3, :3].astype(np.float64), pose[:3, 3].astype(np.float64)
    n = R[:, 2]                                                   # plane normal in the camera frame, passing through t
    c, r = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)
    ray = np.stack([(c - 360.0) / 1075.0, (r - 270.0) / 1073.0, np.ones_like(c)], axis=-1)
    z = (n @ t) / (ray @ n)
    hit = out.numpy() > 0
    assert hit.mean() > 0.9
    assert np.abs(out.numpy()[hit] - z[hit]).max() / z[hit].max() < 1e-6


def test_triangle_lands_in_its_pixel():
    K = (100.0, 100.0, 0.0, 0.0)
    for r, c in ((0, 0), (3, 5), (7, 9)):
        pts = np.array([[c + 0.3, r + 0.3], [c + 0.8, r + 0.4], [c + 0.5, r + 0.8]])
        v = np.concatenate([pts, np.full((3, 1), 100.0)], axis=1).astype(np.float32)      # u = X, v = Y
        out = _render(v, np.array([[0, 1, 2]], dtype=np.int32), np.eye(4)[None], K, (8, 10))[0]
        assert out.nonzero().tolist() == [[r, c]] and out[r, c] == 100.0


def test_shared_edge_is_watertight():
    """two triangles sharing a diagonal through sample centres, rendered one at a time: disjoint, union = the quad"""
    K = (100.0, 100.0, 0.0, 0.0)
    Z = 100.0
    q = np.array([[0.5, 0.5], [12.5, 0.5], [12.5, 12.5], [0.5, 12.5]])
    v = np.concatenate([q, np.full((4, 1), Z)], axis=1).astype(np.float32)               # u = X, v = Y
    for tris in (([0, 1, 2], [0, 2, 3]), ([0, 1, 3], [1, 2, 3])):
        a = _render(v, np.array([tris[0]], dtype=np.int32), np.eye(4)[None], K, (14, 14))[0] > 0
        b = _render(v, np.array([tris[1]], dtype=np.int32), np.eye(4)[None], K, (14, 14))[0] > 0
        both = _render(v, np.array(tris, dtype=np.int32), np.eye(4)[None], K, (14, 14))[0] > 0
        assert not (a & b).any()
        assert torch.equal(a | b, both)
        assert both.sum() == 12 * 12 and both[:12, :12].all()      # the quad owns its top and left edges only


def test_tessellated_plane_has_no_holes():
    """poses at which the plane covers the whole image: every pixel is hit"""
    v, f = ro.plane(23, 17, 400.0, 300.0)
    for pose in (ro.look_pose(0.2, -0.1, 0.3, t=(0, 0, 200)), ro.look_pose(0.5, 0.3, 1.3, t=(3, -2, 120)),
                 ro.look_pose(0.6, -0.4, 2.0, t=(-2, 3, 110))):
        out = _render(v, f, pose[None], (90.0, 90.0, 40.0, 30.0), (60, 80))[0]
        assert (out > 0).all()


def test_winding_order_and_batch_independence():
    v, f = ro.sphere(40.0, 3)
    poses = np.stack([ro.look_pose(0.1 * i, -0.2 * i, 0.3, t=(5 * i, -3 * i, 260)) for i in range(6)])
    K = (130.0, 128.0, 48.7, 36.1)
    base = _render(v, f, poses, K, (72, 96))
    perm = np.random.default_rng(0).permutation(len(f))
    rolled = np.roll(f[perm], 1, axis=1)
    assert same_bits(_render(v, f[:, [0, 2, 1]], poses, K, (72, 96)), base)
    assert same_bits(_render(v, rolled, poses, K, (72, 96)), base)
    for p in (0, 3, 5):
        assert same_bits(_render(v, f, poses[p:p + 1], K, (72, 96)), base[p:p + 1])


def test_faces_out_of_range_are_skipped_by_the_kernel():
    from nope_b200 import _lib
    from nope_b200.vsd import Mesh, render_depth
    v, f = ro.box()
    m = Mesh(v, f)
    m.faces = torch.cat([m.faces, torch.tensor([[0, 1, 99], [-5, 1, 2]], dtype=torch.int32, device="cuda")])
    out = render_depth(m, ro.look_pose(0.3, 0.2, 0.0, t=(0, 0, 300)), _K_SMALL, (60, 80)).cpu()
    ref = ro.render(v, f, ro.look_pose(0.3, 0.2, 0.0, t=(0, 0, 300)), _K_SMALL, (60, 80))
    assert same_bits(out, ref)
    assert (out > 0).any()
    m.faces = torch.tensor([[0, 1, 99], [-5, 1, 2], [2, 3, 8]], dtype=torch.int32, device="cuda")
    assert (render_depth(m, ro.look_pose(0.3, 0.2, 0.0, t=(0, 0, 300)), _K_SMALL, (60, 80)) == 0).all()
    with pytest.raises(_lib.NopeError):
        _lib.check(_lib.load().nope_render_depth(None, 8, None, 1, None, 1, 1.0, 1.0, 0.0, 0.0, 0.05, 4, 4, None,
                                                 None))


def _guard_case(v, f, drop, K, size, znear):
    """render all faces together and the kept ones alone: bitwise equal to the oracle, the dropped faces leave their
    pixels at 0 and the kept faces (neighbours of the dropped ones) render exactly as without them"""
    pose = np.eye(4, dtype=np.float32)[None]
    f = np.asarray(f, dtype=np.int32)
    keep = [i for i in range(len(f)) if i not in drop]
    every = _render(v, f, pose, K, size, znear)[0]
    assert same_bits(every, ro.render(v, f, pose, K, size, znear)[0])
    kept = _render(v, f[keep], pose, K, size, znear)[0]
    assert same_bits(every, kept)
    for i in range(len(f)):
        alone = _render(v, f[i:i + 1], pose, K, size, znear)[0]
        assert same_bits(alone, ro.render(v, f[i:i + 1], pose, K, size, znear)[0])
        assert ((alone > 0).sum() == 0) == (i in drop), i
    return every


def test_znear_drop():
    """a triangle is dropped when one vertex has camera Z < znear (compared in float32): Z one float32 step below znear,
    0, -0 and negative are dropped; Z exactly znear and one step above are kept.  Each triangle's apex sits at that Z,
    its base at Z = 100 mm, in its own column band next to a kept neighbour"""
    znear = 0.05
    zn = np.float32(znear)
    zs = [np.nextafter(zn, np.float32(0)), zn, np.nextafter(zn, np.float32(1)), np.float32(0.0), np.float32(-0.0),
          np.float32(-5.0)]
    K, size = (100.0, 100.0, 0.0, 0.0), (40, 8 + 14 * len(zs))
    v, f, drop = [], [], []
    for i, z in enumerate(zs):
        u = 8.0 + 14 * i
        apex = [z * u / 100.0, z * 6.0 / 100.0, z] if z > 0 else [u, 6.0, z]
        v += [apex, [u - 5.5, 30.5, 100.0], [u + 5.5, 30.5, 100.0],                 # the case (u = X, v = Y at Z = 100)
              [u - 5.5, 31.5, 100.0], [u + 5.5, 31.5, 100.0], [u, 38.5, 100.0]]     # its neighbour, always kept
        f += [[6 * i, 6 * i + 1, 6 * i + 2], [6 * i + 3, 6 * i + 4, 6 * i + 5]]
        if not z >= zn:
            drop.append(2 * i)
    assert len(drop) == 4
    every = _guard_case(np.array(v, dtype=np.float32), f, drop, K, size, znear)
    for i, z in enumerate(zs):
        band = every[:, 14 * i + 2:14 * i + 14]
        assert ((band[:31] > 0).sum() > 0) == (z >= zn), i               # the apex triangle's rows
        assert (band[32:] > 0).sum() > 0                                  # the neighbour's rows


@pytest.mark.parametrize("axis", [0, 1])
@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_projected_coordinate_bound(axis, sign):
    """fx = fy = 1024, c = 0, Z = 1: a vertex at X (or Y) = +-1024 projects exactly to +-2^20 px and is kept; one float32
    step further (+-2^20 + 1/8 px) drops its triangle.  Both triangles reach from that vertex into the image"""
    K, size = (1024.0, 1024.0, 0.0, 0.0), (48, 64)
    far_in = np.float32(1024.0)
    far_out = np.nextafter(far_in, np.float32(2048.0))
    assert float(np.float32(1024.0) * far_out) == 2.0 ** 20 + 0.125
    v, f = [], []
    for j, far in enumerate((far_in, far_out)):
        base = [(10.5 + 20 * j) * 100.0 / 1024.0, 100.0 * 20.5 / 1024.0], [(10.5 + 20 * j) * 100.0 / 1024.0,
                                                                            100.0 * 40.5 / 1024.0]
        if axis == 1:
            base = [b[::-1] for b in base]
        apex = [sign * far, 0.0] if axis == 0 else [0.0, sign * far]
        base = [[b[0], b[1], 100.0] for b in base]
        if sign < 0:   # reach into the image from the negative side: the base on the far edge
            base = [[b[0] + (60.0 * 100.0 / 1024.0 if axis == 0 else 0.0),
                     b[1] + (40.0 * 100.0 / 1024.0 if axis == 1 else 0.0), 100.0] for b in base]
        v += [apex + [1.0]] + base
        f.append([3 * j, 3 * j + 1, 3 * j + 2])
    v = np.array(v, dtype=np.float32)
    every = _guard_case(v, f, [1], K, size, 0.05)
    assert (every > 0).sum() > 20
    # the inside vertex really lies at the bound
    uv = ro._project(torch.from_numpy(v), torch.eye(4), 1024.0, 1024.0, 0.0, 0.0, 0.05)
    assert int(uv[axis][0]) == int(sign * 2 ** 28) and bool(uv[3][0]) and not bool(uv[3][3])


# ------------------------------------------------------------------ VSD kernel
@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "vsd.npz")))


def _golden_inputs(g):
    F, H, W = g["depth_raw"].shape
    gt, est = [], []
    for i in range(F):
        name = ("box", "sphere")[int(g["mesh_of_frame"][i])]
        v, f = g[f"{name}_vertices"], g[f"{name}_faces"]
        gt.append(_render(v, f, g["gt_poses"][i][None], g["K"], (H, W))[0])
        est.append(_render(v, f, g["pred_poses"][i], g["K"], (H, W)))
    return torch.from_numpy(g["depth_raw"] / 10.0), torch.stack(gt), torch.stack(est)


def test_vsd_matches_the_reference(golden):
    from nope_b200.vsd import vsd_errors
    dt, dg, de = _golden_inputs(golden)
    K = torch.from_numpy(np.repeat(golden["K"][None], len(dt), axis=0))
    for s, (delta, tau) in enumerate(golden["settings"]):
        step = vsd_errors(dt.cuda(), dg.cuda(), de.cuda(), K, int(delta), int(tau), "step").cpu().numpy()
        assert np.array_equal(step, golden["vsd_step"][s]), (step, golden["vsd_step"][s])
        tl = vsd_errors(dt.cuda(), dg.cuda(), de.cuda(), K, int(delta), int(tau), "tlinear").cpu().numpy()
        assert np.allclose(tl, golden["vsd_tlinear"][s], rtol=1e-12, atol=0)


def test_vsd_on_gpu_renders_matches_oracle():
    from nope_b200.vsd import vsd_errors
    v, f = ro.sphere(45.0, 2)
    gt = ro.look_pose(0.3, 0.2, 0.1, t=(10, -15, 600))
    preds = np.stack([ro.look_pose(0.3 + d, 0.2 - d, 0.1, t=(10, -15, 600)) for d in (0.0, 0.05, 0.2, 0.6, 1.5)])
    dg = _render(v, f, gt[None], K3, (540, 720))[0]
    de = _render(v, f, preds, K3, (540, 720))
    rng = np.random.default_rng(1)
    dt = dg.double().numpy() + rng.normal(0, 2.0, dg.shape) * (dg.numpy() > 0)
    dt[rng.random(dt.shape) < 0.05] = 0
    dt = np.round(dt * 10) / 10.0
    for cost in ("step", "tlinear"):
        out = vsd_errors(torch.from_numpy(dt)[None].cuda(), dg[None].cuda(), de[None].cuda(), K3[None],
                         cost_type=cost).cpu().numpy()[0]
        ref = ro.vsd(dt, dg.numpy(), de.numpy(), K3, cost_type=cost)
        if cost == "step":
            assert np.array_equal(out, ref), (out, ref)
        else:
            assert np.allclose(out, ref, rtol=1e-12, atol=0)


def test_vsd_empty_union_and_perfect_pose():
    from nope_b200.vsd import vsd_errors
    H, W = 30, 40
    z = torch.zeros(1, H, W, dtype=torch.float64, device="cuda")
    K = torch.tensor([[50.0, 50.0, 20.0, 15.0]], dtype=torch.float64)
    out = vsd_errors(z, z.float(), z.float()[:, None].expand(1, 3, H, W), K)
    assert out.cpu().tolist() == [[1.0, 1.0, 1.0]]
    v, f = ro.box()
    d = _render(v, f, ro.look_pose(0.4, 0.3, 0.0, t=(0, 0, 200))[None], K[0].numpy(), (H, W))
    out = vsd_errors(d.double().cuda(), d.cuda(), d[:, None].cuda(), K, cost_type="tlinear")
    assert out.cpu().tolist() == [[0.0]]
    occl = torch.where(d > 0, d - 50, d).double()            # something 50 mm in front: nothing visible, union empty
    assert vsd_errors(occl.cuda(), d.cuda(), d[:, None].cuda(), K).cpu().tolist() == [[1.0]]


# ------------------------------------------------------------------ eval_vsd / test_step end to end
def test_eval_vsd_end_to_end(gpu_model, tmp_path, monkeypatch):
    import cv2
    from nope_b200 import vsd as V
    batch, cad, _ = tless_batch(tmp_path, models_info=False)
    B = batch["query"].shape[0]
    model = gpu_model
    model.load_mesh(cad, obj_ids=[1])
    model.log_dir = str(tmp_path / "pred")
    model.logged = {}
    # no host synchronisation inside the render and VSD calls
    calls = {"render": 0, "vsd": 0}
    render, vsd = V.render_depth, V.vsd_errors

    def strict(fn, name):
        def inner(*a, **kw):
            calls[name] += 1
            with no_host_sync():
                return fn(*a, **kw)
        return inner
    monkeypatch.setattr(V, "render_depth", strict(render, "render"))
    monkeypatch.setattr(V, "vsd_errors", strict(vsd, "vsd"))
    out = model.test_step({"tless_obj01": batch}, 4)["tless_obj01"]
    assert calls == {"render": B, "vsd": 1}
    monkeypatch.undo()
    keys = [f"top {k}, vsd_median" for k in (1, 3, 5)] + [f"top {k}, vsd_scores 0.3" for k in (1, 3, 5)]
    assert sorted(out) == sorted(keys)
    assert "loss/val_obj01" in model.logged
    for k in keys:
        assert model.logged[f"{k}/val_obj01"] == [float(out[k])]
    # recompute from the returned poses
    _, idx, _ = model.predict_pose(batch["query"], batch["reference"], batch["all_relativeR"], None, k=5)
    idx = idx.cpu()
    mesh = V.Mesh(*ro.box(60.0, 40.0, 30.0))
    err = []
    for b in range(B):
        poses = np.zeros((6, 4, 4), dtype=np.float32)
        poses[0, :3, :3] = batch["query_pose"][b].numpy()
        poses[1:, :3, :3] = batch["template_poses"][b, idx[b]].numpy()
        poses[:, :3, 3] = batch["query_translation"][b, :, 0].numpy()
        poses[:, 3, 3] = 1
        d = V.render_depth(mesh, torch.from_numpy(poses), batch["intrinsic"][b], (72, 96))
        dt = torch.from_numpy(cv2.imread(batch["depth_path"][b], -1) / 10.0).cuda()
        err.append(V.vsd_errors(dt[None], d[None, 0], d[None, 1:], batch["intrinsic"][b:b + 1])[0].cpu().numpy())
    err = np.stack(err)
    for k in (1, 3, 5):
        best = err[:, :k].min(1)
        assert out[f"top {k}, vsd_median"] == np.median(best)
        assert out[f"top {k}, vsd_scores 0.3"] == np.mean((best <= 0.3) * 100.0)
    saved = np.load(os.path.join(model.log_dir, "vsd_obj01_batch4_rank_0.npy"))
    assert np.array_equal(saved, err[:, 0])
    # nothing saved without a log_dir
    model.log_dir = None
    model.eval_vsd(batch, "obj01")
    assert os.listdir(str(tmp_path / "pred")) == ["vsd_obj01_batch4_rank_0.npy"]
