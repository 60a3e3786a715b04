"""TEST INFRASTRUCTURE ONLY -- write tests/golden/vsd.npz from the UNMODIFIED reference's `vsd_obj`
(src/poses/vsd.py:58-137) with only its renderer replaced: `pyrenderer` (pyrender / OpenGL, absent here) becomes
oracle.render_oracle.render, the restatement of nope_b200's depth rasterizer.

Synthetic frames: a box or a sphere at a ground-truth pose, rendered at 0.1 mm units into uint16 depth PNGs with an
occluding plate in front of part of the object, sensor noise and zero holes.  `vsd_obj` reads them with
cv2.imread(path, -1) / 10.0 from frame dicts in the shape it indexes (one per frame) and scores P = 5 estimated
rotations at the ground-truth translation.  Stored: the inputs (meshes, K, poses, raw depth) and the reference's
outputs -- VSD errors for "step" and "tlinear" at two (delta, tau) settings, and for frame 0, pose 2,
depth_im_to_dist_im_fast of the test and estimated depth and the two bop19 visibility masks.  Writes this one fixture
and nothing else.

Run in the build container (CPU):   python -m oracle.make_vsd
"""
import json
import os
import sys
import tempfile

import numpy as np

from . import inputs
from . import render_oracle as ro
from .ref_import import REFERENCE_ROOT, _install_stubs

H, W = 48, 64
K = np.array([[80.0, 0.0, 32.3], [0.0, 81.5, 23.7], [0.0, 0.0, 1.0]])
SETTINGS = [(15, 20), (5, 10)]          # (delta, tau): vsd_obj's defaults and a tighter pair
P = 5


def _rot(axis, deg):
    a = np.deg2rad(deg)
    axis = np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis)
    k = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(a) * k + (1 - np.cos(a)) * k @ k


def _scene(rng):
    meshes = [ro.box(60.0, 40.0, 30.0), ro.sphere(35.0, 1)]
    frames = [(0, (0.4, -0.3, 0.2), (3.0, -2.0, 250.0)), (1, (0.1, 0.7, -0.5), (-4.0, 1.0, 270.0)),
              (0, (-0.8, 0.5, 1.1), (2.0, 3.0, 240.0))]
    plate_v = np.array([[-200, -200, 0], [0, -200, 0], [0, 200, 0], [-200, 200, 0]], dtype=np.float32)
    plate_f = np.array([[0, 1, 2], [0, 2, 3]], dtype=np.int32)
    out = []
    for mi, rot, t in frames:
        gt = ro.look_pose(*rot, t=t).astype(np.float64)
        v, f = meshes[mi]
        obj = ro.render(v, f, gt, K, (H, W))[0].numpy()
        plate = ro.render(plate_v, plate_f, ro.look_pose(0, 0, 0.3, t=(-3.0, 0.0, t[2] - 40.0)), K, (H, W))[0].numpy()
        depth = np.where((plate > 0) & ((obj == 0) | (plate < obj)), plate, obj).astype(np.float64)
        depth = np.where(depth > 0, depth + rng.normal(0.0, 1.5, depth.shape), 0.0)
        depth[rng.random(depth.shape) < 0.05] = 0.0
        raw = np.round(depth * 10.0).clip(0, 65535).astype(np.uint16)
        preds = []
        for deg in (0.0, 4.0, 12.0, 35.0, 120.0):
            Rp = _rot(rng.normal(size=3), deg) @ gt[:3, :3]
            T = np.eye(4)
            T[:3, :3] = Rp
            T[:3, 3] = gt[:3, 3]
            preds.append(T)
        out.append(dict(mesh=mi, gt=gt, pred=np.stack(preds), raw=raw))
    return meshes, out


def write_vsd(out_dir=inputs.GOLDEN_DIR, seed=0):
    _install_stubs()
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    import cv2
    from src.poses import vsd as ref_vsd
    from src.poses.vsd_utils import depth_im_to_dist_im_fast, estimate_visib_mask_est, estimate_visib_mask_gt

    def renderer(obj_poses, BOP_cad_trimesh, intrinsic, img_size):           # pyrenderer's signature and output
        v, f = BOP_cad_trimesh
        if obj_poses.ndim == 2:
            obj_poses = obj_poses[None]
        return [d.numpy() for d in ro.render(v, f, obj_poses, intrinsic, tuple(img_size))]

    ref_vsd.pyrenderer = renderer
    rng = np.random.default_rng(seed)
    meshes, frames = _scene(rng)
    with tempfile.TemporaryDirectory() as tmp:
        data = []
        for i, fr in enumerate(frames):
            path = os.path.join(tmp, f"{i:06d}.png")
            assert cv2.imwrite(path, fr["raw"])
            data.append({"mesh": meshes[fr["mesh"]], "intrinsic": K.reshape(-1).tolist(), "depth_path": path,
                         "pred_poses": fr["pred"].copy(), "query_pose": fr["gt"].reshape(-1).tolist()})
        errs = {}
        for cost in ("step", "tlinear"):
            errs[cost] = np.stack([np.stack([ref_vsd.vsd_obj(i, data, delta_vsd=d, tau_vsd=t, cost_type=cost)
                                             for i in range(len(data))]) for d, t in SETTINGS])
        depth_test = cv2.imread(data[0]["depth_path"], -1) / 10.0
    fr = frames[0]
    v, f = meshes[fr["mesh"]]
    d_gt = ro.render(v, f, fr["gt"], K, (H, W))[0].numpy()
    d_est = ro.render(v, f, fr["pred"][2], K, (H, W))[0].numpy()
    dist_test = depth_im_to_dist_im_fast(depth_test, K)
    dist_gt = depth_im_to_dist_im_fast(d_gt, K)
    dist_est = depth_im_to_dist_im_fast(d_est, K)
    visib_gt = estimate_visib_mask_gt(dist_test, dist_gt, SETTINGS[0][0], visib_mode="bop19")
    visib_est = estimate_visib_mask_est(dist_test, dist_est, visib_gt, SETTINGS[0][0], visib_mode="bop19")
    np.savez_compressed(
        os.path.join(out_dir, "vsd.npz"),
        box_vertices=meshes[0][0], box_faces=meshes[0][1], sphere_vertices=meshes[1][0], sphere_faces=meshes[1][1],
        mesh_of_frame=np.array([fr["mesh"] for fr in frames], dtype=np.int64), K=K,
        gt_poses=np.stack([fr["gt"] for fr in frames]), pred_poses=np.stack([fr["pred"] for fr in frames]),
        depth_raw=np.stack([fr["raw"] for fr in frames]), settings=np.array(SETTINGS, dtype=np.float64),
        vsd_step=errs["step"], vsd_tlinear=errs["tlinear"],
        dist_test0=dist_test, dist_est0=dist_est, visib_gt0=visib_gt, visib_est0=visib_est)
    return {"frames": len(frames), "poses": P, "image": [H, W],
            "vsd_step": errs["step"].round(4).tolist(), "vsd_tlinear": errs["tlinear"].round(4).tolist()}


def main():
    print(json.dumps(write_vsd(), indent=1))


if __name__ == "__main__":
    sys.exit(main())
