"""CPU: template banks (DESIGN.md section 25) without a device -- the save / load round trip, every refusal of the
Python layer (before any device work) and the argument checks of nope_score_topk_grouped in the library."""
import ctypes as C
import types

import pytest
import torch

O, N, CL = 3, 5, 8


def _engine(channels=CL, precision="fp16", encoder_precision="split", name="UNet"):
    """a stand-in engine: what the descriptor reads, and a sweep that must never run"""
    def sweep(*a, **kw):
        raise AssertionError("device work before the refusal")
    cls = type(name, (), {})
    e = cls()
    e.channels, e.precision, e.device = channels, precision, torch.device("cpu")
    e.encoder = types.SimpleNamespace(precision=encoder_precision, latent_dim=channels)
    e.sweep = sweep
    return e


def _bank(ids=(4, 9, 2), seed=0, grid=None):
    from nope_b200.bank import TemplateBank, engine_descriptor
    g = torch.Generator().manual_seed(seed)
    n = len(ids)
    tp = torch.randn(N, 3, 3, generator=g, dtype=torch.float64) if grid is None else grid
    Ng = tp.shape[0]
    return TemplateBank(list(ids), torch.randn(n, Ng, CL, 32, 32, generator=g), torch.randn(n, CL, 32, 32, generator=g),
                        torch.randn(n, Ng, 6, generator=g), tp, engine_descriptor(_engine()))


def test_save_load_round_trip_is_bit_exact(tmp_path):
    from nope_b200.bank import TemplateBank
    b = _bank()
    b.templates[0, 1, 2, 3, 4] = -0.0
    b.templates[1, 0, 0, 0, 0] = float("nan")
    path = tmp_path / "bank.pt"
    b.save(path)
    c = TemplateBank.load(path, "cpu")
    assert c.obj_ids == b.obj_ids == (4, 9, 2) and c.engine == b.engine
    for name in ("templates", "reference_latents", "all_relativeR", "template_poses"):
        x, y = getattr(b, name), getattr(c, name)
        assert x.dtype == y.dtype and x.shape == y.shape
        assert torch.equal(x.view(torch.int32 if x.dtype == torch.float32 else torch.int64),
                           y.view(torch.int32 if y.dtype == torch.float32 else torch.int64)), name
    assert c.slots([2, 4, 2]) == [2, 0, 2]
    assert c.nbytes == O * N * CL * 4096 + O * CL * 4096 + O * N * 6 * 4 + N * 9 * 8
    assert (c.num_objects, c.num_poses, c.latent_dim) == (O, N, CL)


def test_load_refuses_other_files(tmp_path):
    from nope_b200.bank import TemplateBank
    b = _bank()
    b.save(tmp_path / "ok.pt")
    d = torch.load(tmp_path / "ok.pt", weights_only=True)
    for name, change in (("tag", {"format": "something else"}), ("version", {"version": 99}),
                         ("dtype", {"templates": d["templates"].double()}),
                         ("shape", {"reference_latents": d["reference_latents"][:2]}),
                         ("grid", {"template_poses": d["template_poses"][:4]}),
                         ("ids", {"obj_ids": torch.tensor([1, 1, 2])}),
                         ("engine", {"engine": {"engine": "UNet"}})):
        bad = dict(d, **change)
        torch.save(bad, tmp_path / f"{name}.pt")
        with pytest.raises(ValueError):
            TemplateBank.load(tmp_path / f"{name}.pt", "cpu")
    torch.save({"templates": d["templates"]}, tmp_path / "plain.pt")
    with pytest.raises(ValueError, match="not a template bank"):
        TemplateBank.load(tmp_path / "plain.pt", "cpu")


def test_build_refuses_before_the_sweep():
    from nope_b200.bank import TemplateBank
    e = _engine()
    ref, rel, tp = torch.zeros(3, CL, 32, 32), torch.zeros(3, N, 6), torch.zeros(N, 3, 3, dtype=torch.float64)
    with pytest.raises(ValueError, match="duplicate obj_ids"):
        TemplateBank.build(e, ref, [1, 2, 1], rel, tp)
    with pytest.raises(ValueError, match="ref_latents"):
        TemplateBank.build(e, torch.zeros(3, 4, 32, 32), [1, 2, 3], rel, tp)      # not the engine's latent shape
    with pytest.raises(ValueError, match="all_relativeR"):
        TemplateBank.build(e, ref, [1, 2, 3], rel[:2], tp)
    with pytest.raises(ValueError, match="template_poses"):
        TemplateBank.build(e, ref, [1, 2, 3], rel, tp[:4])                          # grid mismatch
    with pytest.raises(AssertionError, match="device work"):                        # the arguments are fine
        TemplateBank.build(e, ref, [1, 2, 3], rel, tp)


def test_constructor_refusals():
    from nope_b200.bank import TemplateBank
    b = _bank()
    args = [list(b.obj_ids), b.templates, b.reference_latents, b.all_relativeR, b.template_poses, b.engine]
    for i, bad in ((0, [4, 4, 2]), (1, b.templates.double()), (2, b.reference_latents[:, :4]), (3, b.all_relativeR[:, 1:]),
                   (4, b.template_poses.float()), (5, dict(b.engine, latent_dim=4)), (5, {"engine": "UNet"})):
        a = list(args)
        a[i] = bad
        with pytest.raises(ValueError):
            TemplateBank(*a)


def test_search_refusals():
    from nope_b200.bank import check_bank_search, search_bank
    b = _bank()
    e = _engine()
    q = torch.zeros(2, 4, CL, 32, 32)
    with pytest.raises(ValueError, match=r"no templates for obj_id \[7\]"):
        search_bank(b, q, [4, 7], e)
    with pytest.raises(ValueError, match="latent shape"):
        search_bank(b, torch.zeros(2, 4, 4, 32, 32), [4, 9], e)
    with pytest.raises(ValueError, match="obj_ids for"):
        search_bank(b, q, [4, 9, 2], e)
    with pytest.raises(ValueError, match="rebuild the bank"):
        search_bank(b, q, [4, 9], _engine(precision="bf16"))
    with pytest.raises(ValueError, match="rebuild the bank"):
        search_bank(b, q, [4, 9], _engine(encoder_precision="fp16"))
    with pytest.raises(ValueError, match="rebuild the bank"):
        search_bank(b, q, [4, 9], _engine(name="UNetModelPose"))
    with pytest.raises(ValueError, match="unknown similarity_metric"):
        search_bank(b, q, [4, 9], e, metric="dot")
    with pytest.raises(ValueError, match="k must be"):
        search_bank(b, q, [4, 9], e, k=65)
    with pytest.raises(ValueError, match="exceeds"):
        search_bank(b, torch.zeros(2, 1, CL, 32, 32), [4, 9], e, k=N + 1)
    with pytest.raises(ValueError, match="angles"):
        check_bank_search(b, e, 2, [4, 9], 0, 1)
    with pytest.raises(ValueError, match="TemplateBank"):
        check_bank_search(object(), e, 2, [4, 9], 4, 1)
    assert check_bank_search(b, e, 3, torch.tensor([2, 2, 9]), 4, 5) == (4, 5, [2, 2, 1])
    with pytest.raises(ValueError, match="pose grid"):
        b.check_grid(b.template_poses[:4])
    with pytest.raises(ValueError, match="pose grid"):
        b.check_grid(b.template_poses + 1e-12)
    b.check_grid(b.template_poses.clone())


def test_row_plan_groups_detections_by_slot():
    from nope_b200.bank import RowPlan
    p = RowPlan([2, 0, 2, 2, 0], 3, "cpu")
    assert p.G == 2 and p.gslots.tolist() == [0, 2] and p.row_off.tolist() == [0, 6, 15]
    assert p.order.tolist() == [1, 4, 0, 2, 3] and p.det_slots.tolist() == [2, 0, 2, 2, 0]
    x = torch.arange(5)
    assert torch.equal(p.restore(p.grouped(x)), x)
    q = RowPlan([0, 1, 1], 2, "cpu")
    assert q.order is None and q.inverse is None and q.row_off.tolist() == [0, 2, 6]


def _model(engine=None):
    from nope_b200.model import PoseConditional
    m = PoseConditional(engine or _engine())
    return m


def test_model_refusals_before_any_device_work():
    from nope_b200.inplane_refine import InplaneRefiner
    from nope_b200.poses import icosphere_object_rotations
    tp = torch.from_numpy(icosphere_object_rotations(0))                       # 42 poses
    b = _bank(grid=tp)
    m = _model()
    crops = torch.zeros(2, 3, 256, 256)
    with pytest.raises(ValueError, match=r"obj_id \[5\]"):
        m.predict_pose_bank(crops, [4, 5], b)
    with pytest.raises(ValueError, match="query"):
        m.predict_pose_bank(crops[0], [4], b)
    with pytest.raises(ValueError, match="k must be"):
        m.predict_pose_bank(crops, [4, 9], b, k=0)
    with pytest.raises(ValueError, match="rebuild the bank"):
        _model(_engine(channels=4)).predict_pose_bank(crops, [4, 9], b)
    m.testing_config.similarity_metric = "dot"
    with pytest.raises(ValueError, match="similarity_metric"):
        m.predict_pose_bank(crops, [4, 9], b)
    m.testing_config.similarity_metric = "l2"
    m.dist = object()
    for fn in (lambda: m.predict_pose_bank(crops, [4, 9], b),
               lambda: m.predict_pose_bank_refined(crops, [4, 9], b, InplaneRefiner(tp, 4, 1))):
        with pytest.raises(NotImplementedError, match="does not shard"):
            fn()
    m.dist = None
    with pytest.raises(ValueError, match="refiner"):
        m.predict_pose_bank_refined(crops, [4, 9], b, object())
    with pytest.raises(ValueError, match=r"\[B, 162, 6\]"):                   # another grid size
        m.predict_pose_bank_refined(crops, [4, 9], b, InplaneRefiner(torch.from_numpy(icosphere_object_rotations(1)), 4, 1))
    with pytest.raises(ValueError, match="pose grid"):                          # 42 poses, other rotations
        m.predict_pose_bank_refined(crops, [4, 9], b, InplaneRefiner(tp.flip(0), 4, 1))
    with pytest.raises(ValueError, match="keep"):
        m.predict_pose_bank_refined(crops, [4, 9], b, InplaneRefiner(tp, 4, 1), keep=17)
    with pytest.raises(ValueError, match="duplicate obj_ids"):
        m.build_template_bank([1, 1], torch.zeros(2, 3, 256, 256), torch.zeros(2, N, 6), torch.zeros(N, 3, 3))
    with pytest.raises(ValueError, match="template_poses"):
        m.build_template_bank([1, 2], torch.zeros(2, 3, 256, 256), torch.zeros(2, N, 6), torch.zeros(N + 1, 3, 3))


def test_predict_pose_frames_takes_a_bank_or_the_references():
    m = _model()
    b = _bank()
    for i in (4, 9):
        m.tless_cad[i] = object()
        m.bop_models[i] = {"diameter": 100.0}
    frames, masks = torch.zeros(1, 8, 8, 3, dtype=torch.uint8), torch.zeros(2, 8, 8, dtype=torch.uint8)
    K = torch.eye(3, dtype=torch.float64)
    with pytest.raises(ValueError, match="not both"):
        m.predict_pose_frames(frames, masks, K, [4, 9], torch.zeros(1, 3, 256, 256), torch.zeros(1, N, 6), None,
                              bank=b)
    with pytest.raises(ValueError, match="or a bank"):
        m.predict_pose_frames(frames, masks, K, [4, 9])
    with pytest.raises(ValueError, match=r"obj_id \[2\]"):
        m.tless_cad[2], m.bop_models[2] = object(), {"diameter": 1.0}
        m.predict_pose_frames(frames, masks, K, [4, 2], bank=_bank(ids=(4, 9, 3)))
    with pytest.raises(ValueError, match="rebuild the bank"):
        m.predict_pose_frames(frames, masks, K, [4, 9], bank=_bank_with(precision="parity"))


def _bank_with(**engine):
    from nope_b200.bank import TemplateBank, engine_descriptor
    b = _bank()
    return TemplateBank(list(b.obj_ids), b.templates, b.reference_latents, b.all_relativeR, b.template_poses,
                        engine_descriptor(_engine(**engine)))


# ------------------------------------------------------------------ the C ABI
def _fake():
    return C.c_void_p(256)       # never dereferenced: every call below fails its argument checks first


def _grouped(R=8, O=3, N=642, G=2, A=4, metric=0, k=5, null=None):
    from nope_b200 import _lib
    lib = _lib.load()
    p = [_fake() for _ in range(7)]
    if null is not None:
        p[null] = None
    rc = lib.nope_score_topk_grouped(p[0], p[1], R, O, N, CL, 1024, p[2], p[3], G, A, metric, 0.2, k, p[4], p[5],
                                     p[6], None)
    return rc, lib.nope_last_error().decode()


def test_grouped_abi_is_declared_and_bound():
    from nope_b200 import _lib
    assert "nope_score_topk_grouped" in _lib.SIGNATURES
    assert hasattr(_lib.load(), "nope_score_topk_grouped")
    assert _lib.load().nope_abi_version() == 3


def test_grouped_abi_refusals():
    for null in range(5):                                   # query, emb, slots, row_off, sim
        rc, msg = _grouped(null=null)
        assert rc == -1 and "null" in msg, null
    for null in (5, 6):                                     # top-k outputs, with k > 0
        rc, msg = _grouped(null=null)
        assert rc == -1 and "top-k" in msg
    for kw, word in (({"G": 0}, "G"), ({"G": 65536}, "G"), ({"R": 10, "A": 4}, "multiple of A"), ({"A": 0}, "A"),
                     ({"k": 65}, "k must"), ({"k": -1}, "k must"), ({"N": 3, "A": 1, "k": 4}, "k must"),
                     ({"O": 65536}, "too many"), ({"R": 4096, "A": 1, "N": 600000}, "too many"),
                     ({"metric": 3}, "metric"), ({"R": 0}, "bad arguments"), ({"N": 0}, "bad arguments")):
        rc, msg = _grouped(**kw)
        assert rc == -1 and word in msg, (kw, msg)
