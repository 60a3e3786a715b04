"""Template banks (DESIGN.md section 25): every object's reference swept once over the pose grid, its templates kept,
and every detection searched against its own object's stored templates.

The templates depend on the reference image, the grid and the weights, never on the query, so a frame pipeline that
sweeps each detection's reference repeats the same sweep for every detection of the object.  A `TemplateBank` holds
the result of one sweep over all objects; a search against it encodes the detection's rotated crops and scores them
against the object's templates (`nope_score_topk_grouped`: rows grouped by template set, each template read once per
group), with the arithmetic of `nope_score_topk_multi`, so the scores are those of `retrieval_inplane` against that
object's templates bit for bit.

A bank records what its templates depend on besides the weights: the engine class, its latent channels, the UNet's
precision and the encoder's.  A search refuses a model whose descriptor differs.  It cannot see a change of weights
under the same architecture and precision: a bank built before `load_state_dict` of other weights is stale, and it is
the caller's to rebuild it.  The bank is independent of the similarity metric: a search scores with the model's
current metric and threshold.  Written against any engine with `sweep()` (`UNet`, `UNetModelPose`)."""

import torch

from . import _lib
from .inplane import check_inplane_args
from .search import _METRICS, check_metric

FORMAT = "nope_b200.template_bank"
VERSION = 1
_DESCRIPTOR_KEYS = ("engine", "latent_dim", "precision", "encoder_precision")


def engine_descriptor(engine):
    """What a bank's templates depend on besides the weights: {"engine": class name, "latent_dim", "precision" (the
    UNet's), "encoder_precision" (None without an encoder)}"""
    enc = getattr(engine, "encoder", None)
    return {"engine": type(engine).__name__, "latent_dim": int(engine.channels), "precision": str(engine.precision),
            "encoder_precision": None if enc is None else getattr(enc, "precision", None)}


def _ids(obj_ids):
    """obj_ids (a sequence, numpy array or tensor) -> list of Python ints, read on the host"""
    if torch.is_tensor(obj_ids):
        obj_ids = obj_ids.detach().cpu().reshape(-1).tolist()
    try:
        return [int(i) for i in obj_ids]
    except TypeError:
        return [int(i) for i in list(obj_ids.reshape(-1))]


class TemplateBank:
    """The templates of O objects over one pose grid of N poses, on one device:
      obj_ids            tuple of O unique ints (host); slot o holds object obj_ids[o]
      templates          float32 [O, N, C, 32, 32]: the sweep's embeddings of reference o at all_relativeR[o]
      reference_latents  float32 [O, C, 32, 32]
      all_relativeR      float32 [O, N, 6]
      template_poses     float64 [N, 3, 3]: the grid's rotations, one for every object
      engine             engine_descriptor() of the engine that swept them
    Memory: templates take O * N * C * 4 KiB (32 KiB per template at C = 8)."""

    def __init__(self, obj_ids, templates, reference_latents, all_relativeR, template_poses, engine):
        ids = _ids(obj_ids)
        if len(set(ids)) != len(ids):
            dup = sorted(set(i for i in ids if ids.count(i) > 1))
            raise ValueError(f"TemplateBank: duplicate obj_ids {dup}")
        O = len(ids)
        if O < 1:
            raise ValueError("TemplateBank: no objects")
        for name, t, dt in (("templates", templates, torch.float32), ("reference_latents", reference_latents,
                             torch.float32), ("all_relativeR", all_relativeR, torch.float32),
                            ("template_poses", template_poses, torch.float64)):
            if not torch.is_tensor(t) or t.dtype != dt:
                raise ValueError(f"TemplateBank: {name} must be a {dt} tensor")
        if templates.dim() != 5 or templates.shape[0] != O or tuple(templates.shape[3:]) != (32, 32) \
                or templates.shape[1] < 1:
            raise ValueError(f"TemplateBank: templates [O = {O}, N, C, 32, 32] expected, got {tuple(templates.shape)}")
        _, N, Cl = templates.shape[:3]
        for name, t, shape in (("reference_latents", reference_latents, (O, Cl, 32, 32)),
                               ("all_relativeR", all_relativeR, (O, N, 6)), ("template_poses", template_poses, (N, 3, 3))):
            if tuple(t.shape) != shape:
                raise ValueError(f"TemplateBank: {name} {shape} expected, got {tuple(t.shape)}")
        dev = templates.device
        if any(t.device != dev for t in (reference_latents, all_relativeR, template_poses)):
            raise ValueError("TemplateBank: every tensor must be on the templates' device")
        if not isinstance(engine, dict) or set(engine) != set(_DESCRIPTOR_KEYS):
            raise ValueError(f"TemplateBank: engine must be a descriptor with the keys {_DESCRIPTOR_KEYS}")
        if engine["latent_dim"] != Cl:
            raise ValueError(f"TemplateBank: the engine's latent_dim {engine['latent_dim']} is not the templates' {Cl}")
        self.obj_ids = tuple(ids)
        self._slot = {i: o for o, i in enumerate(ids)}
        self.templates = templates.contiguous()
        self.reference_latents = reference_latents.contiguous()
        self.all_relativeR = all_relativeR.contiguous()
        self.template_poses = template_poses.contiguous()
        self._template_poses_host = template_poses.detach().cpu()
        self.engine = dict(engine)

    @property
    def device(self):
        return self.templates.device

    @property
    def num_objects(self):
        return len(self.obj_ids)

    @property
    def num_poses(self):
        return int(self.templates.shape[1])

    @property
    def latent_dim(self):
        return int(self.templates.shape[2])

    @property
    def nbytes(self):
        """bytes of the stored tensors on the device"""
        return sum(t.numel() * t.element_size() for t in (self.templates, self.reference_latents, self.all_relativeR,
                                                            self.template_poses))

    # ------------------------------------------------------------------ construction and persistence
    @classmethod
    @torch.no_grad()
    def build(cls, engine, ref_latents, obj_ids, all_relativeR, template_poses):
        """One sweep with want_emb=True of all O references: ref_latents [O, C, 32, 32] (C = the engine's latent
        channels), all_relativeR [O, N, 6], template_poses [N, 3, 3] (the grid's rotations).  The engine chunks the
        O * N hypotheses itself.  Every argument is checked before any device work."""
        ids = _ids(obj_ids)
        if len(set(ids)) != len(ids):
            dup = sorted(set(i for i in ids if ids.count(i) > 1))
            raise ValueError(f"TemplateBank.build: duplicate obj_ids {dup}")
        O, Cl = len(ids), int(engine.channels)
        if O < 1 or tuple(ref_latents.shape) != (O, Cl, 32, 32):
            raise ValueError(f"TemplateBank.build: ref_latents [{O}, {Cl}, 32, 32] expected (one per obj_id, the "
                             f"engine's latent channels), got {tuple(ref_latents.shape)}")
        if all_relativeR.dim() != 3 or all_relativeR.shape[0] != O or all_relativeR.shape[2] != 6 \
                or all_relativeR.shape[1] < 1:
            raise ValueError(f"TemplateBank.build: all_relativeR [{O}, N, 6] expected, got "
                             f"{tuple(all_relativeR.shape)}")
        N = all_relativeR.shape[1]
        tp = torch.as_tensor(template_poses)
        if tuple(tp.shape) != (N, 3, 3):
            raise ValueError(f"TemplateBank.build: template_poses [{N}, 3, 3] expected (the grid of all_relativeR), "
                             f"got {tuple(tp.shape)}")
        dev = engine.device
        emb = engine.sweep(ref_latents, all_relativeR, want_emb=True)["emb"]
        return cls(ids, emb, ref_latents.to(dev, torch.float32), all_relativeR.to(dev, torch.float32),
                   tp.to(dev, torch.float64), engine_descriptor(engine))

    def save(self, path):
        """torch.save of the bank's tensors on the host, with the format tag and version"""
        torch.save({"format": FORMAT, "version": VERSION,
                    "obj_ids": torch.tensor(self.obj_ids, dtype=torch.int64),
                    "templates": self.templates.cpu(), "reference_latents": self.reference_latents.cpu(),
                    "all_relativeR": self.all_relativeR.cpu(), "template_poses": self.template_poses.cpu(),
                    "engine": dict(self.engine)}, path)

    @classmethod
    def load(cls, path, device):
        """A bank written by save(), onto `device`: torch.load(weights_only=True), the format tag, version, shapes and
        dtypes checked (ValueError)."""
        d = torch.load(path, map_location="cpu", weights_only=True)
        if not isinstance(d, dict) or d.get("format") != FORMAT:
            raise ValueError(f"{path}: not a template bank (format tag {FORMAT!r} missing)")
        if d.get("version") != VERSION:
            raise ValueError(f"{path}: template bank version {d.get('version')!r}, this package reads {VERSION}")
        keys = ("obj_ids", "templates", "reference_latents", "all_relativeR", "template_poses", "engine")
        missing = [k for k in keys if k not in d]
        if missing:
            raise ValueError(f"{path}: template bank without {missing}")
        ids = d["obj_ids"]
        if not torch.is_tensor(ids) or ids.dtype != torch.int64 or ids.dim() != 1:
            raise ValueError(f"{path}: obj_ids must be an int64 [O] tensor")
        dev = torch.device(device)
        return cls(ids.tolist(), d["templates"].to(dev), d["reference_latents"].to(dev), d["all_relativeR"].to(dev),
                   d["template_poses"].to(dev), d["engine"])

    # ------------------------------------------------------------------ checks
    def slots(self, obj_ids):
        """the bank slot of every id (host ints); ValueError naming the ids the bank does not hold"""
        ids = _ids(obj_ids)
        missing = sorted(set(i for i in ids if i not in self._slot))
        if missing:
            raise ValueError(f"template bank has no templates for obj_id {missing} (it holds {list(self.obj_ids)})")
        return [self._slot[i] for i in ids]

    def check_engine(self, engine):
        """ValueError unless `engine` has the descriptor the bank was built with (same weights are not checked)"""
        d = engine_descriptor(engine)
        if d != self.engine:
            raise ValueError(f"template bank built by {self.engine}, the model is {d}: rebuild the bank")

    def check_grid(self, template_poses):
        """ValueError unless template_poses [N, 3, 3] is the bank's grid, exactly"""
        tp = torch.as_tensor(template_poses).detach().cpu()
        if tuple(tp.shape) != tuple(self._template_poses_host.shape) or \
                not torch.equal(tp.to(torch.float64), self._template_poses_host):
            raise ValueError(f"the pose grid {tuple(tp.shape)} is not the bank's ({self.num_poses} poses)")


# ---------------------------------------------------------------------- search
def check_bank_search(bank, engine, n_queries, obj_ids, angles, k):
    """The refusals of a bank search, on the host: the bank type, the engine descriptor, n_queries = len(obj_ids) >= 1,
    every id in the bank, check_inplane_args(angles, k, N).  -> (A, k, slots)"""
    if not isinstance(bank, TemplateBank):
        raise ValueError("bank must be a nope_b200.bank.TemplateBank")
    bank.check_engine(engine)
    slots = bank.slots(obj_ids)
    if len(slots) != n_queries or n_queries < 1:
        raise ValueError(f"{len(slots)} obj_ids for {n_queries} queries")
    A, k = check_inplane_args(angles, k, bank.num_poses)
    return A, k, slots


class RowPlan:
    """The grouping of D detections by bank slot, made on the host: detections sorted by slot (stable), the groups'
    slots and row offsets (A rows per detection), and the device copies of those and of the permutation, uploaded
    from pinned memory without blocking.  order / inverse are None when the detections are already grouped."""

    def __init__(self, slots, A, device):
        D = len(slots)
        order = sorted(range(D), key=slots.__getitem__)
        gslots, row_off = [], [0]
        for d in order:
            if not gslots or gslots[-1] != slots[d]:
                gslots.append(slots[d])
                row_off.append(row_off[-1])
            row_off[-1] += A
        grouped = order == list(range(D))
        inverse = [0] * D
        for i, d in enumerate(order):
            inverse[d] = i
        G = self.G = len(gslots)
        host = torch.tensor(gslots + row_off + slots + ([] if grouped else order + inverse), dtype=torch.int32)
        dev = host.pin_memory().to(device, non_blocking=True) if torch.device(device).type == "cuda" else \
            host.to(device)
        self.D, self.A = D, A
        self.gslots, self.row_off, self.det_slots = dev[:G], dev[G:2 * G + 1], dev[2 * G + 1:2 * G + 1 + D]
        base = 2 * G + 1 + D
        self.order = None if grouped else dev[base:base + D]
        self.inverse = None if grouped else dev[base + D:base + 2 * D]

    def grouped(self, x):
        """x [D, ...] in detection order -> in group order"""
        return x if self.order is None else x.index_select(0, self.order)

    def restore(self, x):
        """x [D, ...] in group order -> in detection order"""
        return x if self.inverse is None else x.index_select(0, self.inverse)


def score_rows(bank, query, plan, metric, threshold, k, visible=None):
    """nope_score_topk_grouped on the current stream: query [D, A, C, 32, 32] in the plan's group order against the
    bank -> (sim [D, A, N], top [D, k] at a * N + n | None for k = 0), in group order.  visible [D, A, 32, 32] (the
    rows' visible maps, DESIGN.md section 27): nope_score_topk_visible, each row scored over its visible pixels."""
    D, A, N = plan.D, plan.A, bank.num_poses
    dev = bank.device
    if visible is not None:
        from .visibility import score_visible
        sim, top = score_visible(query.reshape(D * A, *query.shape[2:]), bank.templates, plan.gslots, plan.row_off,
                                 A, visible.reshape(D * A, *visible.shape[2:]), metric, threshold, k)
        return sim.view(D, A, N), top
    q = query.to(dev, torch.float32).contiguous()
    t = bank.templates
    sim = torch.empty((D, A, N), device=dev, dtype=torch.float32)
    topv = torch.empty((D, k), device=dev, dtype=torch.float32)
    topi = torch.empty((D, k), device=dev, dtype=torch.int64)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().nope_score_topk_grouped(
            _lib.ptr(q), _lib.ptr(t), D * A, t.shape[0], N, t.shape[2], t.shape[3] * t.shape[4],
            _lib.ptr(plan.gslots), _lib.ptr(plan.row_off), plan.G, A, _METRICS[metric], float(threshold), k,
            _lib.ptr(sim), _lib.ptr(topv) if k else None, _lib.ptr(topi) if k else None,
            _lib.stream(dev)))
    return sim, (topi if k else None)


def search_bank(bank, query_latents, obj_ids, engine, k=5, metric="l2", threshold=0.2):
    """The bank search on latents: query_latents [D, A, C, 32, 32] (the A rotated copies of each detection's crop,
    e.g. encode_image_inplane) of detections of obj_ids [D], each scored against its object's templates.
    -> (sim [D, A, N], top [D, k] at a * N + n, joint over (angle, pose), ties -> the lowest index) in the
    detections' order.  engine: the model's, for the descriptor check."""
    check_metric(metric)
    if query_latents.dim() != 5 or tuple(query_latents.shape[2:]) != (bank.latent_dim, 32, 32):
        raise ValueError(f"query_latents [D, A, {bank.latent_dim}, 32, 32] expected (the bank's latent shape), got "
                         f"{tuple(query_latents.shape)}")
    A, k, slots = check_bank_search(bank, engine, query_latents.shape[0], obj_ids, query_latents.shape[1], k)
    if bank.device.type != "cuda":
        raise _lib.NopeError("search_bank needs a bank on a CUDA device (no CPU fallback)")
    plan = RowPlan(slots, A, bank.device)
    sim, top = score_rows(bank, plan.grouped(query_latents.to(bank.device)), plan, metric, threshold, k)
    return plan.restore(sim), plan.restore(top)
