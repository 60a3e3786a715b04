"""Host-side mirror of the reference task module `PoseConditional`
(src/model/model.py:32-565), inference surface only: forward (loss), sample,
generate_templates, retrieval, plus predict_pose (= eval_geodesic lines 313-357 without
logging, SURVEY.md F2) and the T-LESS VSD evaluation (eval_vsd, model.py:378-541, on the
CUDA rasterizer and VSD kernels of nope_b200.vsd).  Training and wandb/video logging are out
of scope (SURVEY.md section 8).

Differences that are deliberate and documented:
  * generate_templates batches the whole pose grid through one engine sweep instead of a
    Python loop that re-encodes the reference per pose (model.py:212-222, 115).
  * retrieval raises ValueError for an unknown metric instead of returning None
    (model.py:256 falls through); "cosine" is an extension (SURVEY.md F3).
  * ranking is deterministic: descending score, ties -> lowest index.
"""
import os
import types

import torch
import torch.nn.functional as F

from . import _lib
from .search import (_METRICS, check_metric, coarse_to_fine_search, grid_search, multi_query_form,
                     refined_search)


def _ns(d):
    return d if not isinstance(d, dict) else types.SimpleNamespace(**d)


class PoseConditional:
    def __init__(self, u_net, optim_config=None, testing_config=None, save_dir=None, **kwargs):
        self.u_net = u_net
        self.save_dir = save_dir
        self.optim_config = _ns(optim_config) if optim_config is not None else \
            types.SimpleNamespace(loss_type="l1")
        self.testing_config = _ns(testing_config) if testing_config is not None else \
            types.SimpleNamespace(similarity_metric="l2")
        loss_type = getattr(self.optim_config, "loss_type", "l1")
        self.loss = F.l1_loss if loss_type == "l1" else F.mse_loss
        self.dist = None     # optional nope_b200.dist.ShardedSweep for multi-GPU
        from .metrics import GeodesicError
        self.metric = GeodesicError()              # model.py:56
        self.logged = {}                           # what Lightning's self.log would have received
        self.global_step, self.global_rank = 0, 0
        # model.py:66: per-batch VSD errors go to <save_dir>/predictions (created on first save)
        self.log_dir = None if save_dir is None else os.path.join(save_dir, "predictions")
        self.tless_cad = {}                        # obj_id -> nope_b200.vsd.Mesh (load_mesh)
        self.bop_models = {}                       # obj_id -> {"diameter", "symmetries"} (load_models_info)

    @property
    def device(self):
        return self.u_net.device

    def eval(self):
        self.u_net.eval()
        return self

    def load_state_dict(self, state_dict, strict=True):
        """Accepts a Lightning checkpoint's `state_dict` (keys prefixed `u_net.`) or a bare
        UNet state_dict."""
        if any(k.startswith("u_net.") for k in state_dict):
            state_dict = {k[len("u_net."):]: v for k, v in state_dict.items()
                          if k.startswith("u_net.")}
        self.u_net.load_state_dict(state_dict, strict=strict)
        return self

    def state_dict(self):
        """Lightning-style keys: every UNet / encoder entry under `u_net.` (model.py:33-40)."""
        return {"u_net." + k: v for k, v in self.u_net.state_dict().items()}

    # ------------------------------------------------------------------ model.py:96-111
    def compute_loss(self, pred, gt):
        loss = self.loss(pred, gt, reduction="none")
        return loss.flatten(1).mean(dim=1).mean()

    @torch.no_grad()
    def forward(self, query, reference, relativeR):
        query_feat = self.u_net.encoder.encode_image(query.to(self.device))
        reference_feat = self.u_net.encoder.encode_image(reference.to(self.device), mode="mode")
        pred = self.u_net(reference_feat, relativeR)
        return self.compute_loss(pred, query_feat)

    __call__ = forward

    # ------------------------------------------------------------------ model.py:113-124
    @torch.no_grad()
    def sample(self, reference, relativeR):
        reference_feat = self.u_net.encoder.encode_image(reference.to(self.device), mode="mode")
        pred = self.u_net(reference_feat, relativeR)
        return pred, self._decode(pred)

    # ------------------------------------------------------------------ model.py:193-252
    @torch.no_grad()
    def generate_templates(self, reference, all_relativeR, gt_templates=None, visualize=False):
        reference_feat = self.u_net.encoder.encode_image(reference.to(self.device), mode="mode")
        emb = self.u_net.sweep(reference_feat, all_relativeR, want_emb=True)["emb"]
        images = self._decode(emb.flatten(0, 1))
        if images is not None:
            images = images.view(*emb.shape[:2], *images.shape[1:])
        return emb, images, None

    def _decode(self, latents):
        """unnormalize_to_zero_to_one(decode_latent(latents)) (model.py:119-120, utils.py:12-15) when the encoder is
        a VAE with its decoder weights; None for the template encoder or a VAE loaded without a decoder."""
        enc = self.u_net.encoder
        if not getattr(enc, "has_decoder", False):
            return None
        return ((enc.decode_latent(latents) + 1) * 0.5).clamp(0, 1)

    # ------------------------------------------------------------------ model.py:254-266
    @torch.no_grad()
    def retrieval(self, query, template_feat, k=5, hidden=None):
        """-> (similarity, nearest_idx).  Query and template batches follow the reference's broadcasting
        (model.py:260-262): equal batches give [B,N]; templates [1,N,...] serve every query ([Bq,N]: templates
        generated once, queries streamed); one query against [Bt,N,...] templates gives [Bt,N].  hidden [Bq, 256,
        256] (uint8 or bool, non-zero = may be hidden by an occluder): each query scores only its visible latent
        pixels (DESIGN.md section 27); None, or an all-zero mask, gives the scores without it bit for bit."""
        metric = self._metric()
        hidden = self._hidden("retrieval", hidden, query.shape[:1])
        query_feat = self.u_net.encoder.encode_image(query.to(self.device), mode="mode")
        vis = {}
        if hidden is not None:
            from .visibility import query_visible
            vis["visible"] = query_visible(hidden.to(self.device), query.shape[:1], "retrieval")
        return score_topk(query_feat, template_feat, k=k, metric=metric, threshold=self._occlusion_threshold(), **vis)

    def _occlusion_threshold(self):
        """`threshold` of the template encoder (OcclusionAwareSimilarity, base_template.py:67-75;
        configs/model/template_base.yaml: 0.2)."""
        return float(getattr(self.u_net.encoder, "threshold", 0.2))

    def _metric(self):
        return check_metric(getattr(self.testing_config, "similarity_metric", "l2"))

    def _checked(self, query, reference, unsharded=None, check=None):
        """The refusals of a search, all before anything is encoded: model.dist for a search that runs on one device
        (`unsharded`, its name), the search's own argument check check(), the similarity metric and, given a reference
        (a bank search has none), the query form.
        -> (metric, what check returned)"""
        if unsharded is not None and self.dist is not None:
            raise NotImplementedError(f"{unsharded} does not shard across GPUs: it runs on one device (unset "
                                      "model.dist or use predict_pose)")
        checked = None if check is None else check()
        metric = self._metric()
        if reference is not None:
            multi_query_form(query, reference)
        return metric, checked

    def _hidden(self, name, hidden, lead):
        """The refusals of a search's hidden= (DESIGN.md section 27), before any device work: model.dist set
        (NotImplementedError; the searches under occlusion run on one device) and a mask that is not [*lead, 256,
        256] uint8 or bool (ValueError).  -> hidden as given (None stays None)"""
        if hidden is None:
            return None
        if self.dist is not None:
            raise NotImplementedError(f"{name}(hidden=) does not shard across GPUs: it runs on one device (unset "
                                      "model.dist)")
        from .visibility import check_hidden
        check_hidden(hidden, lead, name)
        return hidden

    def _encode(self, query, reference, metric):
        """The metric set for the sweep's last layer, then queries and references through one encoder call over
        cat([flattened queries, references]).  -> (query latents in the query's form, reference latents)"""
        self.u_net.set_metric(metric, self._occlusion_threshold())
        flat = query.reshape(-1, *query.shape[-3:])
        feats = self.u_net.encoder.encode_image(torch.cat([flat.to(self.device), reference.to(self.device)]))
        n = flat.shape[0]
        return feats[:n].view(*query.shape[:-3], *feats.shape[1:]), feats[n:]

    # ------------------------------------------------------------------ model.py:313-357
    @torch.no_grad()
    def predict_pose(self, query, reference, all_relativeR, template_poses=None, k=5,
                     return_templates=False, hidden=None):
        """-> (R [B,k,3,3] | None, nearest_idx [B,k] int64, similarity [B,N]).  The scores and
        the ranking come out of the sweep's fused last layer; the [B,N,C,32,32] templates are
        only materialised when asked for.

        Several queries of one object share the reference's sweep (the templates do not depend on the query):
          query [B,Q,3,H,W] with reference [B,3,H,W] -> R [B,Q,k,3,3], nearest_idx [B,Q,k], similarity [B,Q,N];
          query [Q,3,H,W] with reference [1,3,H,W] and all_relativeR [1,N,6] -> [Q,k,3,3], [Q,k], [Q,N]
          (the reference's broadcasting of one template set against a query batch).
        Query and reference images go through one encoder call, the templates through one sweep.
        hidden [..., 256, 256] (the query's leading shape; uint8 or bool, non-zero = may be hidden by an occluder):
        every score leaves out the latent pixels those crop pixels reach (DESIGN.md section 27); None, or an all-zero
        mask, gives the scores without it bit for bit."""
        metric, _ = self._checked(query, reference)
        hidden = self._hidden("predict_pose", hidden, query.shape[:-3])
        query_feat, reference_feat = self._encode(query, reference, metric)
        visible = None
        if hidden is not None:
            from .visibility import query_visible
            visible = query_visible(hidden.to(self.device), query.shape[:-3], "predict_pose")
        # under sharding the templates are (local templates, lo, hi): each rank keeps only its slice
        return grid_search(self.u_net, reference_feat, query_feat, all_relativeR, template_poses, k=k,
                           return_templates=return_templates, dist=self.dist, metric=metric,
                           threshold=self._occlusion_threshold(), query_visible=visible)

    @torch.no_grad()
    def predict_pose_coarse_to_fine(self, query, reference, all_relativeR_levels, hierarchy, template_poses=None,
                                    k=5, keep=8):
        """predict_pose over the finest grid of a nested pose hierarchy (nope_b200.hierarchy, DESIGN.md section 9),
        sweeping the coarsest grid and then only the finer poses around each row's best `keep`.
        all_relativeR_levels[l] [B, N_l, 6] per level, coarsest first; hierarchy a PoseHierarchy over the same
        levels; template_poses the finest grid's rotations, for the R lookup.
        -> (R | None, nearest_idx, similarity [..., N_L]) in the shapes of predict_pose (the same three query
        forms); similarity is -inf at poses the search did not score.  Every scored pose has exactly the score
        predict_pose gives it.  One encoder call."""
        from .hierarchy import check_search_args
        metric, _ = self._checked(query, reference, "predict_pose_coarse_to_fine",
                                  lambda: check_search_args(hierarchy, all_relativeR_levels, keep, k))
        query_feat, reference_feat = self._encode(query, reference, metric)
        return coarse_to_fine_search(self.u_net, reference_feat, query_feat, all_relativeR_levels, hierarchy,
                                     template_poses, k=k, keep=keep)

    @torch.no_grad()
    def predict_pose_refined(self, query, reference, all_relativeR, refiner, k=5, keep=2):
        """Poses between the grid poses (nope_b200.refine, DESIGN.md section 10): the exhaustive sweep of
        all_relativeR [B, N, 6] seeds each (reference, query) row with its best `keep` grid poses, and the
        refiner's steps search shrinking rotation lattices around them.  refiner: a PoseRefiner over the same grid.
        -> (R [..., k, 3, 3] = D * template_poses[seed] (float64), seed_idx [..., k], score [..., k]) in the query
        forms of predict_pose; descending score, each exactly the score a sweep of that pose gives.  One encoder
        call.  keep = 2 by default: keep = 4 measured hardly more accurate for up to 1.8x the time (DESIGN.md
        section 6)."""
        from .refine import check_refine_args
        metric, _ = self._checked(query, reference, "predict_pose_refined",
                                  lambda: check_refine_args(refiner, all_relativeR, keep, k, reference.shape[0]))
        query_feat, reference_feat = self._encode(query, reference, metric)
        return refined_search(self.u_net, reference_feat, query_feat, all_relativeR, refiner, k=k, keep=keep)

    def _inplane_sweep(self, query, reference, all_relativeR, metric, A, k, hidden=None):
        """The in-plane search's sweep (DESIGN.md section 11): the references encoded on their own, the A rotated
        copies of each of the B * Q queries by one encode_image_inplane call, one sweep with Q * A query rows per
        reference, and the top-k of each (reference, query) row jointly over (angle, pose).
        -> (sim [B, Q * A, N], top [B * Q, k] at a * N + n, query latents [B * Q, A, C, h, w], the flattened query
        images [B * Q, 3, H, W] and the reference latents, on the device).  hidden: the queries' crop-space masks;
        each rotated copy then scores over its own visible map."""
        enc = self.u_net.encoder
        self.u_net.set_metric(metric, self._occlusion_threshold())
        B, N = reference.shape[0], all_relativeR.shape[1]
        reference_feat = enc.encode_image(reference.to(self.device))
        images = query.reshape(-1, *query.shape[-3:]).to(self.device)
        query_feat = enc.encode_image_inplane(images, A)
        visible = None
        if hidden is not None:
            from .visibility import latent_visibility_inplane
            visible = latent_visibility_inplane(hidden.reshape(-1, *hidden.shape[-2:]).to(self.device), A)
            visible = visible.view(B, -1, *visible.shape[2:])
        vis = {} if visible is None else {"query_visible": visible}
        sim = self.u_net.sweep(reference_feat, all_relativeR, query_feat=query_feat.view(B, -1, *query_feat.shape[2:]),
                               want_emb=False, want_sim=True, k=0, **vis)["sim"]
        _, top = topk(sim.view(-1, A * N), k)
        return sim, top, query_feat, images, reference_feat

    @torch.no_grad()
    def predict_pose_inplane(self, query, reference, all_relativeR, template_poses=None, k=5, angles=36,
                             hidden=None):
        """predict_pose over pose x in-plane angle (nope_b200.inplane, DESIGN.md section 11): every query crop is
        rotated by the A = `angles` angles a * 360 / A and each rotated copy is scored against the same templates.
        -> (R [..., k, 3, 3] = Rz(alpha[angle_idx]) template_poses[nearest_idx] (float64) | None, nearest_idx [..., k],
        angle_idx [..., k], similarity [..., A, N]) in the query forms of predict_pose; the top-k runs jointly over
        (angle, pose), ties -> the lowest a * N + n.  One encoder call for the references, one encode_image_inplane
        call for the queries, one sweep with Q * A query rows per reference.  angles = 1 is predict_pose.  hidden: as
        in predict_pose; each rotated copy scores over the map of its own roll."""
        from .inplane import check_inplane_args, compose

        def check():
            if all_relativeR.dim() != 3 or all_relativeR.shape[0] != reference.shape[0] or all_relativeR.shape[2] != 6:
                raise ValueError(f"all_relativeR [B, N, 6] with B = {reference.shape[0]} references expected, got "
                                 f"{tuple(all_relativeR.shape)}")
            return check_inplane_args(angles, k, all_relativeR.shape[1])

        metric, (A, k) = self._checked(query, reference, "predict_pose_inplane", check)
        hidden = self._hidden("predict_pose_inplane", hidden, query.shape[:-3])
        sim, top, _, _, _ = self._inplane_sweep(query, reference, all_relativeR, metric, A, k, hidden)
        N, lead = all_relativeR.shape[1], tuple(query.shape[:-3])
        nearest, angle = (top % N).view(lead + (k,)), (top // N).view(lead + (k,))
        R = compose(template_poses, nearest, angle, A) if template_poses is not None else None
        return R, nearest, angle, sim.view(lead + (A, N))

    @torch.no_grad()
    def predict_pose_inplane_refined(self, query, reference, all_relativeR, refiner, k=5, keep=2, hidden=None):
        """Roll and viewpoint between the bins and the grid poses (nope_b200.inplane_refine, DESIGN.md section 14):
        the in-plane search over the refiner's A angles seeds each (reference, query) row with its joint top-`keep`
        (angle, pose) pairs, and the refiner's steps refine the viewpoint on the template side and the roll on the
        query side.  refiner: an InplaneRefiner over the grid of all_relativeR [B, N, 6].
        -> (R [..., k, 3, 3] = Rz(rho) D template_poses[seed] (float64), seed [..., k], alpha_deg [..., k] =
        atan2(sin, cos) of the roll rho, score [..., k]) in the query forms of predict_pose; descending score, each
        exactly the score a sweep of that pose against that rolled latent gives.  hidden: as in predict_pose; the
        search and every refinement step score over the visible maps of their rolls."""
        from .inplane_refine import check_inplane_refine_args, pose_rotations, refine_inplane, roll_degrees
        metric, _ = self._checked(
            query, reference, "predict_pose_inplane_refined",
            lambda: check_inplane_refine_args(refiner, all_relativeR, keep, k, reference.shape[0]))
        hidden = self._hidden("predict_pose_inplane_refined", hidden, query.shape[:-3])
        _, top, query_feat, images, reference_feat = self._inplane_sweep(query, reference, all_relativeR, metric,
                                                                         refiner.angles, keep, hidden)
        N = refiner.num_poses
        pose_idx, angle_idx = top % N, top // N
        lat = query_feat[torch.arange(top.shape[0], device=top.device)[:, None], angle_idx]   # [B * Q, keep, C, h, w]
        query, squeeze = multi_query_form(query, reference)
        lead = tuple(query.shape[:-3])
        out = refine_inplane(self.u_net, self.u_net.encoder, reference_feat, images.view(*lead, *query.shape[-3:]),
                             all_relativeR, (pose_idx.view(*lead, keep), angle_idx.view(*lead, keep)),
                             lat.view(*lead, keep, *lat.shape[2:]), refiner, k=k,
                             **({} if hidden is None else {"hidden": hidden.reshape(*lead, *hidden.shape[-2:])}))
        R = pose_rotations(out["D"], out["seed"], out["cossin"], refiner)
        seed, alpha, score = out["seed"], roll_degrees(out["cossin"]), out["score"]
        if squeeze:
            R, seed, alpha, score = R[0], seed[0], alpha[0], score[0]
        return R, seed, alpha, score

    @torch.no_grad()
    def retrieval_inplane(self, query, template_feat, k=5, angles=36, hidden=None):
        """retrieval over pose x in-plane angle, for templates generated once and queries streamed: the A = `angles`
        rotated copies of every query image [Bq, 3, 256, 256] against template_feat [Bt, N, C, h, w], batches
        broadcast as in retrieval.  -> (similarity [rows, A, N], nearest_idx [rows, k], angle_idx [rows, k]); the
        top-k runs jointly over (angle, pose), ties -> the lowest a * N + n.  hidden [Bq, 256, 256]: as in
        predict_pose_inplane."""
        from .inplane import check_inplane_args
        if query.dim() != 4 or template_feat.dim() != 5:
            raise ValueError(f"query [B, 3, H, W] and template_feat [B, N, C, h, w] expected; got "
                             f"{tuple(query.shape)} and {tuple(template_feat.shape)}")
        enc = self.u_net.encoder
        if template_feat.shape[2:] != (enc.latent_dim, 32, 32):
            raise ValueError(f"template_feat [B, N, {enc.latent_dim}, 32, 32] expected, got "
                             f"{tuple(template_feat.shape)}")
        N = template_feat.shape[1]
        A, k = check_inplane_args(angles, k, N)
        metric = self._metric()
        hidden = self._hidden("retrieval_inplane", hidden, query.shape[:1])
        B, Q, Bt, rows = broadcast_batches(query.shape[0], template_feat.shape[0])
        dev = template_feat.device
        if dev.type != "cuda":
            raise _lib.NopeError("retrieval_inplane needs CUDA tensors (no CPU fallback)")
        q = enc.encode_image_inplane(query.to(dev), A)                                     # [Bq, A, C, h, w]
        q = q.reshape(-1, Q * A, *q.shape[2:]).expand(B, Q * A, *q.shape[2:]).contiguous()
        t = template_feat.to(torch.float32).contiguous()
        if hidden is None:
            sim, _, _ = _score_multi(q, t, B, Q * A, metric, self._occlusion_threshold())
        else:
            # the broadcasting as groups: template batch g serves the B * Q * A / Bt rows that follow row_off[g]
            from .visibility import latent_visibility_inplane, score_visible
            vis = latent_visibility_inplane(hidden.to(dev), A)
            vis = vis.reshape(-1, Q * A, *vis.shape[2:]).expand(B, Q * A, *vis.shape[2:]).reshape(-1, *vis.shape[2:])
            slots = torch.arange(Bt, device=dev, dtype=torch.int32)
            row_off = torch.arange(Bt + 1, device=dev, dtype=torch.int32) * (B * Q * A // Bt)
            sim, _ = score_visible(q.view(-1, *q.shape[2:]), t, slots, row_off, A, vis, metric,
                                   self._occlusion_threshold(), 0)
        _, flat = topk(sim.view(rows, A * N), k)
        return sim.view(rows, A, N), flat % N, flat // N

    # ------------------------------------------------------------------ template banks (DESIGN.md section 25)
    @torch.no_grad()
    def build_template_bank(self, obj_ids, reference, all_relativeR, template_poses):
        """Sweep every object's reference once and keep its templates: obj_ids [O] (unique), reference [O, 3, 256,
        256], all_relativeR [O, N, 6], template_poses [N, 3, 3] (one grid for every object).  One encoder call, then
        one sweep (bank.TemplateBank.build).  -> TemplateBank on the model's device; bank.save / TemplateBank.load
        keep it across processes.  The bank holds the templates generate_templates gives, bit for bit."""
        from .bank import TemplateBank
        if reference.dim() != 4 or reference.shape[0] != len(obj_ids):
            raise ValueError(f"reference [O, 3, H, W] with O = {len(obj_ids)} obj_ids expected, got "
                             f"{tuple(reference.shape)}")
        if all_relativeR.dim() != 3 or all_relativeR.shape[0] != reference.shape[0]:
            raise ValueError(f"all_relativeR [O, N, 6] with O = {reference.shape[0]} expected, got "
                             f"{tuple(all_relativeR.shape)}")
        if len(set(int(i) for i in obj_ids)) != len(obj_ids):
            raise ValueError(f"duplicate obj_ids in {list(obj_ids)}")
        if tuple(torch.as_tensor(template_poses).shape) != (all_relativeR.shape[1], 3, 3):
            raise ValueError(f"template_poses [{all_relativeR.shape[1]}, 3, 3] expected (the grid of all_relativeR), "
                             f"got {tuple(torch.as_tensor(template_poses).shape)}")
        reference_feat = self.u_net.encoder.encode_image(reference.to(self.device), mode="mode")
        return TemplateBank.build(self.u_net, reference_feat, obj_ids, all_relativeR, template_poses)

    def _bank_query(self, name, query, obj_ids, bank, angles, k):
        """the refusals of a bank search, before any device work (model.dist, the bank, the engine descriptor, the
        ids, the in-plane arguments, the metric) -> (metric, A, k, the bank slot of every detection)"""
        from .bank import check_bank_search
        if query.dim() != 4 or query.shape[1] != 3:
            raise ValueError(f"{name}: query [D, 3, H, W] (one crop per detection) expected, got {tuple(query.shape)}")
        metric, (A, k, slots) = self._checked(
            query, None, name, lambda: check_bank_search(bank, self.u_net, query.shape[0], obj_ids, angles, k))
        return metric, A, k, slots

    def _bank_scores(self, query, bank, slots, metric, A, k, hidden=None):
        """the detections' crops grouped by slot, their A rotated copies encoded by one encode_image_inplane call and
        scored against the bank by one nope_score_topk_grouped call.  -> (plan, query latents, sim [D, A, N], top
        [D, k]), all in the plan's group order"""
        from .bank import RowPlan, score_rows
        plan = RowPlan(slots, A, bank.device)
        images = plan.grouped(query.to(self.device))
        lat = self.u_net.encoder.encode_image_inplane(images, A)
        visible = None
        if hidden is not None:
            from .visibility import latent_visibility_inplane
            visible = latent_visibility_inplane(plan.grouped(hidden.to(self.device)), A)
        vis = {} if visible is None else {"visible": visible}
        sim, top = score_rows(bank, lat, plan, metric, self._occlusion_threshold(), k, **vis)
        return plan, lat, sim, top

    @torch.no_grad()
    def predict_pose_bank(self, query, obj_ids, bank, k=5, angles=36, hidden=None):
        """predict_pose_inplane against a template bank: query [D, 3, 256, 256], one crop per detection, obj_ids [D]
        (host) its objects, each held by `bank` (build_template_bank).  -> (R [D, k, 3, 3] = Rz(alpha[angle_idx])
        template_poses[nearest_idx] (float64), nearest_idx [D, k], angle_idx [D, k], similarity [D, A, N]) in the
        detections' order: what predict_pose_inplane returns for reference[slot], with each detection scored against
        its object's stored templates (the arithmetic of retrieval_inplane) instead of a sweep.  Detections of one
        object share each template read.  One encode_image_inplane call over all D crops, one scoring call, no host
        synchronisation.  angles = 1 is the plain grid search.  Scores use the model's current metric.  hidden
        [D, 256, 256]: as in predict_pose_inplane, the scores of retrieval_inplane with the same hidden."""
        from .inplane import compose
        metric, A, k, slots = self._bank_query("predict_pose_bank", query, obj_ids, bank, angles, k)
        hidden = self._hidden("predict_pose_bank", hidden, query.shape[:1])
        plan, _, sim, top = self._bank_scores(query, bank, slots, metric, A, k, hidden)
        sim, top = plan.restore(sim), plan.restore(top)
        N = bank.num_poses
        nearest, angle = top % N, top // N
        return compose(bank.template_poses, nearest, angle, A), nearest, angle, sim

    @torch.no_grad()
    def predict_pose_bank_refined(self, query, obj_ids, bank, refiner, k=5, keep=2, hidden=None):
        """predict_pose_inplane_refined against a template bank: the bank search over the refiner's angles seeds each
        detection with its joint top-`keep` (angle, pose) pairs, and refine_inplane continues from them with the
        detection's reference_latents[slot] and all_relativeR[slot].  refiner: an InplaneRefiner over the bank's grid.
        -> (R [D, k, 3, 3], seed [D, k], alpha_deg [D, k], score [D, k]) as predict_pose_inplane_refined returns.
        hidden [D, 256, 256]: as in predict_pose_inplane_refined."""
        from .inplane_refine import (InplaneRefiner, check_inplane_refine_args, pose_rotations, refine_inplane,
                                     roll_degrees)
        if not isinstance(refiner, InplaneRefiner):
            raise ValueError("refiner must be a nope_b200.inplane_refine.InplaneRefiner")
        metric, A, _, slots = self._bank_query("predict_pose_bank_refined", query, obj_ids, bank, refiner.angles,
                                               keep)
        check_inplane_refine_args(refiner, bank.all_relativeR, keep, k)
        bank.check_grid(refiner.template_poses)
        hidden = self._hidden("predict_pose_bank_refined", hidden, query.shape[:1])
        plan, lat, _, top = self._bank_scores(query, bank, slots, metric, A, keep, hidden)
        N = bank.num_poses
        pose_idx, angle_idx = top % N, top // N
        seed_lat = lat[torch.arange(plan.D, device=top.device)[:, None], angle_idx]     # [D, keep, C, h, w]
        pose_idx, angle_idx, seed_lat = plan.restore(pose_idx), plan.restore(angle_idx), plan.restore(seed_lat)
        ref_feat = bank.reference_latents.index_select(0, plan.det_slots)
        rel = bank.all_relativeR.index_select(0, plan.det_slots)
        out = refine_inplane(self.u_net, self.u_net.encoder, ref_feat, query.to(self.device), rel,
                             (pose_idx, angle_idx), seed_lat, refiner, k=k, **({} if hidden is None else
                                                                               {"hidden": hidden}))
        R = pose_rotations(out["D"], out["seed"], out["cossin"], refiner)
        return R, out["seed"], roll_degrees(out["cossin"]), out["score"]

    # ------------------------------------------------------------------ model.py:185-191, 268-376, 550-565
    def log(self, name, value, **kwargs):
        self.logged.setdefault(name, []).append(float(value))

    def log_score(self, dict_scores, split_name):
        for key, value in dict_scores.items():
            self.log(f"{key}/{split_name}", value, sync_dist=True)

    @torch.no_grad()
    def eval_geodesic(self, batch, data_name, visualize=False, save_prediction=False):
        """`eval_geodesic` of the reference without the wandb / image logging (the template encoder has
        no decoder, so the reference itself sets visualize=False on this path, model.py:269-274):
        validation loss under the ground-truth pose, template sweep + retrieval, geodesic accuracy."""
        query, reference = batch["query"], batch["reference"]
        loss = self.forward(query=query, relativeR=batch["gt_relativeR"], reference=reference)
        self.log(f"loss/val_{data_name}", loss)
        template_poses = batch["template_poses"][0]
        predR, nearest_idx, similarity = self.predict_pose(query, reference, batch["all_relativeR"],
                                                           template_poses, k=5)
        error, acc = self.metric(predR=predR, gtR=batch["query_pose"].to(predR.device),
                                 symmetry=batch["symmetry"].reshape(-1).to(predR.device))
        self.log_score(acc, split_name=f"val_{data_name}")
        if save_prediction and self.save_dir is not None:
            import os
            import numpy as np
            os.makedirs(os.path.join(self.save_dir, "predictions"), exist_ok=True)
            np.savez(os.path.join(self.save_dir, "predictions",
                                  f"pred_{data_name}_step{self.global_step}_rank{self.global_rank}"),
                     query_pose=batch["query_pose"].cpu().numpy(), similarity=similarity.cpu().numpy(),
                     nearest_idx=nearest_idx.cpu().numpy())
        return error, nearest_idx, similarity

    # ------------------------------------------------------------------ model.py:378-541 (T-LESS, DESIGN.md section 12)
    def load_mesh(self, cad_dir, obj_ids=range(1, 31)):
        """model.py:378-389: the T-LESS CAD models obj_{id:06d}.ply of `cad_dir` (ids 1 ... 30) as device meshes in
        self.tless_cad."""
        from .vsd import Mesh
        for obj_id in obj_ids:
            self.tless_cad[int(obj_id)] = Mesh.from_ply(os.path.join(cad_dir, f"obj_{int(obj_id):06d}.ply"),
                                                        device=self.device)
        return self

    _VSD_KEYS = ("query", "reference", "gt_relativeR", "all_relativeR", "template_poses", "query_pose",
                 "query_translation", "intrinsic", "depth_path", "obj_id")

    def _check_vsd_batch(self, batch):
        for key in self._VSD_KEYS:
            if key not in batch:
                raise KeyError(f"eval_vsd: the batch has no {key!r}")
        B = batch["query"].shape[0]
        tp, qp, qt, K = batch["template_poses"], batch["query_pose"], batch["query_translation"], batch["intrinsic"]
        ar = batch["all_relativeR"]
        if batch["query"].dim() != 4 or tuple(batch["reference"].shape) != tuple(batch["query"].shape) or B < 1:
            raise ValueError(f"eval_vsd: query and reference [B, 3, H, W] expected, got "
                             f"{tuple(batch['query'].shape)} and {tuple(batch['reference'].shape)}")
        if tp.dim() != 4 or tp.shape[0] != B or tuple(tp.shape[2:]) != (3, 3) or ar.dim() != 3 or ar.shape[0] != B \
                or ar.shape[1] != tp.shape[1]:
            raise ValueError(f"eval_vsd: template_poses [B, N, 3, 3] and all_relativeR [B, N, 6] with B = {B} expected, "
                             f"got {tuple(tp.shape)} and {tuple(ar.shape)}")
        if tuple(qp.shape) != (B, 3, 3) or tuple(qt.shape) != (B, 3, 1):
            raise ValueError(f"eval_vsd: query_pose [B, 3, 3] and query_translation [B, 3, 1] expected, got "
                             f"{tuple(qp.shape)} and {tuple(qt.shape)}")
        if K.numel() != B * 9:
            raise ValueError(f"eval_vsd: intrinsic [B, 3, 3] expected, got {tuple(K.shape)}")
        if len(batch["depth_path"]) != B or batch["obj_id"].numel() != B:
            raise ValueError(f"eval_vsd: {B} depth_path entries and obj_id values expected, got "
                             f"{len(batch['depth_path'])} and {batch['obj_id'].numel()}")
        ids = [int(i) for i in batch["obj_id"].reshape(-1).tolist()]
        missing = sorted(set(i for i in ids if i not in self.tless_cad))
        if missing:
            raise ValueError(f"eval_vsd: no mesh loaded for obj_id {missing} (load_mesh)")
        return B, ids

    @torch.no_grad()
    def eval_vsd(self, batch, data_name, save_path=None):
        """`eval_vsd` of the reference (model.py:391-541) without wandb and images: the validation loss under the
        ground-truth pose, the top-5 template retrieval, and the VSD errors of the retrieved rotations at the
        ground-truth translation (delta 15, tau 20, "step": vsd_obj's defaults), rendered and scored on the GPU.
        Returns and logs the reference's final_scores; saves the top-1 errors to save_path (.npy) when given."""
        import numpy as np
        from . import vsd as _vsd
        B, ids = self._check_vsd_batch(batch)
        query, reference = batch["query"], batch["reference"]
        loss = self.forward(query=query, relativeR=batch["gt_relativeR"], reference=reference)
        self.log(f"loss/val_{data_name}", loss)
        R = self._grid_rotations(batch, B)
        depth_test, rendered, _, K4 = self._render_frames(batch, B, ids, R)
        vsd_error = _vsd.vsd_errors(depth_test, rendered[:, 0], rendered[:, 1:], K4)
        vsd_error = vsd_error.cpu().numpy()                                                    # B x k
        final_scores = {}
        for kk in [1, 3, 5]:
            best_vsd = np.min(vsd_error[:, :kk], 1)
            final_scores[f"top {kk}, vsd_median"] = np.median(best_vsd)
            for threshold in [0.3]:
                final_scores[f"top {kk}, vsd_scores {threshold}"] = np.mean((best_vsd <= threshold) * 100.0)
        self.log_score(final_scores, split_name=f"val_{data_name}")
        if save_path is not None:
            os.makedirs(os.path.dirname(os.path.abspath(save_path)), exist_ok=True)
            np.save(save_path, vsd_error[:, 0])
        return final_scores

    def _grid_rotations(self, batch, B):
        """the grid retrieval's top-5 rotations template_poses[nearest_idx] [B, 5, 3, 3] float32 (model.py:469-509)"""
        _, nearest_idx, _ = self.predict_pose(batch["query"], batch["reference"], batch["all_relativeR"], None, k=5)
        dev = nearest_idx.device
        tp = batch["template_poses"].to(dev, torch.float32)
        k = nearest_idx.shape[1]
        return tp[torch.arange(B, device=dev)[:, None].expand(B, k), nearest_idx]

    @staticmethod
    def _read_sensor_depth(batch):
        """The sensor depth of every frame of a T-LESS batch, its "depth_path" PNG / 10.0 (mm, 0 = no reading), as the
        reference's vsd.py:72-74 reads it: -> float64 [B, H, W] on the host."""
        import cv2
        import numpy as np
        depth = []
        for path in batch["depth_path"]:
            d = cv2.imread(path, -1)
            if d is None:
                raise FileNotFoundError(f"eval_vsd: cannot read depth image {path!r}")
            depth.append(d / 10.0)
        if any(d.shape != depth[0].shape or d.ndim != 2 for d in depth):
            raise ValueError("eval_vsd: the depth images of a batch must share one (H, W) size")
        return torch.from_numpy(np.stack(depth))

    def _render_frames(self, batch, B, ids, R, t_est=None):
        """The sensor depth of every frame and the model rendered at the ground-truth pose and at the rotations R
        [B, k, 3, 3] with the ground-truth translation, or with t_est [B, k, 3] when given: -> (depth_test [B, H, W]
        float64, rendered [B, 1 + k, H, W], K [B, 3, 3] float64 on the host, K4 [B, 4] on the device)."""
        from . import vsd as _vsd
        dev = self.device
        k = R.shape[1]
        t = batch["query_translation"].to(dev, torch.float32)                                  # [B, 3, 1]
        poses = torch.zeros((B, 1 + k, 4, 4), device=dev, dtype=torch.float32)
        poses[:, 0, :3, :3] = batch["query_pose"].to(dev, torch.float32)
        poses[:, 1:, :3, :3] = R
        poses[:, :, :3, 3] = t[:, None, :, 0]
        if t_est is not None:
            poses[:, 1:, :3, 3] = t_est
        poses[:, :, 3, 3] = 1.0
        # vsd.py:72-74: the intrinsics and the sensor depth of every frame (PNG / 10.0), read on the host
        K = batch["intrinsic"].detach().cpu().to(torch.float64).reshape(B, 3, 3)
        depth_test = self._read_sensor_depth(batch)
        H, W = depth_test.shape[1:]
        depth_test = depth_test.pin_memory().to(dev, non_blocking=True)
        K4 = torch.stack([K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2]], dim=1)
        K4 = K4.pin_memory().to(dev, non_blocking=True)
        rendered = torch.stack([_vsd.render_depth(self.tless_cad[ids[b]], poses[b], K[b], (H, W))
                                for b in range(B)])                                            # [B, 1 + k, H, W]
        return depth_test, rendered, K, K4

    # ------------------------------------------------------------------ BOP 2019 average recall (DESIGN.md section 15)
    def load_models_info(self, path):
        """A BOP models_info.json: the diameter (mm) and the symmetry transforms [S, 3, 4] of every object, in
        self.bop_models[obj_id] = {"diameter", "symmetries", "info"}; "info" is the `bop.load_models_info` entry, whose
        discrete and continuous symmetries `select_distinct` uses."""
        from . import bop
        for obj_id, info in bop.load_models_info(path).items():
            self.bop_models[obj_id] = {"diameter": info["diameter"], "symmetries": bop.symmetry_transformations(info),
                                       "info": info}
        return self

    @torch.no_grad()
    def select_distinct(self, sim, rotations, obj_ids=None, k=5, *, min_angle_deg):
        """k distinct pose hypotheses per row of a search's similarity (`distinct.distinct_topk`, DESIGN.md section
        21): the best-scoring entries such that no two rotations lie within min_angle_deg of each other, modulo the
        object's symmetries, in place of the search's top-k, which are mostly grid neighbours of one mode.
          sim        [B, N], [B, Q, N] or [Q, N] from predict_pose (or predict_pose_coarse_to_fine: its -inf entries
                     were not scored and are never taken);
          rotations  [B | 1, N, 3, 3] the entries' rotations, e.g. template_poses;
          obj_ids    None (no symmetry) or one object id per index of sim's first dimension, looked up in
                     self.bop_models (load_models_info first);
          min_angle_deg  theta in [0, 180] degrees.  It has no default: no value has been chosen from measured
                     accuracy.
        In-plane search: pass sim.flatten(-2) ([..., A * N]) and, for every (angle a, pose n) at a * N + n,
        inplane.compose(template_poses, n, a, A); then angle_idx, nearest_idx = divmod(idx, N) for idx >= 0.
        -> (R float64 [..., k, 3, 3] (zeros at padding), idx int64 [..., k] (-1 at padding), score float32 [..., k]
        (-inf at padding)) on sim's device, without synchronising.  R goes unchanged into estimate_translation,
        refine_depth, refine_contour and eval_bop(R_est=)."""
        import numpy as np
        from .distinct import distinct_topk
        syms = None
        if obj_ids is not None:
            ids = [int(i) for i in np.asarray(obj_ids.detach().cpu() if torch.is_tensor(obj_ids) else obj_ids)
                   .reshape(-1).tolist()]
            missing = sorted(set(i for i in ids if i not in self.bop_models))
            if missing:
                raise ValueError(f"select_distinct: no models_info entry for obj_id {missing} (load_models_info)")
            syms = [self.bop_models[i]["info"] for i in ids]
        score, idx = distinct_topk(sim, rotations, k, min_angle_deg, syms)
        rot = torch.as_tensor(np.asarray(rotations) if not torch.is_tensor(rotations) else rotations)
        rot = rot.to(idx.device, torch.float64)
        lead = idx.shape[:-1]
        rows = idx.reshape(lead[0] if lead else 1, -1)
        if rot.shape[0] == 1:
            R = rot[0][rows.clamp_min(0)]
        else:
            R = rot[torch.arange(rot.shape[0], device=idx.device)[:, None], rows.clamp_min(0)]
        R = torch.where((rows >= 0)[..., None, None], R, torch.zeros((), dtype=R.dtype, device=R.device))
        return R.reshape(idx.shape + (3, 3)), idx, score

    def _pose_fit_batch(self, name, batch, keys, R, t=None, masks=None, models_info=True):
        """The arguments of a pose fit on a T-LESS batch, checked: the batch's `keys`, R [B, k, 3, 3], t [B, k, 3] and
        masks [B, H, W] when given, and a mesh (with models_info, also a models_info entry) for every object.
        -> (ids, R, t, masks, K float64 [B, 3, 3] on the host); errors name the fit."""
        from ._posefit import _tensor
        for key in keys:
            if key not in batch:
                raise KeyError(f"{name}: the batch has no {key!r}")
        ids = [int(i) for i in batch["obj_id"].reshape(-1).tolist()]
        B = len(ids)
        R = _tensor(R)
        if R.dim() != 4 or R.shape[0] != B or R.shape[2:] != (3, 3) or R.shape[1] < 1:
            raise ValueError(f"{name}: R [B, k, 3, 3] with B = {B} expected, got {tuple(R.shape)}")
        k = R.shape[1]
        if t is not None:
            t = _tensor(t)
            if tuple(t.shape) != (B, k, 3):
                raise ValueError(f"{name}: t [{B}, {k}, 3] expected, got {tuple(t.shape)}")
        if masks is not None:
            masks = _tensor(masks)
            if masks.dim() != 3 or masks.shape[0] != B:
                raise ValueError(f"{name}: masks [B, H, W] with B = {B} expected, got {tuple(masks.shape)}")
        missing = sorted(set(i for i in ids if i not in self.tless_cad or (models_info and i not in self.bop_models)))
        if missing:
            raise ValueError(f"{name}: no mesh or models_info entry for obj_id {missing} (load_mesh, load_models_info)"
                             if models_info else f"{name}: no mesh for obj_id {missing} (load_mesh)")
        K = batch["intrinsic"].detach().cpu().to(torch.float64).reshape(B, 3, 3)
        return ids, R, t, masks, K

    def _object_rows(self, ids):
        """The rows of a batch split by object: yields (obj, ri, rd, pick) for every distinct obj_id in ascending
        order, with the object's row indices ri on the host and rd on the model's device, and pick(x) x's rows (by rd
        for a CUDA tensor, by ri otherwise; None stays None)."""
        for obj in sorted(set(ids)):
            ri = torch.tensor([b for b, i in enumerate(ids) if i == obj], dtype=torch.int64)
            rd = ri.pin_memory().to(self.device, non_blocking=True)
            yield obj, ri, rd, lambda x, ri=ri, rd=rd: None if x is None else x[rd if x.device.type == "cuda" else ri]

    @staticmethod
    def _rerank(score, *xs):
        """each row of score [B, k] and of every x [B, k, ...] sorted by descending score (stable, NaN last):
        -> (*xs, score)"""
        order = torch.sort(-score, dim=1, stable=True).indices                     # NaN sorts last
        rows = torch.arange(score.shape[0], device=score.device)[:, None]
        return tuple(x[rows, order] for x in xs) + (score[rows, order],)

    @torch.no_grad()
    def estimate_translation(self, batch, R, masks, iters=4, occluders=None):
        """The translation of every rotation hypothesis R [B, k, 3, 3] of a T-LESS batch (the `eval_vsd` schema; its
        "intrinsic" and "obj_id" are used) fitted to the object's mask of each frame, masks [B, H, W] (uint8 or bool,
        nonzero = object), starting from `translation.initial_translation` with the object's diameter
        (load_models_info) and the mesh of load_mesh; DESIGN.md section 18.  occluders [B, H, W] (uint8 or bool,
        nonzero = something may hide the object there) make the fit ignore those pixels (DESIGN.md section 24); None
        is the plain fit.  One call per distinct object.  -> (t float64 [B, k, 3] mm, iou float64 [B, k]) on the
        model's device, without synchronising."""
        from . import translation
        ids, R, _, masks, K = self._pose_fit_batch("estimate_translation", batch, ("intrinsic", "obj_id"), R,
                                                   masks=masks)
        occluders = self._occluders("estimate_translation", occluders, masks)
        B, k = R.shape[:2]
        t = torch.empty((B, k, 3), device=self.device, dtype=torch.float64)
        iou = torch.empty((B, k), device=self.device, dtype=torch.float64)
        for obj, ri, rd, pick in self._object_rows(ids):
            t[rd], iou[rd] = translation.estimate_translation(
                self.tless_cad[obj], pick(R), K[ri], pick(masks), diameter=self.bop_models[obj]["diameter"],
                iters=iters, occluders=pick(occluders))
        return t, iou

    @staticmethod
    def _occluders(name, occluders, masks):
        """occluders [B, H, W] with the masks' shape, or None; errors name the fit"""
        if occluders is None:
            return None
        from ._posefit import _tensor
        occluders = _tensor(occluders)
        if tuple(occluders.shape) != tuple(masks.shape):
            raise ValueError(f"{name}: occluders {tuple(masks.shape)} (the masks' shape) expected, got "
                             f"{tuple(occluders.shape)}")
        return occluders

    @torch.no_grad()
    def refine_depth(self, batch, R, t, masks=None, iters=None, rerank=False):
        """Refine every pose hypothesis (R [B, k, 3, 3], t [B, k, 3] mm, e.g. a search's rotations with
        `estimate_translation`) of a T-LESS batch (the `eval_vsd` schema; its "intrinsic", "depth_path" and "obj_id"
        are used) against each frame's sensor depth, read as `eval_vsd` reads it, by point-to-plane ICP
        (`depth_refine.refine_pose_depth`, DESIGN.md section 19) with the mesh of load_mesh and the default tolerance
        schedule of the object's diameter (load_models_info); masks [B, H, W] (uint8 or bool, nonzero = object) limit
        the pairs to the object, None uses every pixel.  One call per distinct object.  -> (R float64 [B, k, 3, 3],
        t float64 [B, k, 3], score float64 [B, k]) on the model's device, score = the share of the mask's sensor
        pixels explained by the refined pose (NaN for a frame without readings); with rerank, each row's hypotheses
        sorted by descending score (stable, NaN last).  The output feeds eval_bop(R_est=R, t_est=t)."""
        from . import depth_refine
        iters = depth_refine.DEFAULT_ITERS if iters is None else iters
        ids, R, t, masks, K = self._pose_fit_batch("refine_depth", batch, ("intrinsic", "obj_id", "depth_path"), R, t,
                                                   masks)
        B, k = R.shape[:2]
        if len(batch["depth_path"]) != B:
            raise ValueError(f"refine_depth: {B} depth_path entries expected, got {len(batch['depth_path'])}")
        depth = self._read_sensor_depth(batch)
        R_out = torch.empty((B, k, 3, 3), device=self.device, dtype=torch.float64)
        t_out = torch.empty((B, k, 3), device=self.device, dtype=torch.float64)
        score = torch.empty((B, k), device=self.device, dtype=torch.float64)
        for obj, ri, rd, pick in self._object_rows(ids):
            tau = depth_refine.default_tau(self.bop_models[obj]["diameter"], iters)
            R_out[rd], t_out[rd], fit = depth_refine.refine_pose_depth(
                self.tless_cad[obj], pick(R), pick(t), K[ri], depth[ri], masks=pick(masks), iters=iters, tau=tau)
            score[rd] = fit["score"]
        return self._rerank(score, R_out, t_out) if rerank else (R_out, t_out, score)

    @torch.no_grad()
    def refine_contour(self, batch, R, t, masks, iters=None, rerank=False, occluders=None):
        """Refine every pose hypothesis (R [B, k, 3, 3], t [B, k, 3] mm, e.g. a search's rotations with
        `estimate_translation`) of a T-LESS batch (the `eval_vsd` schema; its "intrinsic" and "obj_id" are used)
        against each frame's object mask masks [B, H, W] (uint8 or bool, nonzero = object; (H, W) the frame size) by
        aligning the rendered silhouette's contour with the mask's (`contour_refine.refine_pose_contour`, DESIGN.md
        section 20), with the mesh of load_mesh and the default tolerance schedule.  No depth image is read.
        occluders [B, H, W] (uint8 or bool, nonzero = something may hide the object there) keep the fit off those
        pixels (DESIGN.md section 24); None is the plain refinement.  One call per distinct object.  -> (R float64 [B, k, 3, 3], t float64 [B, k, 3], iou float64 [B, k]) on the model's
        device, iou = the refined pose's silhouette IoU with the mask (NaN for a frame whose mask is empty or full);
        with rerank, each row's hypotheses sorted by descending IoU (stable, NaN last).  The output feeds
        eval_bop(R_est=R, t_est=t); refine_depth can follow when the frame has depth."""
        from . import contour_refine
        iters = contour_refine.DEFAULT_ITERS if iters is None else iters
        ids, R, t, masks, K = self._pose_fit_batch("refine_contour", batch, ("intrinsic", "obj_id"), R, t, masks,
                                                   models_info=False)
        occluders = self._occluders("refine_contour", occluders, masks)
        B, k = R.shape[:2]
        R_out = torch.empty((B, k, 3, 3), device=self.device, dtype=torch.float64)
        t_out = torch.empty((B, k, 3), device=self.device, dtype=torch.float64)
        iou = torch.empty((B, k), device=self.device, dtype=torch.float64)
        for obj, ri, rd, pick in self._object_rows(ids):
            R_out[rd], t_out[rd], fit = contour_refine.refine_pose_contour(
                self.tless_cad[obj], pick(R), pick(t), K[ri], pick(masks), iters=iters, occluders=pick(occluders))
            iou[rd] = fit["iou"]
        return self._rerank(iou, R_out, t_out) if rerank else (R_out, t_out, iou)

    @torch.no_grad()
    def predict_pose_frames(self, frames, masks, K, obj_ids, reference=None, all_relativeR=None, template_poses=None,
                            angles=36, k=5, refiner=None, refine=None, frame_idx=None, occluders=None, bank=None,
                            occluded_search=False):
        """6D poses of B detections in camera frames (DESIGN.md section 23): `crop.frame_crops` cuts a keep_inplane
        crop around each mask's `initial_translation` t0, the in-plane search (`predict_pose_inplane`, or
        `predict_pose_inplane_refined` with a refiner) finds the rotation in the crop's camera, `crop.to_camera`
        re-expresses it in the real camera, and `translation.estimate_translation` fits t from t0, with
        `contour_refine.refine_pose_contour` after it for refine="contour".
          frames     uint8 [F, H, W, 3] RGB; masks uint8 or bool [B, H, W] (one per detection, nonzero = object)
          K          [3, 3] or [B, 3, 3] intrinsics, read on the host; obj_ids B ids on the host, each with a mesh
                     (load_mesh) and a models_info entry (load_models_info: the diameter)
          reference  [1 | B, 3, 256, 256], all_relativeR [1 | B, N, 6] and template_poses [N, 3, 3] as
                     predict_pose_inplane takes them: the templates' rotations in the query crop's camera
          frame_idx  integer [B], or None when F == B
          angles     the search's in-plane bins; a refiner brings its own (refiner.angles)
          occluders  None; [B, H, W] uint8 or bool (nonzero = something may hide the detection's object there); or
                     "detections": each detection's occluders are the other detections of its frame
                     (`crop.detection_occluders`).  The translation fit and the contour refinement then ignore those
                     pixels (DESIGN.md section 24); None is the plain fits, bit for bit.
          bank       a TemplateBank (build_template_bank) holding every obj_id, in place of reference, all_relativeR
                     and template_poses: the search is then predict_pose_bank (predict_pose_bank_refined with a
                     refiner), which scores each crop against its object's stored templates instead of sweeping the
                     reference (DESIGN.md section 25).  Give either the bank or reference and all_relativeR.
          occluded_search  True: the search too leaves out what the occluders may hide -- its hidden= is
                     crop_hidden of the occluders through each crop's map (DESIGN.md section 27); needs occluders.
                     False is the search without them, bit for bit.
        -> {"R": float64 [B, k, 3, 3] in the real camera, "t": float64 [B, k, 3] mm, "score": the search's [B, k],
        "iou": the silhouette IoU [B, k], "R_crop": the search's rotations [B, k, 3, 3], "t0": [B, 3],
        "crops": [B, 3, 256, 256]}.  R and t go unchanged into eval_bop(R_est=, t_est=), refine_depth and
        select_distinct.  The only host synchronisation beyond the search's is frame_crops' copy of t0."""
        from .crop import frame_crops
        ids = self._frame_ids("predict_pose_frames", masks, obj_ids, refine, occluders, occluded_search)
        B = len(ids)
        self._frame_templates("predict_pose_frames", B, ids, bank, reference, all_relativeR, template_poses,
                              getattr(refiner, "angles", angles))
        crops, t0, Rv, inv_maps = frame_crops(frames, masks, K, self._diameters(ids), image_size=256,
                                              frame_idx=frame_idx)
        occ = {}                                   # the search's hidden=, passed only when there is one
        if occluded_search:
            occluders = self._frame_occluders("predict_pose_frames", frames, masks, frame_idx, occluders)
            occ["hidden"] = self._crop_hidden(occluders, inv_maps)
        if bank is not None and refiner is None:
            R_crop, nearest, angle, sim = self.predict_pose_bank(crops, ids, bank, k=k, angles=angles, **occ)
            N = sim.shape[-1]
            score = sim.reshape(B, -1).gather(1, angle * N + nearest)
        elif bank is not None:
            R_crop, _, _, score = self.predict_pose_bank_refined(crops, ids, bank, refiner, k=k, **occ)
        elif refiner is None:
            R_crop, nearest, angle, sim = self.predict_pose_inplane(crops, reference, all_relativeR, template_poses,
                                                                    k=k, angles=angles, **occ)
            N = sim.shape[-1]
            score = sim.reshape(B, -1).gather(1, angle * N + nearest)
        else:
            R_crop, _, _, score = self.predict_pose_inplane_refined(crops, reference, all_relativeR, refiner, k=k,
                                                                    **occ)
        return self._frame_fits("predict_pose_frames", frames, masks, K, ids, frame_idx, occluders, refine, R_crop,
                                score, crops, t0, Rv)

    def _frame_ids(self, name, masks, obj_ids, refine, occluders, occluded_search=False):
        """The refusals of a pose from camera frames that do not depend on the search: refine, occluders (and
        occluded_search without them, or with model.dist), one obj_id per mask and a mesh and models_info entry for
        each.  -> the ids (host ints)"""
        import numpy as np
        if refine not in (None, "contour"):
            raise ValueError(f"refine must be None or 'contour', got {refine!r}")
        if isinstance(occluders, str) and occluders != "detections":
            raise ValueError(f"occluders must be None, a tensor or 'detections', got {occluders!r}")
        if occluded_search and occluders is None:
            raise ValueError(f"{name}: occluded_search=True needs occluders (a tensor or 'detections')")
        if occluded_search and self.dist is not None:
            raise NotImplementedError(f"{name}(occluded_search=True) does not shard across GPUs: it runs on one "
                                      "device (unset model.dist)")
        ids = [int(i) for i in np.asarray(obj_ids.detach().cpu() if torch.is_tensor(obj_ids) else obj_ids)
               .reshape(-1).tolist()]
        B = len(ids)
        if masks.shape[0] != B:
            raise ValueError(f"{name}: {B} obj_ids for {masks.shape[0]} masks")
        missing = sorted(set(i for i in ids if i not in self.tless_cad or i not in self.bop_models))
        if missing:
            raise ValueError(f"{name}: no mesh or models_info entry for obj_id {missing} (load_mesh, "
                             "load_models_info)")
        return ids

    def _frame_templates(self, name, B, ids, bank, reference, all_relativeR, template_poses, angles):
        """The refusals of where a frame search's templates come from: either a bank holding every id (checked
        with `angles` bins) or reference [1 | B] and all_relativeR"""
        if bank is not None:
            if reference is not None or all_relativeR is not None or template_poses is not None:
                raise ValueError(f"{name}: give either a bank or reference, all_relativeR and template_poses, not "
                                 "both")
            from .bank import check_bank_search
            # the bank, the engine and the ids before the crops; the search checks its own k / keep again
            check_bank_search(bank, self.u_net, B, ids, angles, 1)
        elif reference is None or all_relativeR is None:
            raise ValueError(f"{name}: reference and all_relativeR (with template_poses), or a bank, expected")
        elif reference.shape[0] not in (1, B):
            raise ValueError(f"{name}: reference [1 | B, 3, 256, 256] with B = {B} expected, got "
                             f"{tuple(reference.shape)}")

    def _frame_occluders(self, name, frames, masks, frame_idx, occluders):
        """occluders as the fits take them: "detections" becomes crop.detection_occluders of the masks (on the
        device), a tensor is checked against the masks' shape"""
        from .crop import _tensor, detection_occluders
        masks = _tensor(masks)
        if isinstance(occluders, str):
            from .bop import _to_dev
            md = masks if masks.device.type == "cuda" else _to_dev(masks, self.device, masks.dtype)
            occluders = detection_occluders(md, frame_idx, num_frames=_tensor(frames).shape[0])
        return self._occluders(name, occluders, masks)

    def _crop_hidden(self, occluders, inv_maps):
        """the search's hidden= of occluders [B, H, W] through the crops' maps (crop_hidden)"""
        from .crop import _to_device
        from .visibility import crop_hidden
        return crop_hidden(_to_device(self.device, occluders), inv_maps)

    def _diameters(self, ids):
        import numpy as np
        return np.array([self.bop_models[i]["diameter"] for i in ids], dtype=np.float64)

    def _frame_fits(self, name, frames, masks, K, ids, frame_idx, occluders, refine, R_crop, score, crops, t0, Rv):
        """The stages of a pose from camera frames after the search: crop-camera rotations R_crop [B, k, 3, 3] to the
        real camera, the occluders, the translation fit from t0 and, for refine="contour", the contour refinement.
        -> the dict of predict_pose_frames"""
        from . import contour_refine, translation
        from .crop import _as_numpy, _tensor, to_camera
        import numpy as np
        B = len(ids)
        R = to_camera(R_crop.to(self.device), Rv.to(self.device))
        masks = _tensor(masks)
        occluders = self._frame_occluders(name, frames, masks, frame_idx, occluders)
        Kh = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(_as_numpy(K, "K").reshape(-1, 3, 3), (B, 3, 3))))
        kk = R.shape[1]
        t = torch.empty((B, kk, 3), device=self.device, dtype=torch.float64)
        iou = torch.empty((B, kk), device=self.device, dtype=torch.float64)
        R_out = torch.empty_like(R) if refine == "contour" else R
        for obj, ri, rd, pick in self._object_rows(ids):
            mesh = self.tless_cad[obj]
            t_o, iou_o = translation.estimate_translation(mesh, pick(R), Kh[ri], pick(masks), t_init=pick(t0),
                                                          occluders=pick(occluders))
            if refine == "contour":
                R_o, t_o, fit = contour_refine.refine_pose_contour(mesh, pick(R), t_o, Kh[ri], pick(masks),
                                                                   occluders=pick(occluders))
                R_out[rd], iou_o = R_o, fit["iou"]
            t[rd], iou[rd] = t_o, iou_o
        return {"R": R_out, "t": t, "score": score, "iou": iou, "R_crop": R_crop, "t0": t0, "crops": crops}

    @torch.no_grad()
    def track_pose_frames(self, frames, masks, K, obj_ids, R_prior, refiner, bank=None, reference=None,
                          all_relativeR=None, template_poses=None, k=5, refine=None, frame_idx=None, occluders=None,
                          occluded_search=False):
        """predict_pose_frames with the search replaced by a refinement from prior rotations (DESIGN.md section 26):
        R_prior [B, P, 3, 3] (1 <= P <= 16) in the real camera, e.g. the previous frame's R[:, :keep], is taken into
        each new crop's camera (crop.to_crop), mapped to refinement centres and refined by the refiner's steps
        (track.track_inplane), without the A rotated copies of a search.  refiner: an InplaneRefiner over the grid of
        the bank or of all_relativeR (template_poses, when given, must be that grid).  frames, masks, K, obj_ids, bank
        or reference / all_relativeR, refine, frame_idx, occluders and occluded_search as predict_pose_frames takes
        them.
        -> predict_pose_frames' dict, "score" the refined score of each of the k poses.  Per detection it encodes P *
        (1 + 2 * steps) rotated crops and sweeps 9 * P * steps hypotheses; the host synchronises as often as in
        predict_pose_frames."""
        from .crop import frame_crops, to_crop
        from .inplane_refine import InplaneRefiner, pose_rotations
        from .track import check_track_args, track_inplane
        if self.dist is not None:
            raise NotImplementedError("track_pose_frames does not shard across GPUs: it runs on one device (unset "
                                      "model.dist)")
        if not isinstance(refiner, InplaneRefiner):
            raise ValueError("refiner must be a nope_b200.inplane_refine.InplaneRefiner")
        ids = self._frame_ids("track_pose_frames", masks, obj_ids, refine, occluders, occluded_search)
        B = len(ids)
        self._frame_templates("track_pose_frames", B, ids, bank, reference, all_relativeR, template_poses,
                              refiner.angles)
        R_prior = R_prior if torch.is_tensor(R_prior) else torch.as_tensor(R_prior)
        if bank is not None:
            bank.check_grid(refiner.template_poses)
            check_track_args(refiner, bank.all_relativeR, R_prior, k, B)
        else:
            check_track_args(refiner, all_relativeR, R_prior, k, B, reference.shape[0])
            if template_poses is not None and not torch.equal(
                    torch.as_tensor(template_poses).detach().cpu().to(torch.float64), refiner.template_poses):
                raise ValueError("track_pose_frames: template_poses is not the refiner's grid")
        metric = self._metric()
        crops, t0, Rv, inv_maps = frame_crops(frames, masks, K, self._diameters(ids), image_size=256,
                                              frame_idx=frame_idx)
        occ = {}
        if occluded_search:
            occluders = self._frame_occluders("track_pose_frames", frames, masks, frame_idx, occluders)
            occ["hidden"] = self._crop_hidden(occluders, inv_maps)
        dev = self.device
        R_prior_crop = to_crop(R_prior.to(dev), Rv.to(dev))
        self.u_net.set_metric(metric, self._occlusion_threshold())
        if bank is not None:
            from .track import _index
            slots = _index(bank.slots(ids), bank.device)
            ref_feat = bank.reference_latents.index_select(0, slots)
            rel = bank.all_relativeR.index_select(0, slots)
        else:
            ref_feat = self.u_net.encoder.encode_image(reference.to(dev))
            ref_feat = ref_feat.expand(B, *ref_feat.shape[1:])
            rel = all_relativeR.to(dev).expand(B, *all_relativeR.shape[1:])
        out = track_inplane(self.u_net, self.u_net.encoder, ref_feat, crops, rel, R_prior_crop, refiner, k=k, **occ)
        R_crop = pose_rotations(out["D"], out["seed"], out["cossin"], refiner)
        return self._frame_fits("track_pose_frames", frames, masks, K, ids, frame_idx, occluders, refine, R_crop,
                                out["score"], crops, t0, Rv)

    @torch.no_grad()
    def eval_bop(self, batch, data_name, R_est=None, save_path=None, t_est=None):
        """BOP 2019 average recall of a T-LESS batch (the `eval_vsd` schema): the grid retrieval's top-5 rotations, or
        R_est [B, k, 3, 3] from any search, at the ground-truth translation, or at t_est [B, k, 3] (mm, e.g. from
        `estimate_translation`) when given: the estimates are then rendered, and MSSD / MSPD computed, at t_est; the
        ground truth keeps its pose.  Each frame is rendered once (ground truth and k estimates); one multi-tau VSD
        call (tau = 0.05 ... 0.5 x diameter) and one pose_errors call per distinct object.  Logs and returns
        {"top kk, ar_vsd" / "ar_mssd" / "ar_mspd" / "ar"} for kk in {1, 3, 5} (up to k): the per-metric minimum over
        the first kk estimates; kk = 1 is the BOP figure.  Saves the errors (vsd [B, k, 10], mssd [B, k], mspd [B, k],
        obj_id [B]) to save_path (.npz) when given."""
        import numpy as np
        from . import bop
        from . import vsd as _vsd
        B, ids = self._check_vsd_batch(batch)
        missing = sorted(set(i for i in ids if i not in self.bop_models))
        if missing:
            raise ValueError(f"eval_bop: no models_info entry for obj_id {missing} (load_models_info)")
        if R_est is None:
            R = self._grid_rotations(batch, B)
        else:
            R = torch.as_tensor(np.asarray(R_est) if not torch.is_tensor(R_est) else R_est)
            if R.dim() != 4 or R.shape[0] != B or R.shape[2:] != (3, 3) or R.shape[1] < 1:
                raise ValueError(f"eval_bop: R_est [B, k, 3, 3] with B = {B} expected, got {tuple(R.shape)}")
            R = R.to(self.device)
        k = R.shape[1]
        if t_est is not None:
            t_est = torch.as_tensor(np.asarray(t_est) if not torch.is_tensor(t_est) else t_est)
            if tuple(t_est.shape) != (B, k, 3):
                raise ValueError(f"eval_bop: t_est [{B}, {k}, 3] expected, got {tuple(t_est.shape)}")
            t_est = bop._to_dev(t_est, self.device, torch.float64)
        depth_test, rendered, K, K4 = self._render_frames(batch, B, ids, R, t_est)
        W = depth_test.shape[2]
        dev = rendered.device
        vsd = torch.empty((B, k, len(bop.VSD_TAUS)), device=dev, dtype=torch.float64)
        mssd = torch.empty((B, k), device=dev, dtype=torch.float64)
        mspd = torch.empty((B, k), device=dev, dtype=torch.float64)
        gt = torch.cat([batch["query_pose"].detach().to(torch.float64).reshape(B, 3, 3),
                        batch["query_translation"].detach().to(torch.float64).reshape(B, 3, 1)], dim=2)
        gt = gt.pin_memory().to(dev, non_blocking=True) if gt.device.type == "cpu" else gt.to(dev)
        R_gt, t_gt = gt[:, :, :3], gt[:, :, 3]
        diameter = np.array([self.bop_models[i]["diameter"] for i in ids])
        for obj, ri, rd, _ in self._object_rows(ids):
            info = self.bop_models[obj]
            vsd[rd] = _vsd.vsd_errors(depth_test[rd], rendered[rd, 0], rendered[rd, 1:], K[ri],
                                      tau=bop.VSD_TAUS * info["diameter"])
            e_mssd, e_mspd = bop.pose_errors(self.tless_cad[obj].vertices, R[rd], t_gt[rd] if t_est is None else
                                             t_est[rd], R_gt[rd], t_gt[rd], K[ri], info["symmetries"])
            mssd[rd], mspd[rd] = e_mssd, e_mspd
        vsd, mssd, mspd = vsd.cpu().numpy(), mssd.cpu().numpy(), mspd.cpu().numpy()
        final_scores = {}
        for kk in [1, 3, 5]:
            if kk > k:
                continue
            ar = bop.average_recall(vsd[:, :kk], mssd[:, :kk], mspd[:, :kk], diameter, W)
            for name, value in ar.items():
                final_scores[f"top {kk}, {name}"] = value
        self.log_score(final_scores, split_name=f"val_{data_name}")
        if save_path is not None:
            os.makedirs(os.path.dirname(os.path.abspath(save_path)), exist_ok=True)
            np.savez(save_path, vsd=vsd, mssd=mssd, mspd=mspd, obj_id=np.array(ids))
        return final_scores

    def test_step(self, batch, idx_batch):
        """model.py:550-565: one entry per dataloader, keyed "<dataset>_<category>"; tless_<category> goes to eval_vsd
        (saving to log_dir when the model has one), anything else to eval_geodesic."""
        out = {}
        for dataloader_name in batch.keys():
            data_name, category = dataloader_name.split("_")
            if data_name in ["tless"]:
                save_path = None if self.log_dir is None else os.path.join(
                    self.log_dir, f"vsd_{category}_batch{idx_batch}_rank_{self.global_rank}.npy")
                out[dataloader_name] = self.eval_vsd(batch[dataloader_name], category, save_path=save_path)
                continue
            out[dataloader_name] = self.eval_geodesic(batch[dataloader_name], category, visualize=True,
                                                      save_prediction=True)
        self.global_step += 1
        return out


def broadcast_batches(bq, bt):
    """Batch rule of the reference's retrieval (model.py:260-262), where [Bq,1,...] queries meet [Bt,N,...]
    templates: -> (B, Q, Bt, rows of the result) in the terms of nope_score_topk_multi.  Equal batches pair
    up, a template batch of 1 serves every query, a query batch of 1 is scored against every template batch;
    anything else raises ValueError (torch would not broadcast it either)."""
    if bq < 1 or bt < 1:
        raise ValueError(f"empty batch (query {bq}, templates {bt})")
    if bq == bt:
        return bq, 1, bt, bq
    if bt == 1:
        return 1, bq, 1, bq
    if bq == 1:
        return bt, 1, bt, bt        # the one query is repeated per template batch
    raise ValueError(f"query batch {bq} and template batch {bt} do not broadcast (equal, or one of them 1)")


def score_topk(query_feat, template_feat, k=5, metric="l2", idx_base=0, threshold=0.2, visible=None):
    """similarity [B,N] and nearest_idx [B,k] of materialised templates
    (the arithmetic of model.py:260-265) on the GPU.  query_feat [Bq,C,h,w] and template_feat [Bt,N,C,h,w]
    broadcast as in the reference (broadcast_batches): B = max(Bq, Bt).  visible [Bq, 32, 32] (uint8 or bool,
    DESIGN.md section 27): each query scores only the latent pixels its map marks non-zero."""
    check_metric(metric)
    if template_feat.dim() != 5 or query_feat.dim() != 4 or tuple(query_feat.shape[1:]) != tuple(template_feat.shape[2:]):
        raise ValueError(f"query_feat [B,C,h,w] and template_feat [B,N,C,h,w] expected; got "
                         f"{tuple(query_feat.shape)} and {tuple(template_feat.shape)}")
    B, Q, _, _ = broadcast_batches(query_feat.shape[0], template_feat.shape[0])
    dev = template_feat.device
    if dev.type != "cuda":
        raise _lib.NopeError("score_topk needs CUDA tensors (no CPU fallback)")
    N = template_feat.shape[1]
    if k > N:
        raise RuntimeError(f"selected index k out of range (k={k}, N={N})")  # torch.topk's error
    q = query_feat.to(dev, torch.float32)
    if q.shape[0] != B * Q:
        q = q.expand(B * Q, *q.shape[1:])
    if visible is not None:
        from .visibility import score_visible
        if visible.dtype not in (torch.uint8, torch.bool) or tuple(visible.shape) != (query_feat.shape[0], 32, 32):
            raise ValueError(f"visible [{query_feat.shape[0]}, 32, 32] uint8 or bool expected, got "
                             f"{tuple(visible.shape)} {visible.dtype}")
        vis = visible.to(dev)
        if vis.shape[0] != B * Q:
            vis = vis.expand(B * Q, *vis.shape[1:])
        Bt = template_feat.shape[0]
        # the broadcasting as groups: template batch g serves rows [g * B * Q / Bt, (g + 1) * B * Q / Bt)
        slots = torch.arange(Bt, device=dev, dtype=torch.int32)
        row_off = torch.arange(Bt + 1, device=dev, dtype=torch.int32) * (B * Q // Bt)
        sim, topi = score_visible(q.contiguous(), template_feat.to(torch.float32).contiguous(), slots, row_off, 1, vis,
                                  metric, threshold, k)
        if topi is None:
            topi = torch.empty((B * Q, 0), device=dev, dtype=torch.int64)
        return sim, (topi + idx_base if idx_base else topi)
    sim, _, topi = _score_multi(q.contiguous(), template_feat.to(torch.float32).contiguous(), B, Q, metric,
                                threshold, k, idx_base)
    return sim, topi


def _score_multi(q, t, B, Q, metric, threshold, k=0, idx_base=0):
    """nope_score_topk_multi on the current stream: q [B * Q, C, h, w] scored against t [Bt, N, C, h, w] (float32,
    contiguous, on one CUDA device) -> (sim [B * Q, N], topv [B * Q, k], topi [B * Q, k])"""
    dev = t.device
    sim = torch.empty((B * Q, t.shape[1]), device=dev, dtype=torch.float32)
    topv = torch.empty((B * Q, k), device=dev, dtype=torch.float32)
    topi = torch.empty((B * Q, k), device=dev, dtype=torch.int64)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().nope_score_topk_multi(
            _lib.ptr(q), _lib.ptr(t), B, Q, t.shape[0], t.shape[1], t.shape[2], t.shape[3] * t.shape[4],
            _METRICS[metric], float(threshold), k, _lib.ptr(sim), _lib.ptr(topv), _lib.ptr(topi), idx_base,
            _lib.stream(dev)))
    return sim, topv, topi


def topk(sim, k, idx_base=0):
    """Deterministic top-k of sim [B,N] on the GPU (descending, ties -> lowest index)."""
    lib = _lib.load()
    sim = sim.contiguous()
    B, N = sim.shape
    topv = torch.empty((B, k), device=sim.device, dtype=torch.float32)
    topi = torch.empty((B, k), device=sim.device, dtype=torch.int64)
    with torch.cuda.device(sim.device):
        _lib.check(lib.nope_topk(_lib.ptr(sim), B, N, k, _lib.ptr(topv), _lib.ptr(topi), idx_base,
                                 _lib.stream(sim.device)))
    return topv, topi


def build_model(u_net_dim=192, descriptor_size=8, device="cuda:0", chunk=642,
                similarity_metric="l2", precision="fp16"):
    """The one configuration the reference resolves: configs/model/template_base.yaml.
    precision: "fp16" (fast), "fp16_w2" (exact weights), "parity" (split precision, meets the
    1e-3 embedding tolerance of the fp32 reference with margin: 2.2e-4), "parity_fast" (the same with single-fp16
    tensors inside the ResnetBlocks: ~5e-4, 15 % faster) or "bf16" (BASELINE configs[2]: bf16 storage, ~1e-2)."""
    from .encoder import FeatureExtractor
    from .unet import UNet
    enc = FeatureExtractor(descriptor_size=descriptor_size, threshold=0.2, normalize=False)
    unet = UNet(u_net_dim=u_net_dim, rot_representation_dim=6, encoder=enc,
                pose_mlp_name="single_layer", device=device, chunk=chunk, precision=precision)
    return PoseConditional(unet, optim_config={"loss_type": "l1"},
                           testing_config={"similarity_metric": similarity_metric}, save_dir=None)
