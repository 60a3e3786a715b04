"""The pose-search front end shared by `PoseConditional` (images) and `UNetModelPose` (latents): the query forms, the
similarity metrics, the rotation lookup and the grid, coarse-to-fine and refined searches on latents, written against
any engine with `sweep()` (`UNet`, `UNetModelPose`).  Each search returns in the query form it was given."""
import torch

_METRICS = {"l2": 0, "cosine": 1, "cosine_occlusion": 2}     # NOPE_METRIC_* of include/nope_b200.h


def check_metric(metric):
    """ValueError for a similarity metric no kernel scores; -> metric"""
    if metric not in _METRICS:
        raise ValueError(f"unknown similarity_metric {metric!r} (supported: {sorted(_METRICS)})")
    return metric


def multi_query_form(query, reference):
    """-> (query, squeeze).  query [B,...] with reference [B,...]: one query per reference, as given.
    query [B,Q,...]: Q queries per reference, as given.  query [Q,...] with reference [1,...]: the broadcast form,
    returned as [1,Q,...] with squeeze=True (outputs lose the leading 1).  Anything else raises ValueError."""
    B, rest = reference.shape[0], tuple(reference.shape[1:])
    if query.dim() == reference.dim() and tuple(query.shape[1:]) == rest:
        if query.shape[0] == B:
            return query, False
        if B == 1 and query.shape[0] >= 1:
            return query.unsqueeze(0), True
    elif query.dim() == reference.dim() + 1 and tuple(query.shape[2:]) == rest and query.shape[0] == B \
            and query.shape[1] >= 1:
        return query, False
    raise ValueError(f"query {tuple(query.shape)} does not fit reference {tuple(reference.shape)}: expected "
                     f"[B, ...], [B, Q, ...] or (one reference) [Q, ...]")


def query_rows(query_feat, ref_feat, rest=None):
    """(Q, leading output shape) of a sweep's queries: [B, *rest] is one query per reference (outputs [B, ...]),
    [B, Q, *rest] Q queries per reference (outputs [B, Q, ...]); rest defaults to the reference's per-image shape."""
    B = ref_feat.shape[0]
    rest = tuple(ref_feat.shape[1:]) if rest is None else tuple(rest)
    if query_feat.dim() == 1 + len(rest) and tuple(query_feat.shape) == (B,) + rest:
        return 1, (B,)
    if query_feat.dim() == 2 + len(rest) and query_feat.shape[0] == B and \
            tuple(query_feat.shape[2:]) == rest and query_feat.shape[1] >= 1:
        return int(query_feat.shape[1]), (B, int(query_feat.shape[1]))
    raise ValueError(f"query_feat must be [B, ...] or [B, Q, ...] with the per-query shape {(B,) + rest}; got "
                     f"{tuple(query_feat.shape)}")


def row_pairs(device, ref_feat, query, rest=None):
    """The (reference, query) rows that the fine stages of a search sweep, one reference row per query (Q = 1).
    ref_feat [B, C, h, w]; query [B, *rest] or [B, Q, *rest] (rest as in query_rows).  -> (ref_feat, query as float32
    contiguous on `device`, Q, lead, ref_rows [B * Q, C, h, w] (each reference repeated for its queries), query rows
    [B * Q, *rest])."""
    Q, lead = query_rows(query, ref_feat, rest)
    ref_feat = ref_feat.to(device, torch.float32).contiguous()
    query = query.to(device, torch.float32).contiguous()
    B, ref_rest = ref_feat.shape[0], ref_feat.shape[1:]
    ref_rows = ref_feat[:, None].expand(B, Q, *ref_rest).reshape(B * Q, *ref_rest)
    return ref_feat, query, Q, lead, ref_rows, query.reshape(B * Q, *query.shape[len(lead):])


def lookup_rotations(template_poses, idx):
    """template_poses[idx] on idx's device: template_poses [N, 3, 3] as given, [B, N, 3, 3] by its row 0 (the
    reference's template_poses[0][nearest_idx], model.py:352)."""
    tp = template_poses[0] if template_poses.dim() == 4 else template_poses
    return tp.to(idx.device)[idx]


def _unsqueezed(squeeze, *xs):
    """xs without their leading 1 in the broadcast form"""
    return tuple(x[0] for x in xs) if squeeze else xs


def grid_search(engine, ref_feat, query_feat, all_relativeR, template_poses=None, k=5, return_templates=False,
                dist=None, metric="l2", threshold=0.2, query_visible=None):
    """The exhaustive search: one sweep of all_relativeR [B, N, 6] scores every query in its last layer.
    k is clamped to N.  dist: a nope_b200.dist.ShardedSweep to split the grid across GPUs (it selects the metric).
    query_visible (the query's leading shape + [32, 32]): each query scores only its visible latent pixels.
    -> (R | None, nearest_idx, similarity[, templates]) in the query form of query_feat; under dist the templates are
    this rank's (local templates, lo, hi)."""
    query_feat, squeeze = multi_query_form(query_feat, ref_feat)
    if query_visible is not None and squeeze:
        query_visible = query_visible.unsqueeze(0)
    k = min(k, all_relativeR.shape[1])
    if dist is not None:
        sim, topi, emb = dist.sweep(engine, ref_feat, all_relativeR, query_feat, k=k, metric=metric,
                                    want_emb=return_templates, threshold=threshold)
    else:
        vis = {} if query_visible is None else {"query_visible": query_visible}
        out = engine.sweep(ref_feat, all_relativeR, query_feat=query_feat, want_emb=return_templates, k=k, **vis)
        sim, topi, emb = out["sim"], out["topi"], out["emb"]
    sim, topi = _unsqueezed(squeeze, sim, topi)
    R = None if template_poses is None else lookup_rotations(template_poses, topi)
    return (R, topi, sim, emb) if return_templates else (R, topi, sim)


def coarse_to_fine_search(engine, ref_feat, query_feat, all_relativeR_levels, hierarchy, template_poses=None, k=5,
                          keep=8):
    """hierarchy.search in the query form of query_feat: -> (R | None, nearest_idx, similarity [..., N_L])"""
    from .hierarchy import search
    query_feat, squeeze = multi_query_form(query_feat, ref_feat)
    out = search(engine, ref_feat, query_feat, all_relativeR_levels, hierarchy, keep=keep, k=k)
    sim, topi = _unsqueezed(squeeze, out["sim"], out["topi"])
    R = None if template_poses is None else lookup_rotations(template_poses, topi)
    return R, topi, sim


def refined_search(engine, ref_feat, query_feat, all_relativeR, refiner, k=5, keep=2):
    """The sweep's top-`keep` grid poses of every (reference, query) row, refined by refine.refine, in the query form
    of query_feat: -> (R = D * template_poses[seed] (float64), seed_idx, score)"""
    from .refine import check_refine_args, refine, template_rotations
    check_refine_args(refiner, all_relativeR, keep, k, ref_feat.shape[0])
    query_feat, squeeze = multi_query_form(query_feat, ref_feat)
    seeds = engine.sweep(ref_feat, all_relativeR, query_feat=query_feat, want_emb=False, want_sim=False,
                         k=keep)["topi"]
    out = refine(engine, ref_feat, query_feat, all_relativeR, seeds, refiner, k=k)
    D, seed, score = _unsqueezed(squeeze, out["D"], out["seed"], out["score"])
    return template_rotations(D, seed, refiner), seed, score
