"""Searches under occlusion (DESIGN.md section 27): the latent pixels an occluder may hide are left out of every
score.  A detection's occluders become a crop-space hidden mask through the crop's own warp (`crop_hidden`), each
rolled copy of the crop a visible map over the 32 x 32 latent grid (`latent_visibility`), and the sweeps and the
standalone scores take those maps (`UNet.sweep(query_visible=)`, `bank.score_rows(visible=)`).  All of it runs in
CUDA kernels; there is no CPU fallback."""
import torch

from . import _lib

IMAGE_SIZE = 256           # crops of 256 x 256 pixels: the 32 x 32 latent grid of the encoders
LATENT_SIDE = 32


def check_hidden(hidden, lead, name):
    """ValueError unless hidden is a crop-space mask [*lead, 256, 256] of dtype uint8 or bool (non-zero = may be
    hidden).  -> hidden as uint8 [prod(lead), 256, 256]"""
    lead = tuple(int(x) for x in lead)
    if not isinstance(hidden, torch.Tensor) or hidden.dtype not in (torch.uint8, torch.bool):
        raise ValueError(f"{name}: hidden must be a uint8 or bool tensor, got "
                         f"{getattr(hidden, 'dtype', type(hidden).__name__)}")
    if tuple(hidden.shape) != lead + (IMAGE_SIZE, IMAGE_SIZE):
        raise ValueError(f"{name}: hidden {lead + (IMAGE_SIZE, IMAGE_SIZE)} (the query's form) expected, got "
                         f"{tuple(hidden.shape)}")
    return hidden.reshape(-1, IMAGE_SIZE, IMAGE_SIZE)


def _u8(x, device):
    """x on `device` as contiguous uint8; host tensors travel through pinned memory, without blocking"""
    from .crop import _to_device
    return _to_device(device, x).to(torch.uint8).contiguous()


def crop_hidden(occluders, inv_maps, image_size=IMAGE_SIZE):
    """occluders [B, H, W] (uint8 or bool, non-zero = something may hide the object there), inv_maps [B, 3, 3]
    float64 (crop_frames' maps) -> hidden [B, S, S] uint8 on the occluders' device: crop pixel (x, y) is 1 when one
    of the taps of its crop_frames sample has a non-zero weight, lies inside the frame and is occluded."""
    if image_size != IMAGE_SIZE:
        raise ValueError(f"image_size must be {IMAGE_SIZE} (the 32 x 32 latent grid), got {image_size}")
    if not isinstance(occluders, torch.Tensor) or occluders.dim() != 3 or \
            occluders.dtype not in (torch.uint8, torch.bool):
        raise ValueError("occluders [B, H, W] uint8 or bool expected")
    B, H, W = occluders.shape
    maps = torch.as_tensor(inv_maps, dtype=torch.float64)
    if tuple(maps.shape) not in ((B, 3, 3), (B, 9)):
        raise ValueError(f"inv_maps [{B}, 3, 3] expected, got {tuple(maps.shape)}")
    dev = occluders.device
    if dev.type != "cuda":
        raise _lib.NopeError("crop_hidden needs CUDA tensors (no CPU fallback)")
    occ = _u8(occluders, dev)
    from .crop import _to_device
    maps = _to_device(dev, maps.reshape(B, 9))
    out = torch.empty((B, image_size, image_size), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().nope_crop_hidden(_lib.ptr(occ), H, W, _lib.ptr(maps), B, image_size, _lib.ptr(out),
                                                _lib.stream(dev)))
    return out


def latent_visibility(hidden, cossin, image_idx=None):
    """hidden [B, 256, 256] (uint8 or bool), pairs cossin [P, 2] fp32 and image_idx [P] (None: pair p is image p,
    P = B) -> visible [P, 32, 32] uint8 on hidden's device: 0 where the 8 x 8 block holds a pixel of image
    image_idx[p] rolled by cossin[p] that may be hidden.  An image index outside [0, B) gives an all-visible row."""
    hidden = check_hidden(hidden, hidden.shape[:-2], "latent_visibility")
    dev = hidden.device
    if dev.type != "cuda":
        raise _lib.NopeError("latent_visibility needs CUDA tensors (no CPU fallback)")
    from .crop import _to_device
    cossin = _to_device(dev, torch.as_tensor(cossin)).to(torch.float32).contiguous()
    if cossin.dim() != 2 or cossin.shape[1] != 2 or cossin.shape[0] < 1:
        raise ValueError(f"cossin [P, 2] expected, got {tuple(cossin.shape)}")
    P, B = cossin.shape[0], hidden.shape[0]
    if image_idx is None:
        if P != B:
            raise ValueError(f"without image_idx, cossin needs one pair per image ({B}), got {P}")
        image_idx = torch.arange(B, device=dev, dtype=torch.int32)
    image_idx = _to_device(dev, torch.as_tensor(image_idx)).to(torch.int32).contiguous()
    if tuple(image_idx.shape) != (P,):
        raise ValueError(f"image_idx [{P}] expected, got {tuple(image_idx.shape)}")
    hidden = _u8(hidden, dev)
    out = torch.empty((P, LATENT_SIDE, LATENT_SIDE), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().nope_latent_visibility(_lib.ptr(hidden), B, IMAGE_SIZE, _lib.ptr(image_idx),
                                                      _lib.ptr(cossin), P, _lib.ptr(out), _lib.stream(dev)))
    return out


def latent_visibility_inplane(hidden, A):
    """The in-plane table form: hidden [B, 256, 256] -> visible [B, A, 32, 32], row (b, a) the map of image b rolled
    by inplane_table(A)[a], as encode_image_inplane rolls the crops."""
    from .inplane import _on_device, inplane_table
    hidden = check_hidden(hidden, hidden.shape[:-2], "latent_visibility_inplane")
    B, dev = hidden.shape[0], hidden.device
    table = _on_device(inplane_table, A, dev)
    idx = torch.arange(B, device=dev, dtype=torch.int32).repeat_interleave(A)
    return latent_visibility(hidden, table.repeat(B, 1), idx).view(B, A, LATENT_SIDE, LATENT_SIDE)


def query_visible(hidden, lead, name):
    """The maps of unrolled queries: hidden [*lead, 256, 256] -> visible [*lead, 32, 32] (roll (1, 0))."""
    flat = check_hidden(hidden, lead, name)
    cs = torch.zeros((flat.shape[0], 2), dtype=torch.float32, device=flat.device)
    cs[:, 0] = 1.0                                   # filled on the device: no host copy
    return latent_visibility(flat, cs).view(*lead, LATENT_SIDE, LATENT_SIDE)


def score_visible(query, templates, slots, row_off, A, visible, metric, threshold, k):
    """nope_score_topk_visible on the current stream: query rows [R, C, 32, 32] with their visible maps [R, 32, 32]
    against templates [O, N, C, 32, 32]; group g's rows [row_off[g], row_off[g + 1]) against template set slots[g]
    (int32 device tensors).  -> (sim [R, N], top [R / A, k] at a * N + n jointly over every A consecutive rows | None
    for k = 0)"""
    from .search import _METRICS
    dev = templates.device
    R, N = query.shape[0], templates.shape[1]
    q = query.to(dev, torch.float32).contiguous()
    vis = visible.to(dev).to(torch.uint8).contiguous()
    if tuple(vis.shape) != (R, LATENT_SIDE, LATENT_SIDE):
        raise ValueError(f"visible [{R}, 32, 32] expected, got {tuple(vis.shape)}")
    sim = torch.empty((R, N), device=dev, dtype=torch.float32)
    # the entry point writes the top-k scores beside the indices; the searches rank by the indices and read the scores
    # from sim, as with nope_score_topk_grouped
    topv = torch.empty((R // A, k), device=dev, dtype=torch.float32) if k else None
    topi = torch.empty((R // A, k), device=dev, dtype=torch.int64) if k else None
    with torch.cuda.device(dev):
        _lib.check(_lib.load().nope_score_topk_visible(
            _lib.ptr(q), _lib.ptr(templates), R, templates.shape[0], N, templates.shape[2],
            templates.shape[3] * templates.shape[4], _lib.ptr(slots), _lib.ptr(row_off), slots.shape[0], A,
            _lib.ptr(vis), _METRICS[metric], float(threshold), k, _lib.ptr(sim), _lib.ptr(topv), _lib.ptr(topi),
            _lib.stream(dev)))
    return sim, topi
