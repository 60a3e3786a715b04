"""Host-side mirror of the reference `UNet` (src/model/u_net/denoising_diffusion_pytorch/
u_net.py:27-198) on top of the C ABI in include/nope_b200.h.

Same constructor arguments and the attributes the task module reads (`.encoder`,
`.channels`, `.name`, `__call__(x, pose)`); `load_state_dict` takes the reference's keys
unchanged.  All arithmetic runs in libnope_b200.so; this file only moves pointers.
"""
import ctypes as C

import torch

from . import _lib
from .search import _METRICS, query_rows

# precision option of the engine (include/nope_b200.h, nope_unet_set_option)
PRECISIONS = {"fp16": 0, "fp16_w2": 1, "parity": 2, "bf16": 3, "parity_fast": 4}


class _Incompatible:
    """return value of load_state_dict(strict=False), torch-style"""

    def __init__(self, missing, unexpected):
        self.missing_keys, self.unexpected_keys = missing, unexpected

    def __repr__(self):
        return f"<missing_keys={self.missing_keys}, unexpected_keys={self.unexpected_keys}>"


def encoder_entries(state_dict, encoder):
    """The `encoder.*` entries of a UNet state_dict that `encoder` loads, prefix stripped.  The SD VAE
    (nope_b200.vae.VAE_StableDiffusion) takes `encoder.encoder.*`: the AutoencoderKL it wraps
    (AutoencoderKL.py:16).  The template encoder takes `encoder.backbone.*` / `encoder.projector.*`; its
    `encoder.encoder.*` aliases (template.py:40) repeat the same tensors and are skipped."""
    from .vae import VAE_StableDiffusion
    out = {}
    for k, v in state_dict.items():
        if not k.startswith("encoder."):
            continue
        kk = k[len("encoder."):]
        if isinstance(encoder, VAE_StableDiffusion):
            if kk.startswith("encoder."):
                out[kk[len("encoder."):]] = v
        elif kk.startswith("backbone.") or kk.startswith("projector."):
            out[kk] = v
    return out


class SweepEngine:
    """What UNet and UNetModelPose share on top of their nope_<kind>_* engine: the handle, chunk and options, the
    launch profile and count, the sweep, forward and the debug tap.  A subclass provides `_create_args()` and
    `_configure(lib, h)`, which every handle gets before its weights."""

    def __init__(self, kind, chunk, tap_channels):
        self._native = _lib.Engine(kind)
        self._chunk = chunk
        self._options = {}                  # nope_<kind>_set_option name -> value, applied to every engine
        self._tap_channels = tap_channels   # debug_tap's output capacity: channels at 32 x 32 per pose

    def _handle(self):
        return self._native.handle(self._create_args(), self._configure)

    def _reserve(self, hyps, refs, scores):
        """Sizes the caller-owned workspace before a launch (UNet.reserve); the LDM engine has none."""

    def set_chunk(self, hyps):
        self._chunk = hyps
        if self._native.h is not None:
            self._native.call("set_chunk", hyps)

    def set_option(self, name, value):
        """Named engine option (include/nope_b200.h, nope_<kind>_set_option), e.g. the LDM engine's 'hoist'.  It is
        applied at once, to a weightless engine if none is built yet, and kept for every later build; unknown names
        raise NopeError and are not kept."""
        self._handle()
        self._native.call("set_option", name.encode(), int(value))
        self._options[name] = int(value)

    @property
    def last_launch_count(self):
        self._handle()
        return self._native.launch_count()

    def profile(self, enable):
        self._handle()
        self._native.call("profile", 1 if enable else 0)

    def sweep(self, ref_feat, poses, query_feat=None, want_emb=True, want_sim=None, k=0, idx_base=0, out=None,
              query_visible=None):
        """ref_feat [B,C,32,32], poses [B,N,6] (+ query_feat [B,C,32,32]) ->
        dict(emb [B,N,C,32,32] | None, sim [B,N] | None, topv/topi [B,k] | None).
        query_feat may also be [B,Q,C,32,32]: Q queries per reference share the one sweep and
        sim is [B,Q,N], topv/topi [B,Q,k].
        `out` may carry preallocated contiguous `sim` / `topv` / `topi` tensors to write into (the
        multi-GPU path points them into its all-gather record).
        query_visible (uint8 or bool, the query's leading shape + [32, 32], DESIGN.md section 27): each row scores
        only the latent pixels its map marks non-zero (nope_*_sweep_visible)."""
        if not self._native.finalized:
            raise _lib.NopeError("load_state_dict() must be called before the sweep")
        dev = self.device
        if query_visible is not None and query_feat is None:
            raise ValueError("query_visible needs query_feat")
        ref_feat, poses, query_feat, Q, emb, sim, topv, topi = stage_sweep(self, ref_feat, poses, query_feat,
                                                                           want_emb, want_sim, k, out)
        B, N = poses.shape[0], poses.shape[1]
        if query_visible is not None:
            lead = tuple(query_feat.shape[:-3])
            if query_visible.dtype not in (torch.uint8, torch.bool) or tuple(query_visible.shape) != lead + (32, 32):
                raise ValueError(f"query_visible {lead + (32, 32)} uint8 or bool expected, got "
                                 f"{tuple(query_visible.shape)} {query_visible.dtype}")
            query_visible = query_visible.to(dev).to(torch.uint8).contiguous()
        self._reserve(min(self._chunk, B * N), B, B * Q * N if query_feat is not None else 0)
        with torch.cuda.device(dev):
            if query_visible is None:
                self._native.call("sweep_multi", _lib.ptr(ref_feat), _lib.ptr(poses), B, N, _lib.ptr(query_feat), Q,
                                  _lib.ptr(emb), _lib.ptr(sim), k, _lib.ptr(topv), _lib.ptr(topi), idx_base,
                                  _lib.stream(dev))
            else:
                self._native.call("sweep_visible", _lib.ptr(ref_feat), _lib.ptr(poses), B, N, _lib.ptr(query_feat),
                                  Q, _lib.ptr(query_visible), _lib.ptr(emb), _lib.ptr(sim), k, _lib.ptr(topv),
                                  _lib.ptr(topi), idx_base, _lib.stream(dev))
        return {"emb": emb, "sim": sim, "topv": topv, "topi": topi}

    def __call__(self, x, pose):
        """forward(x [B,C,32,32], pose [B,6]) -> [B,C,32,32] (u_net.py:160-198, adapt_openaimodel.py)."""
        return self.sweep(x, pose[:, None, :], want_emb=True)["emb"][:, 0]

    forward = __call__

    def debug_tap(self, ref_feat, poses, tap):
        """Activation named `tap` (oracle tap names) for poses [N,6] of ONE reference."""
        dev = self.device
        ref_feat = ref_feat.to(dev, torch.float32).contiguous()
        poses = poses.to(dev, torch.float32).contiguous()
        N = poses.shape[0]
        cap = N * 32 * 32 * self._tap_channels
        out = torch.empty(cap, device=dev, dtype=torch.float32)
        c, s = C.c_int(), C.c_int()
        self._reserve(N, 1, 0)
        self._handle()
        with torch.cuda.device(dev):
            self._native.call("debug_tap", _lib.ptr(ref_feat), _lib.ptr(poses), N, tap.encode(), _lib.ptr(out), cap,
                              C.byref(c), C.byref(s), _lib.stream(dev))
        return out[: N * c.value * s.value * s.value].view(N, c.value, s.value, s.value)


class UNet(SweepEngine):
    def __init__(self, u_net_dim, rot_representation_dim, encoder, pose_mlp_name="single_layer",
                 init_dim=None, out_dim=None, use_hard_up_down=True, dim_mults=(1, 2, 4, 8),
                 resnet_block_groups=8, device="cuda:0", chunk=642, precision="fp16", **kwargs):
        # only the configuration the reference actually ships resolves to a valid model
        # (configs/model/template_base.yaml; SURVEY.md F7)
        if pose_mlp_name != "single_layer":
            raise ValueError("only pose_mlp_name='single_layer' is implemented")
        if rot_representation_dim != 6 or tuple(dim_mults) != (1, 2, 4, 8) or \
                resnet_block_groups != 8 or not use_hard_up_down or \
                (init_dim not in (None, u_net_dim)) or \
                (out_dim not in (None, encoder.latent_dim)):
            raise ValueError("unsupported UNet configuration (template_base.yaml values only)")
        if precision not in PRECISIONS:
            raise ValueError(f"precision must be one of {sorted(PRECISIONS)}")
        self.encoder = encoder
        self.channels = encoder.latent_dim
        self.name = encoder.name
        self.u_net_dim = u_net_dim
        self.rot_representation_dim = rot_representation_dim
        self.device = torch.device(device)
        self.precision = precision
        super().__init__("unet", chunk, 8 * u_net_dim)
        self._ws = None            # torch-owned workspace (uint8), handed to the engine
        self._ws_shape = (0, 0, 0)
        self._state = None         # last loaded UNet tensors (CPU fp32), kept for reload / partial load

    # ------------------------------------------------------------------ lifetime
    def _create_args(self):
        if self.device.type != "cuda":
            raise _lib.NopeError("nope_b200.UNet needs a CUDA device (no CPU fallback)")
        return self.u_net_dim, self.channels, 32, self.device.index or 0

    def _configure(self, lib, h):
        """chunk, precision and options: applied to every engine before its weights"""
        _lib.check(lib.nope_unet_set_chunk(h, self._chunk))
        _lib.check(lib.nope_unet_set_option(h, b"precision", PRECISIONS[self.precision]))
        for k, v in self._options.items():
            _lib.check(lib.nope_unet_set_option(h, k.encode(), v))

    def to(self, device):
        if self._native.h is not None and torch.device(device) != self.device:
            raise _lib.NopeError("cannot move a finalized engine; construct it on the target device")
        self.device = torch.device(device)
        self.encoder.to(self.device)
        return self

    def cuda(self, device=None):
        return self.to(torch.device("cuda", 0 if device is None else device))

    def eval(self):
        self.encoder.eval()
        return self

    # ------------------------------------------------------------------ weights
    def expected_shapes(self):
        """key -> shape of the 301 UNet tensors the engine expects (u_net.py:27-158)."""
        from .synth_weights import unet_param_shapes
        return dict(unet_param_shapes(self.u_net_dim, self.channels, self.rot_representation_dim))

    def load_state_dict(self, state_dict, strict=True):
        """Accepts the reference UNet state_dict: 301 UNet tensors plus `encoder.*` entries
        (SURVEY.md 8b).  May be called again (the engine is rebuilt).  strict=False follows torch:
        unexpected keys are skipped, missing keys keep their previous values (first load: error),
        and the (missing, unexpected) lists are returned.  A shape mismatch always raises, as
        nn.Module.load_state_dict does; the shape-FILTERED load of the reference
        (src/utils/weight.py:6-37) is nope_b200.weight.load_checkpoint."""
        want = self.expected_shapes()
        unet_sd, unexpected = {}, []
        enc_sd = encoder_entries(state_dict, self.encoder)
        for k, v in state_dict.items():
            if k.startswith("encoder."):
                continue
            if k not in want:
                unexpected.append(k)
                continue
            if tuple(v.shape) != tuple(want[k]):
                raise RuntimeError(f"size mismatch for {k}: checkpoint {tuple(v.shape)} vs model {tuple(want[k])}")
            unet_sd[k] = v.detach().to("cpu", torch.float32).contiguous()
        missing = [k for k in want if k not in unet_sd]
        if strict and (missing or unexpected):
            raise RuntimeError(f"Error(s) in loading state_dict for UNet: missing keys {missing[:5]}"
                               f"{'...' if len(missing) > 5 else ''}, unexpected keys {unexpected[:5]}")
        merged = dict(self._state or {})
        merged.update(unet_sd)
        still = [k for k in want if k not in merged]
        if still:
            raise RuntimeError(f"UNet tensors never provided: {still[:5]}{'...' if len(still) > 5 else ''}")
        create_args = self._create_args()
        if enc_sd:
            self.encoder.load_state_dict(enc_sd, strict=strict)
        self._native.destroy()    # weights are repacked at finalize: every load builds a fresh engine
        self._ws, self._ws_shape = None, (0, 0, 0)
        self._native.build(create_args, merged.items(), self._configure)
        self._state = merged
        self.encoder.to(self.device)
        return _Incompatible(missing, unexpected) if not strict else self

    def state_dict(self):
        """Reference-schema state_dict (CPU fp32): the UNet tensors last loaded (zeros for tensors never
        provided -- unlike the reference module this mirror has no random initialisation) plus the
        encoder's entries under `encoder.`."""
        want = self.expected_shapes()
        sd = {k: (self._state[k] if self._state and k in self._state else torch.zeros(shape))
              for k, shape in want.items()}
        if hasattr(self.encoder, "state_dict"):
            for k, v in self.encoder.state_dict().items():
                sd["encoder." + k] = v.detach().to("cpu")
        return sd

    def set_metric(self, metric, threshold=0.2):
        """Similarity metric of the scoring fused onto the sweep: 'l2' (the reference's, model.py:254-266),
        'cosine' or 'cosine_occlusion' (extensions; include/nope_b200.h NOPE_METRIC_*)."""
        _lib.check(_lib.load().nope_unet_set_metric(self._handle(), _METRICS[metric], float(threshold)))

    def set_conv_impl(self, impl):
        """'tcgen05_2cta': the clustered kernel with the fused epilogues, the engine's only convolution.  Anything else
        raises NopeError; the call changes nothing in the engine."""
        if impl != "tcgen05_2cta":
            raise _lib.NopeError(f"unknown conv impl {impl!r}: the only convolution is 'tcgen05_2cta' (conv_tc2_kernel)")

    def profile_read(self):
        """-> dict(conv_ms, conv_flops (executed), conv_alg_flops, conv_launches, max_launch_tflops)."""
        ms, fl, alg, n, best = C.c_double(), C.c_double(), C.c_double(), C.c_int64(), C.c_double()
        _lib.check(_lib.load().nope_unet_profile_read(self._handle(), C.byref(ms), C.byref(fl),
                                                      C.byref(alg), C.byref(n), C.byref(best)))
        return {"conv_ms": ms.value, "conv_flops": fl.value, "conv_alg_flops": alg.value,
                "conv_launches": n.value, "max_launch_tflops": best.value}

    # ------------------------------------------------------------------ workspace
    def reserve(self, hyps, refs, scores):
        """Size the engine's workspace from the torch caching allocator (SURVEY.md 8b ownership:
        no hidden cudaMalloc inside the sweep).  Grows only."""
        h, r, s = self._ws_shape
        if hyps <= h and refs <= r and scores <= s and self._ws is not None:
            return
        hyps, refs, scores = max(hyps, h), max(refs, r), max(scores, s)
        lib = _lib.load()
        need = lib.nope_unet_workspace_bytes(self._handle(), hyps, refs, scores)
        if need < 0:
            _lib.check(-1)
        ws = torch.empty(int(need), dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(lib.nope_unet_set_workspace(self._handle(), C.c_void_p(ws.data_ptr()), int(need),
                                                   hyps, refs, scores))
        self._ws, self._ws_shape = ws, (hyps, refs, scores)

    _reserve = reserve


def stage_sweep(engine, ref_feat, poses, query_feat, want_emb, want_sim, k, out):
    """The tensors of one sweep by `engine` (UNet or UNetModelPose): the inputs as contiguous float32 on its device,
    and the outputs, allocated or taken from `out` (preallocated `sim` / `topv` / `topi`, ValueError unless each has
    the output's shape and dtype, on the device, contiguous).  want_sim None means: when there are queries.
    -> (ref_feat, poses, query_feat | None, Q, emb | None, sim | None, topv | None, topi | None)"""
    dev = engine.device
    ref_feat = ref_feat.to(dev, torch.float32).contiguous()
    poses = poses.to(dev, torch.float32).contiguous()
    B, N = poses.shape[0], poses.shape[1]
    assert ref_feat.shape == (B, engine.channels, 32, 32), ref_feat.shape
    assert poses.shape[2] == engine.rot_representation_dim
    if want_sim is None:
        want_sim = query_feat is not None
    Q, lead = 1, (B,)
    if query_feat is not None:
        query_feat = query_feat.to(dev, torch.float32).contiguous()
        Q, lead = query_rows(query_feat, ref_feat)
    emb = torch.empty((B, N, engine.channels, 32, 32), device=dev, dtype=torch.float32) if want_emb else None
    out = out or {}
    sim = out.get("sim") if want_sim else None
    if want_sim and sim is None:
        sim = torch.empty(lead + (N,), device=dev, dtype=torch.float32)
    topv, topi = (out.get("topv"), out.get("topi")) if k > 0 else (None, None)
    if k > 0 and topv is None:
        topv = torch.empty(lead + (k,), device=dev, dtype=torch.float32)
        topi = torch.empty(lead + (k,), device=dev, dtype=torch.int64)
    for t, shape, dt in ((sim, lead + (N,), torch.float32), (topv, lead + (k,), torch.float32),
                         (topi, lead + (k,), torch.int64)):
        if t is not None and (tuple(t.shape) != shape or t.dtype != dt or not t.is_contiguous() or t.device != dev):
            raise ValueError("preallocated output has the wrong shape / dtype / device or is not contiguous")
    return ref_feat, poses, query_feat, Q, emb, sim, topv, topi
