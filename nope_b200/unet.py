"""Host-side mirror of the reference `UNet` (src/model/u_net/denoising_diffusion_pytorch/
u_net.py:27-198) on top of the C ABI in include/nope_b200.h.

Same constructor arguments and the attributes the task module reads (`.encoder`,
`.channels`, `.name`, `__call__(x, pose)`); `load_state_dict` takes the reference's keys
unchanged.  All arithmetic runs in libnope_b200.so; this file only moves pointers.
"""
import ctypes as C

import torch

from . import _lib

# precision option of the engine (include/nope_b200.h, nope_unet_set_option)
PRECISIONS = {"fp16": 0, "fp16_w2": 1, "parity": 2, "bf16": 3, "parity_fast": 4}


class _Incompatible:
    """return value of load_state_dict(strict=False), torch-style"""

    def __init__(self, missing, unexpected):
        self.missing_keys, self.unexpected_keys = missing, unexpected

    def __repr__(self):
        return f"<missing_keys={self.missing_keys}, unexpected_keys={self.unexpected_keys}>"


class UNet:
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
        self._chunk = chunk
        self._h = None
        self._finalized = False
        self._options = {}
        self._ws = None            # torch-owned workspace (uint8), handed to the engine
        self._ws_shape = (0, 0, 0)
        self._state = None         # last loaded UNet tensors (CPU fp32), kept for reload / partial load

    # ------------------------------------------------------------------ lifetime
    def _handle(self):
        if self._h is None:
            lib = _lib.load()
            if self.device.type != "cuda":
                raise _lib.NopeError("nope_b200.UNet needs a CUDA device (no CPU fallback)")
            h = C.c_void_p()
            _lib.check(lib.nope_unet_create(C.byref(h), self.u_net_dim, self.channels, 32,
                                            self.device.index or 0))
            self._h = h
            _lib.check(lib.nope_unet_set_chunk(h, self._chunk))
            _lib.check(lib.nope_unet_set_option(h, b"precision", PRECISIONS[self.precision]))
            for k, v in self._options.items():
                _lib.check(lib.nope_unet_set_option(h, k.encode(), int(v)))
        return self._h

    def _destroy(self):
        if self._h is not None:
            _lib.load().nope_unet_destroy(self._h)
            self._h = None
        self._finalized = False
        self._ws, self._ws_shape = None, (0, 0, 0)

    def __del__(self):
        try:
            self._destroy()
        except Exception:
            pass

    def to(self, device):
        if self._h is not None and torch.device(device) != self.device:
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
        lib = _lib.load()
        want = self.expected_shapes()
        enc_sd, unet_sd, unexpected = {}, {}, []
        for k, v in state_dict.items():
            if k.startswith("encoder."):
                kk = k[len("encoder."):]
                if kk.startswith("backbone.") or kk.startswith("projector."):
                    enc_sd[kk] = v
                continue      # the `encoder.encoder.*` aliases (template.py:40) repeat the same tensors
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
        if self._h is not None and self._finalized:
            self._destroy()       # weights are repacked at finalize: a reload builds a fresh engine
        h = self._handle()
        for k, t in merged.items():
            shape = (C.c_int64 * t.dim())(*t.shape)
            _lib.check(lib.nope_unet_load_tensor(h, k.encode(), C.c_void_p(t.data_ptr()), shape, t.dim()))
        if enc_sd:
            self.encoder.load_state_dict(enc_sd, strict=strict)
        _lib.check(lib.nope_unet_finalize(h))
        self._state = merged
        self._finalized = True
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

    def set_chunk(self, hyps):
        self._chunk = hyps
        if self._h is not None:
            _lib.check(_lib.load().nope_unet_set_chunk(self._h, hyps))

    def set_option(self, name, value):
        """'fuse_gn' (1: GroupNorm/SiLU/pose bias/residual in the conv epilogue, default)."""
        self._options[name] = int(value)
        if self._h is not None:
            _lib.check(_lib.load().nope_unet_set_option(self._h, name.encode(), int(value)))

    def set_metric(self, metric, threshold=0.2):
        """Similarity metric of the scoring fused onto the sweep: 'l2' (the reference's, model.py:254-266),
        'cosine' or 'cosine_occlusion' (extensions; include/nope_b200.h NOPE_METRIC_*)."""
        from .model import _METRICS
        _lib.check(_lib.load().nope_unet_set_metric(self._handle(), _METRICS[metric], float(threshold)))

    def set_conv_impl(self, impl):
        """'tcgen05_2cta' (clustered kernel with the fused epilogues, default), 'tcgen05' (single-CTA
        wgmma kernel) or 'simt' (debug twin); the names are kept from the first version of the engine."""
        _lib.check(_lib.load().nope_unet_set_conv_impl(
            self._handle(), {"tcgen05": 0, "simt": 1, "tcgen05_2cta": 2}[impl]))

    @property
    def last_launch_count(self):
        return int(_lib.load().nope_unet_last_launch_count(self._handle()))

    def profile(self, enable):
        _lib.check(_lib.load().nope_unet_profile(self._handle(), 1 if enable else 0))

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

    # ------------------------------------------------------------------ hot path
    def sweep(self, ref_feat, poses, query_feat=None, want_emb=True, want_sim=None, k=0,
              idx_base=0, out=None):
        """ref_feat [B,C,32,32], poses [B,N,6] (+ query_feat [B,C,32,32]) ->
        dict(emb [B,N,C,32,32] | None, sim [B,N] | None, topv/topi [B,k] | None).
        `out` may carry preallocated contiguous `sim` / `topv` / `topi` tensors to write into (the
        multi-GPU path points them into its all-gather record)."""
        if not self._finalized:
            raise _lib.NopeError("load_state_dict() must be called before the sweep")
        lib = _lib.load()
        dev = self.device
        ref_feat = ref_feat.to(dev, torch.float32).contiguous()
        poses = poses.to(dev, torch.float32).contiguous()
        B, N = poses.shape[0], poses.shape[1]
        assert ref_feat.shape == (B, self.channels, 32, 32), ref_feat.shape
        assert poses.shape[2] == self.rot_representation_dim
        if want_sim is None:
            want_sim = query_feat is not None
        if query_feat is not None:
            query_feat = query_feat.to(dev, torch.float32).contiguous()
            assert query_feat.shape == ref_feat.shape
        emb = torch.empty((B, N, self.channels, 32, 32), device=dev, dtype=torch.float32) \
            if want_emb else None
        out = out or {}
        sim = out.get("sim") if want_sim else None
        if want_sim and sim is None:
            sim = torch.empty((B, N), device=dev, dtype=torch.float32)
        topv, topi = (out.get("topv"), out.get("topi")) if k > 0 else (None, None)
        if k > 0 and topv is None:
            topv = torch.empty((B, k), device=dev, dtype=torch.float32)
            topi = torch.empty((B, k), device=dev, dtype=torch.int64)
        for t, shape, dt in ((sim, (B, N), torch.float32), (topv, (B, k), torch.float32), (topi, (B, k), torch.int64)):
            if t is not None:
                assert t.is_contiguous() and tuple(t.shape) == shape and t.dtype == dt and t.device == dev
        self.reserve(min(self._chunk, B * N), B, B * N if query_feat is not None else 0)
        stream = torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev):
            _lib.check(lib.nope_unet_sweep(self._handle(), _lib.ptr(ref_feat), _lib.ptr(poses), B, N,
                                           _lib.ptr(query_feat), _lib.ptr(emb), _lib.ptr(sim), k,
                                           _lib.ptr(topv), _lib.ptr(topi), idx_base,
                                           C.c_void_p(stream)))
        return {"emb": emb, "sim": sim, "topv": topv, "topi": topi}

    def __call__(self, x, pose):
        """UNet.forward(x [B,C,32,32], pose [B,6]) -> [B,C,32,32] (u_net.py:160-198)."""
        out = self.sweep(x, pose[:, None, :], want_emb=True)["emb"]
        return out[:, 0]

    forward = __call__

    def debug_tap(self, ref_feat, poses, tap):
        """Activation named `tap` (oracle tap names) for poses [N,6] of ONE reference."""
        lib = _lib.load()
        dev = self.device
        ref_feat = ref_feat.to(dev, torch.float32).contiguous()
        poses = poses.to(dev, torch.float32).contiguous()
        N = poses.shape[0]
        cap = N * 32 * 32 * 8 * self.u_net_dim
        out = torch.empty(cap, device=dev, dtype=torch.float32)
        c, s = C.c_int(), C.c_int()
        self.reserve(N, 1, 0)
        stream = torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev):
            _lib.check(lib.nope_unet_debug_tap(self._handle(), _lib.ptr(ref_feat), _lib.ptr(poses), N,
                                               tap.encode(), _lib.ptr(out), cap, C.byref(c),
                                               C.byref(s), C.c_void_p(stream)))
        return out[: N * c.value * s.value * s.value].view(N, c.value, s.value, s.value)
