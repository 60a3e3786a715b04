"""Host-side mirror of the reference's LDM-variant UNet, `UNetModelPose`
(src/model/u_net/ldm/adapt_openaimodel.py:14-158; configs/model/vae_cin_ldm.yaml), on top of the
C ABI in include/nope_b200.h (nope_ldm_*).

Same constructor keywords as the reference class; `load_state_dict` takes its 628 keys unchanged;
`__call__(x, pose)` is `UNetModelPose.forward`; `sweep` batches all pose hypotheses of a
reference latent and fuses the l2 score + top-k like `nope_b200.unet.UNet.sweep`.  All arithmetic
runs in libnope_b200.so.  The VAE encoder of this variant (diffusers AutoencoderKL,
src/model/encoder/AutoencoderKL.py:16-47) is nope_b200.vae.VAE_StableDiffusion (DESIGN.md section 16);
any object with `latent_dim` / `name` (and `encode_image` if images are to be encoded) may stand in.
"""
import ctypes as C

import torch

from . import _lib
from .search import coarse_to_fine_search, grid_search, refined_search
from .unet import SweepEngine


class UNetModelPose(SweepEngine):
    def __init__(self, injecting_condition_twice=False, pose_mlp_name="single_layer",
                 rot_representation_dim=6, encoder=None, image_size=32, in_channels=4,
                 model_channels=256, out_channels=4, num_res_blocks=2,
                 attention_resolutions=(4, 2, 1), dropout=0, channel_mult=(1, 2, 4),
                 num_head_channels=32, use_spatial_transformer=True, transformer_depth=1,
                 context_dim=512, device="cuda:0", chunk=256, precision="fp16", **kwargs):
        # the configuration the reference ships (vae_cin_ldm.yaml:2-31); everything else raises
        if injecting_condition_twice or pose_mlp_name != "single_layer":
            raise ValueError("only injecting_condition_twice=False / pose_mlp_name='single_layer'")
        if rot_representation_dim != 6 or tuple(channel_mult) != (1, 2, 4) or num_res_blocks != 2 \
                or sorted(attention_resolutions) != [1, 2, 4] or num_head_channels != 32 \
                or not use_spatial_transformer or transformer_depth != 1 or image_size != 32 \
                or in_channels != out_channels or dropout != 0:
            raise ValueError("unsupported UNetModelPose configuration (vae_cin_ldm.yaml values only)")
        for k in ("use_scale_shift_norm", "resblock_updown", "num_classes", "n_embed", "use_fp16"):
            if kwargs.get(k):
                raise ValueError(f"unsupported option {k}")
        self.encoder = encoder
        self.channels = in_channels if encoder is None else encoder.latent_dim
        self.name = "VAE" if encoder is None else encoder.name
        if self.channels != in_channels:
            raise ValueError("encoder.latent_dim must equal in_channels")
        self.model_channels = model_channels
        self.context_dim = context_dim
        self.rot_representation_dim = rot_representation_dim
        self.device = torch.device(device)
        # "fp16": fp16 weights (fast); "fp16_w2": exact weights as fp16 (hi, lo) K-segments, 2x the MMA work --
        # the mode that meets the 1e-3 embedding bar (the weight rounding alone is 0.6e-3 of the fp16 mode's 1.1e-3)
        if precision not in ("fp16", "fp16_w2"):
            raise ValueError("UNetModelPose precision: 'fp16' or 'fp16_w2'")
        self.precision = precision
        super().__init__("ldm", chunk, 2 * model_channels)

    def _create_args(self):
        if self.device.type != "cuda":
            raise _lib.NopeError("nope_b200.UNetModelPose needs a CUDA device (no CPU fallback)")
        return self.model_channels, self.context_dim, self.channels, 32, self.device.index or 0

    def _configure(self, lib, h):
        """chunk, precision and options: applied to every engine before its weights"""
        _lib.check(lib.nope_ldm_set_chunk(h, self._chunk))
        if self.precision == "fp16_w2":
            _lib.check(lib.nope_ldm_set_option(h, b"precision", 1))
        for k, v in self._options.items():
            _lib.check(lib.nope_ldm_set_option(h, k.encode(), v))

    def eval(self):
        return self

    def load_state_dict(self, state_dict, strict=True):
        """Reference UNetModelPose.state_dict() keys; `encoder.*` entries are skipped, except that a
        VAE_StableDiffusion encoder receives the `encoder.encoder.*` entries (AutoencoderKL keys).  May be called
        again: every call builds a fresh engine (the weights are packed at finalize)."""
        from .unet import encoder_entries
        from .vae import VAE_StableDiffusion
        self._native.build(self._create_args(),
                           ((k, v) for k, v in state_dict.items() if not k.startswith("encoder.")), self._configure)
        if isinstance(self.encoder, VAE_StableDiffusion):
            vae_sd = encoder_entries(state_dict, self.encoder)
            if vae_sd:
                self.encoder.load_state_dict(vae_sd, strict=strict)
        return self

    def profile_read(self):
        """-> {'gemm': {...}, 'attention': {...}} with ms / flops / launches since profile(True)."""
        ms, fl, n = (C.c_double * 2)(), (C.c_double * 2)(), (C.c_int64 * 2)()
        _lib.check(_lib.load().nope_ldm_profile_read(self._handle(), ms, fl, n))
        return {k: {"ms": ms[i], "flops": fl[i], "launches": n[i]} for i, k in enumerate(("gemm", "attention"))}

    def set_metric(self, metric="l2", threshold=0.2):
        """nope_b200.dist.ShardedSweep selects the score through this call; the LDM engine fuses the reference's
        "l2" score only (model.py:260-262)."""
        if metric != "l2":
            raise ValueError("UNetModelPose fuses the 'l2' similarity only")

    def sweep(self, ref_latent, poses, query_latent=None, want_emb=True, want_sim=None, k=0, idx_base=0,
              query_feat=None, out=None, query_visible=None):
        """ref_latent [B,C,32,32], poses [B,N,6] (+ query_latent) -> dict(emb, sim, topv, topi).
        query_latent [B,C,32,32] gives sim [B,N] / topv, topi [B,k]; [B,Q,C,32,32] (Q queries per reference, one
        sweep) gives [B,Q,N] / [B,Q,k].
        `query_feat` is an alias of `query_latent` and `out` may carry preallocated `sim` / `topv` / `topi`
        tensors (the keywords nope_b200.unet.UNet.sweep and nope_b200.dist.ShardedSweep use), so the pose grid
        shards across GPUs the same way.  query_visible: the rows' visible maps, as in UNet.sweep."""
        if query_feat is not None:
            query_latent = query_feat
        return super().sweep(ref_latent, poses, query_latent, want_emb, want_sim, k, idx_base, out, query_visible)

    def predict_pose(self, query_latent, ref_latent, all_relativeR, template_poses, k=5):
        """Latent-space form of nope_b200.model.PoseConditional.predict_pose for this UNet:
        -> (R [B,k,3,3], nearest_idx [B,k], similarity [B,N]).  As there, query_latent [B,Q,C,32,32] gives
        [B,Q,...] outputs, and query_latent [Q,C,32,32] with one reference (ref_latent [1,...], all_relativeR
        [1,N,6]) gives [Q,...]; both run one sweep.  k is clamped to N; template_poses [B,N,3,3] is read at row 0."""
        return grid_search(self, ref_latent, query_latent, all_relativeR, template_poses, k=k)

    def predict_pose_coarse_to_fine(self, query_latent, ref_latent, all_relativeR_levels, hierarchy,
                                    template_poses=None, k=5, keep=8):
        """Latent-space form of nope_b200.model.PoseConditional.predict_pose_coarse_to_fine for this UNet:
        -> (R | None, nearest_idx, similarity [..., N_L]) over the finest grid of `hierarchy`, -inf where the search
        scored nothing; the query forms of predict_pose."""
        return coarse_to_fine_search(self, ref_latent, query_latent, all_relativeR_levels, hierarchy, template_poses,
                                     k=k, keep=keep)

    def predict_pose_refined(self, query_latent, ref_latent, all_relativeR, refiner, k=5, keep=2):
        """Latent-space form of nope_b200.model.PoseConditional.predict_pose_refined for this UNet:
        -> (R [..., k, 3, 3] = D * template_poses[seed], seed_idx [..., k], score [..., k]); the query forms of
        predict_pose."""
        return refined_search(self, ref_latent, query_latent, all_relativeR, refiner, k=k, keep=keep)

    # ------------------------------------------------------------------ debug / parity hooks
    def run_block(self, name, x0, x1=None, poses=None, out_channels=None, out_side=None):
        """One module in isolation (fp32 NCHW in / out); see nope_ldm_run_block."""
        lib = _lib.load()
        dev = self.device
        x0 = x0.to(dev, torch.float32).contiguous()
        n, C0, S = x0.shape[0], x0.shape[1], x0.shape[2]
        C1 = 0
        if x1 is not None:
            x1 = x1.to(dev, torch.float32).contiguous()
            C1 = x1.shape[1]
        if poses is not None:
            poses = poses.to(dev, torch.float32).contiguous()
        out = torch.empty((n, out_channels, out_side, out_side), device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            _lib.check(lib.nope_ldm_run_block(self._handle(), name.encode(), _lib.ptr(x0), C0, _lib.ptr(x1), C1,
                                              S, n, _lib.ptr(poses), _lib.ptr(out), _lib.stream(dev)))
        return out


def mh_attention(qkv):
    """Multi-head self-attention core on qkv [n_img, n_tok, 3C] (CUDA fp32) -> [n_img, n_tok, C]."""
    lib = _lib.load()
    qkv = qkv.to(torch.float32).contiguous()
    n_img, n_tok, c3 = qkv.shape
    out = torch.empty((n_img, n_tok, c3 // 3), device=qkv.device, dtype=torch.float32)
    with torch.cuda.device(qkv.device):
        _lib.check(lib.nope_op_mh_attention(_lib.ptr(qkv), _lib.ptr(out), n_img, n_tok, c3 // 3,
                                            _lib.stream(qkv.device)))
    return out
