"""ctypes binding of include/nope_b200.h.  There is no CPU fallback: if the shared
library is missing, or a call fails, the product path raises."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_DEFAULT_LIB_PATH = os.path.join(_HERE, "lib", "libnope_b200.so")
LIB_PATH = _DEFAULT_LIB_PATH

c_f32p = C.c_void_p   # raw device / host pointers travel as integers
c_i64p = C.c_void_p

# symbol -> (restype, argtypes); mirrors include/nope_b200.h one to one
SIGNATURES = {
    "nope_last_error": (C.c_char_p, []),
    "nope_abi_version": (C.c_int, []),
    "nope_build_arch": (C.c_char_p, []),
    "nope_unet_set_chunk": (C.c_int, [C.c_void_p, C.c_int]),
    "nope_unet_sweep_multi": (C.c_int, [C.c_void_p, c_f32p, c_f32p, C.c_int, C.c_int, c_f32p, C.c_int, c_f32p,
                                        c_f32p, C.c_int, c_f32p, c_i64p, C.c_int64, C.c_void_p]),
    "nope_unet_last_launch_count": (C.c_int64, [C.c_void_p]),
    "nope_unet_profile": (C.c_int, [C.c_void_p, C.c_int]),
    "nope_unet_profile_read": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                         C.POINTER(C.c_double), C.POINTER(C.c_int64), C.POINTER(C.c_double)]),
    "nope_unet_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int]),
    "nope_unet_workspace_bytes": (C.c_int64, [C.c_void_p, C.c_int, C.c_int, C.c_int]),
    "nope_unet_set_workspace": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int]),
    "nope_op_conv_gn_fused": (C.c_int, [C.c_int, C.c_int, c_f32p, C.c_int, c_f32p, C.c_int, c_f32p, c_f32p,
                                        c_f32p, c_f32p, C.c_int, C.c_int, c_f32p, c_f32p, C.c_int, c_f32p,
                                        c_f32p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "nope_encoder_encode": (C.c_int, [C.c_void_p, c_f32p, C.c_int, c_f32p, C.c_void_p]),
    "nope_encoder_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int]),
    "nope_vae_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int]),
    "nope_encoder_last_launch_count": (C.c_int64, [C.c_void_p]),
    "nope_inplane_rotate": (C.c_int, [c_f32p, C.c_int, C.c_int, C.c_int, c_f32p, C.c_int, c_f32p, C.c_void_p]),
    "nope_encoder_encode_inplane": (C.c_int, [C.c_void_p, c_f32p, C.c_int, c_f32p, C.c_int, c_f32p, C.c_void_p]),
    "nope_inplane_rotate_pairs": (C.c_int, [c_f32p, C.c_int, C.c_int, C.c_int, C.c_void_p, c_f32p, C.c_int, c_f32p,
                                            C.c_void_p]),
    "nope_encoder_encode_rotated": (C.c_int, [C.c_void_p, c_f32p, C.c_int, C.c_void_p, c_f32p, C.c_int, c_f32p,
                                              C.c_void_p]),
    "nope_vae_encode": (C.c_int, [C.c_void_p, c_f32p, C.c_int, c_f32p, C.c_void_p]),
    "nope_vae_encode_inplane": (C.c_int, [C.c_void_p, c_f32p, C.c_int, c_f32p, C.c_int, c_f32p, C.c_void_p]),
    "nope_vae_encode_rotated": (C.c_int, [C.c_void_p, c_f32p, C.c_int, C.c_void_p, c_f32p, C.c_int, c_f32p,
                                          C.c_void_p]),
    "nope_vae_last_launch_count": (C.c_int64, [C.c_void_p]),
    "nope_vae_decoder_decode": (C.c_int, [C.c_void_p, c_f32p, C.c_int, c_f32p, C.c_void_p]),
    "nope_vae_decoder_last_launch_count": (C.c_int64, [C.c_void_p]),
    "nope_encoder_run_block": (C.c_int, [C.c_void_p, C.c_char_p, c_f32p, C.c_int, C.c_int, C.c_int, c_f32p,
                                         C.c_int64, C.c_void_p]),
    "nope_vae_run_block": (C.c_int, [C.c_void_p, C.c_char_p, c_f32p, C.c_int, C.c_int, C.c_int, c_f32p, c_f32p,
                                     C.c_int64, C.c_void_p]),
    "nope_vae_decoder_run_block": (C.c_int, [C.c_void_p, C.c_char_p, c_f32p, C.c_int, C.c_int, C.c_int, c_f32p,
                                             c_f32p, C.c_int64, C.c_void_p]),
    "nope_render_depth":(C.c_int, [c_f32p, C.c_int, C.c_void_p, C.c_int, c_f32p, C.c_int, C.c_float, C.c_float,
                                    C.c_float, C.c_float, C.c_float, C.c_int, C.c_int, c_f32p, C.c_void_p]),
    "nope_vsd_error": (C.c_int, [C.c_void_p, c_f32p, c_f32p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                 C.c_double, C.c_double, C.c_int, C.c_void_p, C.c_void_p]),
    "nope_vsd_error_taus": (C.c_int, [C.c_void_p, c_f32p, c_f32p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                      C.c_double, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "nope_fit_translation_occluded": (C.c_int, [c_f32p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                                C.c_int, C.c_float, C.c_int, c_f32p, C.c_void_p, C.c_void_p,
                                                C.c_void_p, C.c_void_p]),
    "nope_refine_depth": (C.c_int, [c_f32p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_void_p,
                                    C.c_int, C.c_float, c_f32p, C.c_void_p, C.c_void_p, C.c_void_p, c_i64p,
                                    C.c_void_p]),
    "nope_mask_sdf": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "nope_refine_contour_occluded": (C.c_int, [c_f32p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                               C.c_double, C.c_void_p, C.c_int, C.c_float, c_f32p, C.c_void_p,
                                               C.c_void_p, C.c_void_p, c_i64p, C.c_void_p]),
    "nope_pose_errors": (C.c_int, [c_f32p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "nope_crop_frames": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_int, C.c_int, c_f32p, C.c_void_p]),
    "nope_crop_camera": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "nope_crop_rotate": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "nope_track_seeds": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, c_f32p, C.c_void_p, c_f32p,
                                   C.c_void_p]),
    "nope_score_topk_multi": (C.c_int, [c_f32p, c_f32p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                        C.c_int, C.c_float, C.c_int, c_f32p, c_f32p, c_i64p, C.c_int64,
                                        C.c_void_p]),
    "nope_score_topk_grouped": (C.c_int, [c_f32p, c_f32p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                          C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, c_f32p, c_f32p,
                                          c_i64p, C.c_void_p]),
    "nope_unet_set_metric": (C.c_int, [C.c_void_p, C.c_int, C.c_float]),
    "nope_topk": (C.c_int, [c_f32p, C.c_int, C.c_int, C.c_int, c_f32p, c_i64p, C.c_int64, C.c_void_p]),
    "nope_distinct_topk": (C.c_int, [c_f32p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_double, c_i64p, c_f32p,
                                     C.c_void_p]),
    "nope_pose_cells_expand": (C.c_int, [c_i64p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, c_f32p, C.c_int,
                                         C.c_int, C.c_int, C.c_int, C.c_void_p, c_f32p, C.c_void_p]),
    "nope_pose_cells_rank": (C.c_int, [c_f32p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, c_f32p, c_f32p,
                                       c_i64p, C.c_void_p]),
    "nope_pose_refine_propose": (C.c_int, [c_f32p, C.c_void_p, C.c_int, C.c_int, c_f32p, C.c_int, C.c_int, C.c_int,
                                           c_f32p, c_f32p, C.c_void_p, c_f32p, c_f32p, C.c_void_p]),
    "nope_pose_refine_select": (C.c_int, [c_f32p, c_f32p, C.c_void_p, c_f32p, C.c_int, C.c_int, C.c_int, C.c_float,
                                          c_f32p, C.c_void_p, c_f32p, c_f32p, C.c_void_p]),
    "nope_pose_refine_inplane_propose": (C.c_int, [c_f32p, C.c_void_p, c_f32p, C.c_int, C.c_int, c_f32p, C.c_int,
                                                   C.c_int, C.c_int, c_f32p, C.c_float, C.c_float, c_f32p, C.c_void_p,
                                                   c_f32p, c_f32p, c_f32p, C.c_void_p]),
    "nope_pose_refine_inplane_select": (C.c_int, [c_f32p, c_f32p, C.c_void_p, c_f32p, c_f32p, C.c_int, C.c_int,
                                                  C.c_int, C.c_float, c_f32p, C.c_void_p, c_f32p, C.c_void_p, c_f32p,
                                                  c_f32p, C.c_void_p]),
    "nope_topk_pack_floats": (C.c_int64, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "nope_topk_merge": (C.c_int, [c_f32p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                  c_f32p, c_f32p, c_i64p, C.c_void_p]),
    "nope_op_conv": (C.c_int, [C.c_int, c_f32p, C.c_int, c_f32p, C.c_int, c_f32p, c_f32p,
                               c_f32p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "nope_op_conv_gn": (C.c_int, [C.c_int, c_f32p, C.c_int, c_f32p, C.c_int, c_f32p, c_f32p,
                                  c_f32p, c_f32p, C.c_int, C.c_int, c_f32p, C.c_int, C.c_int, C.c_int,
                                  C.c_int, C.c_void_p]),
    "nope_op_linear_attention": (C.c_int, [C.c_int, c_f32p, c_f32p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "nope_op_attention": (C.c_int, [c_f32p, c_f32p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "nope_op_upsample2x": (C.c_int, [c_f32p, c_f32p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "nope_ldm_set_chunk": (C.c_int, [C.c_void_p, C.c_int]),
    "nope_ldm_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int]),
    "nope_ldm_sweep_multi": (C.c_int, [C.c_void_p, c_f32p, c_f32p, C.c_int, C.c_int, c_f32p, C.c_int, c_f32p,
                                       c_f32p, C.c_int, c_f32p, c_i64p, C.c_int64, C.c_void_p]),
    "nope_ldm_last_launch_count": (C.c_int64, [C.c_void_p]),
    "nope_ldm_profile": (C.c_int, [C.c_void_p, C.c_int]),
    "nope_ldm_profile_read": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                        C.POINTER(C.c_int64)]),
    "nope_ldm_debug_tap": (C.c_int, [C.c_void_p, c_f32p, c_f32p, C.c_int, C.c_char_p, c_f32p,
                                     C.c_int64, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p]),
    "nope_ldm_run_block": (C.c_int, [C.c_void_p, C.c_char_p, c_f32p, C.c_int, c_f32p, C.c_int, C.c_int,
                                     C.c_int, c_f32p, c_f32p, C.c_void_p]),
    "nope_op_mh_attention": (C.c_int, [c_f32p, c_f32p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "nope_unet_debug_tap": (C.c_int, [C.c_void_p, c_f32p, c_f32p, C.c_int, C.c_char_p, c_f32p,
                                      C.c_int64, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p]),
    "nope_crop_hidden": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                   C.c_void_p]),
    "nope_latent_visibility": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, c_f32p, C.c_int, C.c_void_p,
                                         C.c_void_p]),
    "nope_unet_sweep_visible": (C.c_int, [C.c_void_p, c_f32p, c_f32p, C.c_int, C.c_int, c_f32p, C.c_int, C.c_void_p,
                                          c_f32p, c_f32p, C.c_int, c_f32p, c_i64p, C.c_int64, C.c_void_p]),
    "nope_ldm_sweep_visible": (C.c_int, [C.c_void_p, c_f32p, c_f32p, C.c_int, C.c_int, c_f32p, C.c_int, C.c_void_p,
                                         c_f32p, c_f32p, C.c_int, c_f32p, c_i64p, C.c_int64, C.c_void_p]),
    "nope_score_topk_visible": (C.c_int, [c_f32p, c_f32p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                          C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_float, C.c_int,
                                          c_f32p, c_f32p, c_i64p, C.c_void_p]),
}

# the lifecycle entries of the five weight-holding engines: kind -> nope_<kind>_create's arguments after the out handle
ENGINE_CREATE_ARGS = {"unet": 4, "encoder": 2, "vae": 1, "vae_decoder": 1, "ldm": 5}
for _kind, _n in ENGINE_CREATE_ARGS.items():
    SIGNATURES.update({
        f"nope_{_kind}_create": (C.c_int, [C.POINTER(C.c_void_p)] + [C.c_int] * _n),
        f"nope_{_kind}_destroy": (None, [C.c_void_p]),
        f"nope_{_kind}_load_tensor": (C.c_int, [C.c_void_p, C.c_char_p, c_f32p, C.POINTER(C.c_int64), C.c_int]),
        f"nope_{_kind}_finalize": (C.c_int, [C.c_void_p]),
    })

EXPECTED_ABI = 3     # include/nope_b200.h "ABI version"; a stale build with other signatures must not bind
MAX_TOPK = 64        # the most entries a ranking call selects per row (k, keep): mirrors kMaxTopK in csrc/rank.cuh

_lib = None


class NopeError(RuntimeError):
    pass


def load():
    """Load libnope_b200.so (raises if it has not been built)."""
    global _lib
    if _lib is not None:
        return _lib
    if LIB_PATH == _DEFAULT_LIB_PATH and not os.environ.get("NOPE_NO_AUTOBUILD"):
        # the library is built in-tree by `python -m nope_b200.build` / __graft_entry__.build();
        # on a fresh checkout, or when a source file is newer than the binary, compile it now
        # (nvcc, sm_90a) -- still the CUDA path, never a fallback.  A box without nvcc keeps the
        # shipped binary (its ABI version is checked below).
        from . import build as _build
        if not os.path.exists(LIB_PATH) or (_build.is_stale() and _build.have_nvcc()):
            try:
                _build.build()
            except Exception as exc:
                if not os.path.exists(LIB_PATH):
                    raise NopeError(f"{LIB_PATH} is missing and building it failed: {exc}") from exc
    if not os.path.exists(LIB_PATH):
        raise NopeError(
            f"{LIB_PATH} is missing: build it with `python -m nope_b200.build` "
            "(nope_b200 has no CPU or PyTorch fallback)")
    lib = C.CDLL(LIB_PATH)
    lib.nope_abi_version.restype = C.c_int
    abi = lib.nope_abi_version()
    if abi != EXPECTED_ABI:
        raise NopeError(f"{LIB_PATH} has ABI version {abi}, this package binds version {EXPECTED_ABI}: "
                        "rebuild with `python -m nope_b200.build --force`")
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)      # AttributeError if the export is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise NopeError(load().nope_last_error().decode("utf-8", "replace"))


def ptr(t):
    """Device/host pointer of a torch tensor (None -> NULL)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream(device):
    """The current CUDA stream of `device`, as the last argument of every launching entry point takes it."""
    import torch
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def build_engine(kind, create_args, tensors, configure=None):
    """Builds a `kind` engine ("unet", "encoder", "vae", "vae_decoder" or "ldm"): nope_<kind>_create(&h,
    *create_args), then configure(lib, h) (options that must precede the weights), then every (key, tensor) of
    `tensors` staged as contiguous CPU fp32, then nope_<kind>_finalize.  tensors None stops before the weights: the
    engine is weightless and not finalized.  Returns the handle; if any step raises, the engine is destroyed first."""
    import torch
    lib = load()
    h = C.c_void_p()
    check(getattr(lib, f"nope_{kind}_create")(C.byref(h), *create_args))
    try:
        if configure is not None:
            configure(lib, h)
        if tensors is not None:
            load_tensor = getattr(lib, f"nope_{kind}_load_tensor")
            for k, v in tensors:
                t = v.detach().to("cpu", torch.float32).contiguous()
                shape = (C.c_int64 * t.dim())(*t.shape)
                check(load_tensor(h, k.encode(), C.c_void_p(t.data_ptr()), shape, t.dim()))
            check(getattr(lib, f"nope_{kind}_finalize")(h))
    except BaseException:
        getattr(lib, f"nope_{kind}_destroy")(h)
        raise
    return h


class Engine:
    """Owns one nope_<kind>_* handle `h` (None while there is none).  `handle` creates it weightless and configured,
    `build` builds it with weights (destroying the previous one first), `destroy` releases it; a handle a build
    leaves half made is destroyed by build_engine, so `h` is either None or a whole engine."""

    def __init__(self, kind):
        self.kind, self.h, self.finalized = kind, None, False

    def handle(self, create_args, configure=None):
        """The handle; a weightless one, configured, if there is none yet."""
        if self.h is None:
            self.h = build_engine(self.kind, create_args, None, configure)
        return self.h

    def build(self, create_args, tensors, configure=None):
        self.destroy()
        self.h = build_engine(self.kind, create_args, tensors, configure)
        self.finalized = True
        return self.h

    def destroy(self):
        h, self.h, self.finalized = self.h, None, False
        if h is not None:
            getattr(load(), f"nope_{self.kind}_destroy")(h)

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass

    def call(self, name, *args):
        """nope_<kind>_<name>(h, *args), raising NopeError if it fails."""
        check(getattr(load(), f"nope_{self.kind}_{name}")(self.h, *args))

    def launch_count(self):
        """Kernels the handle's last call launched; 0 without a handle."""
        return 0 if self.h is None else int(getattr(load(), f"nope_{self.kind}_last_launch_count")(self.h))
