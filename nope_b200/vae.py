"""Stable Diffusion VAE: encoder image [B,3,256,256] in [-1, 1] -> latent [B,4,32,32], decoder back.

Mirrors reference `VAE_StableDiffusion` (src/model/encoder/AutoencoderKL.py:6-47), the encoder of the LDM
variant (configs/model/vae_cin_ldm.yaml) and of configs/model/vae_base.yaml: `encode_image` is
diffusers `AutoencoderKL.encode(x).latent_dist.mode() * 0.18215` for the Stable Diffusion v1 VAE
configuration (SD_V1_CONFIG), computed by the native engine in libnope_b200.so (`nope_vae_*`,
csrc/vae.cuh, DESIGN.md section 16): every convolution on the wgmma kernel with split-precision fp16
(hi, lo) operands, fp32-accurate.  `decode_latent` is diffusers `AutoencoderKL.decode(z / 0.18215).sample`
(AutoencoderKL.py:44-47), computed by a second engine (`nope_vae_decoder_*`, DESIGN.md section 17) that is
built on the first decode.  There is no CPU path; the KL distribution of `using_KL=True` and the training
loss are out of scope.

Weights use the diffusers AutoencoderKL state_dict layout.  The mid-block attention projections are
accepted under both of diffusers' namings (`query` / `key` / `value` / `proj_attn` and `to_q` / `to_k` /
`to_v` / `to_out.0`), in the decoder's mid block as in the encoder's.  The decoder's 140 `decoder.*` /
`post_quant_conv.*` tensors are optional: each one present is checked, and `decode_latent` is available once
all of them are.
"""
from collections import OrderedDict
import ctypes as C
import json
import os

import torch

from . import _lib

# the encoder-side fields of the Stable Diffusion v1 AutoencoderKL config.json (the only configuration the engine is
# built for), and diffusers' defaults for a field the file leaves out
SD_V1_CONFIG = {
    "in_channels": 3,
    "latent_channels": 4,
    "block_out_channels": [128, 256, 512, 512],
    "down_block_types": ["DownEncoderBlock2D"] * 4,
    "layers_per_block": 2,
    "norm_num_groups": 32,
    "act_fn": "silu",
    "double_z": True,
}
_CONFIG_DEFAULTS = {"in_channels": 3, "latent_channels": 4, "block_out_channels": [64],
                    "down_block_types": ["DownEncoderBlock2D"], "layers_per_block": 1, "norm_num_groups": 32,
                    "act_fn": "silu", "double_z": True}
_ATTN = "encoder.mid_block.attentions.0."
_ATTN_RENAME = {"to_q.": "query.", "to_k.": "key.", "to_v.": "value.", "to_out.0.": "proj_attn."}


def check_config(cfg):
    """Raises ValueError unless `cfg` (a parsed config.json) has the SD v1 encoder configuration.  Decoder-only
    fields (out_channels, up_block_types) and sample_size do not change the encoder and are not checked."""
    for k, want in SD_V1_CONFIG.items():
        got = cfg.get(k, _CONFIG_DEFAULTS[k])
        if isinstance(got, tuple):
            got = list(got)
        if got != want or type(got) is not type(want):
            raise ValueError(f"unsupported AutoencoderKL config: {k} = {got!r} (the engine is built for {want!r})")


def vae_param_shapes():
    """key -> shape of the 108 AutoencoderKL encoder tensors (0.14-era attention names) the engine loads."""
    s = OrderedDict()

    def conv(p, cout, cin, k):
        s[p + ".weight"] = (cout, cin, k, k)
        s[p + ".bias"] = (cout,)

    def norm(p, c):
        s[p + ".weight"] = (c,)
        s[p + ".bias"] = (c,)

    def resnet(p, cin, cout):
        norm(p + ".norm1", cin)
        conv(p + ".conv1", cout, cin, 3)
        norm(p + ".norm2", cout)
        conv(p + ".conv2", cout, cout, 3)
        if cin != cout:
            conv(p + ".conv_shortcut", cout, cin, 1)

    conv("encoder.conv_in", 128, 3, 3)
    cin = 128
    for i, c in enumerate(SD_V1_CONFIG["block_out_channels"]):
        for j in range(2):
            resnet(f"encoder.down_blocks.{i}.resnets.{j}", cin, c)
            cin = c
        if i < 3:
            conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", c, c, 3)
    resnet("encoder.mid_block.resnets.0", 512, 512)
    norm(_ATTN + "group_norm", 512)
    for n in ("query", "key", "value", "proj_attn"):
        s[_ATTN + n + ".weight"] = (512, 512)
        s[_ATTN + n + ".bias"] = (512,)
    resnet("encoder.mid_block.resnets.1", 512, 512)
    norm("encoder.conv_norm_out", 512)
    conv("encoder.conv_out", 8, 512, 3)
    conv("quant_conv", 8, 8, 1)
    return s


def map_state_dict(sd):
    """AutoencoderKL state_dict (either attention naming) -> {schema key: CPU fp32 tensor}.  Ignores `decoder.*`
    and `post_quant_conv.*`; raises KeyError for a missing or unknown key and ValueError for a wrong shape."""
    want = vae_param_shapes()
    out = {}
    for k, v in sd.items():
        if k.startswith("decoder.") or k.startswith("post_quant_conv."):
            continue
        kk = k
        if k.startswith(_ATTN):
            rest = k[len(_ATTN):]
            for a, b in _ATTN_RENAME.items():
                if rest.startswith(a):
                    kk = _ATTN + b + rest[len(a):]
        if kk not in want:
            raise KeyError(f"unexpected AutoencoderKL state_dict key: {k}")
        if kk in out:
            raise KeyError(f"AutoencoderKL state_dict has {kk} under both attention namings")
        if tuple(v.shape) != tuple(want[kk]):
            raise ValueError(f"size mismatch for {k}: checkpoint {tuple(v.shape)} vs model {tuple(want[kk])}")
        out[kk] = v.detach().to("cpu", torch.float32).contiguous()
    missing = [k for k in want if k not in out]
    if missing:
        raise KeyError(f"AutoencoderKL state_dict is missing {len(missing)} encoder keys: {missing[:5]}")
    return out


_DEC_ATTN = "decoder.mid_block.attentions.0."
# the decoder-side fields of the SD v1 config.json the decoder engine is built for, and diffusers' defaults
SD_V1_DECODER_CONFIG = {"out_channels": 3, "up_block_types": ["UpDecoderBlock2D"] * 4}
_DECODER_CONFIG_DEFAULTS = {"out_channels": 3, "up_block_types": ["UpDecoderBlock2D"]}


def check_decoder_config(cfg):
    """Raises ValueError unless `cfg` has the SD v1 decoder fields (out_channels 3, up_block_types
    4 x UpDecoderBlock2D); the other decoder dimensions are the encoder's fields, which check_config checks."""
    for k, want in SD_V1_DECODER_CONFIG.items():
        got = cfg.get(k, _DECODER_CONFIG_DEFAULTS[k])
        if isinstance(got, tuple):
            got = list(got)
        if got != want or type(got) is not type(want):
            raise ValueError(f"unsupported AutoencoderKL config: {k} = {got!r} (the decoder is built for {want!r})")


def vae_decoder_param_shapes():
    """key -> shape of the 140 AutoencoderKL decoder tensors (post_quant_conv and decoder.*, 0.14-era attention
    names) the decoder engine loads."""
    s = OrderedDict()

    def conv(p, cout, cin, k):
        s[p + ".weight"] = (cout, cin, k, k)
        s[p + ".bias"] = (cout,)

    def norm(p, c):
        s[p + ".weight"] = (c,)
        s[p + ".bias"] = (c,)

    def resnet(p, cin, cout):
        norm(p + ".norm1", cin)
        conv(p + ".conv1", cout, cin, 3)
        norm(p + ".norm2", cout)
        conv(p + ".conv2", cout, cout, 3)
        if cin != cout:
            conv(p + ".conv_shortcut", cout, cin, 1)

    conv("post_quant_conv", 4, 4, 1)
    conv("decoder.conv_in", 512, 4, 3)
    resnet("decoder.mid_block.resnets.0", 512, 512)
    norm(_DEC_ATTN + "group_norm", 512)
    for n in ("query", "key", "value", "proj_attn"):
        s[_DEC_ATTN + n + ".weight"] = (512, 512)
        s[_DEC_ATTN + n + ".bias"] = (512,)
    resnet("decoder.mid_block.resnets.1", 512, 512)
    cin = 512
    for i, c in enumerate(reversed(SD_V1_CONFIG["block_out_channels"])):
        for j in range(3):
            resnet(f"decoder.up_blocks.{i}.resnets.{j}", cin, c)
            cin = c
        if i < 3:
            conv(f"decoder.up_blocks.{i}.upsamplers.0.conv", c, c, 3)
    norm("decoder.conv_norm_out", 128)
    conv("decoder.conv_out", 3, 128, 3)
    return s


def map_decoder_state_dict(sd):
    """The `decoder.*` / `post_quant_conv.*` entries of an AutoencoderKL state_dict (either attention naming) ->
    {schema key: CPU fp32 tensor}; other entries are left to map_state_dict.  Raises KeyError for an unknown key and
    ValueError for a wrong shape; missing keys are allowed (a checkpoint without a decoder)."""
    want = vae_decoder_param_shapes()
    out = {}
    for k, v in sd.items():
        if not (k.startswith("decoder.") or k.startswith("post_quant_conv.")):
            continue
        kk = k
        if k.startswith(_DEC_ATTN):
            rest = k[len(_DEC_ATTN):]
            for a, b in _ATTN_RENAME.items():
                if rest.startswith(a):
                    kk = _DEC_ATTN + b + rest[len(a):]
        if kk not in want:
            raise KeyError(f"unexpected AutoencoderKL state_dict key: {k}")
        if kk in out:
            raise KeyError(f"AutoencoderKL state_dict has {kk} under both attention namings")
        if tuple(v.shape) != tuple(want[kk]):
            raise ValueError(f"size mismatch for {k}: checkpoint {tuple(v.shape)} vs model {tuple(want[kk])}")
        out[kk] = v.detach().to("cpu", torch.float32).contiguous()
    return OrderedDict((k, out[k]) for k in want if k in out)


def load_pretrained(path):
    """<path>/config.json (checked) and <path>/diffusion_pytorch_model.bin (or .safetensors) -> state_dict."""
    with open(os.path.join(path, "config.json")) as f:
        check_config(json.load(f))
    b = os.path.join(path, "diffusion_pytorch_model.bin")
    if os.path.exists(b):
        return torch.load(b, map_location="cpu", weights_only=True)
    st = os.path.join(path, "diffusion_pytorch_model.safetensors")
    if not os.path.exists(st):
        raise FileNotFoundError(f"{path} holds neither diffusion_pytorch_model.bin nor .safetensors")
    from safetensors.torch import load_file
    return load_file(st, device="cpu")


def _vae_block_out(name):
    """(C, H, W) of the output of an encoder or decoder engine module (VAE_StableDiffusion.run_block); (1, 1, 1) for
    an unknown name, which the engine refuses."""
    fixed = {"encoder.conv_in": (128, 256), "encoder.conv_out": (4, 32), "decoder.conv_in": (512, 32),
             "decoder.conv_out": (3, 256)}
    for p in ("encoder.mid_block.", "decoder.mid_block."):
        fixed.update({p + "resnets.0": (512, 32), p + "resnets.1": (512, 32), p + "attentions.0": (512, 32)})
    for i, c in enumerate((128, 256, 512, 512)):
        fixed.update({f"encoder.down_blocks.{i}.resnets.{j}": (c, 256 >> i) for j in range(2)})
        if i < 3:
            fixed[f"encoder.down_blocks.{i}.downsamplers.0"] = (c, 128 >> i)
    for i, c in enumerate((512, 512, 256, 128)):
        fixed.update({f"decoder.up_blocks.{i}.resnets.{j}": (c, 32 << i) for j in range(3)})
        if i < 3:
            fixed[f"decoder.up_blocks.{i}.upsamplers.0"] = (c, 64 << i)
    c, s = fixed.get(name, (1, 1))
    return (c, s, s)


class VAE_StableDiffusion:
    """Same constructor and attributes as the reference (AutoencoderKL.py:6-27)."""

    def __init__(self, pretrained_path=None, latent_dim=4, name="vae", using_KL=False, device="cuda:0", **kwargs):
        self._h = None
        self._dec_h = None
        if using_KL:
            raise ValueError("using_KL=True (the latent distribution of the training-only KL loss) is not supported")
        if latent_dim != 4:
            raise ValueError("latent_dim must be 4 (the SD v1 VAE's latent channels)")
        self.latent_dim = latent_dim
        self.name = name
        self.using_KL = using_KL
        self.encode_mode = "mode"
        self.device = torch.device(device)
        self._sd = None
        self._dec_sd = {}
        self._dec_config_error = None     # why the config.json's decoder fields cannot be decoded, if they cannot
        if pretrained_path is not None:
            self.load_state_dict(load_pretrained(pretrained_path))
            with open(os.path.join(pretrained_path, "config.json")) as f:
                try:
                    check_decoder_config(json.load(f))
                except ValueError as e:
                    self._dec_config_error = str(e)

    # ------------------------------------------------------------------ weights
    def load_state_dict(self, state_dict, strict=True):
        """AutoencoderKL keys (see map_state_dict and map_decoder_state_dict); the engines are rebuilt on the next
        encode / decode."""
        sd = map_state_dict(state_dict)
        dec = map_decoder_state_dict(state_dict)
        self._sd, self._dec_sd = sd, dec
        self._drop_engine()
        return self

    def state_dict(self):
        """The module's keys as in the reference (`encoder.` + AutoencoderKL key): the encoder tensors, and the
        decoder's when all of them are loaded."""
        if self._sd is None:
            return {}
        out = {"encoder." + k: v for k, v in self._sd.items()}
        if len(self._dec_sd) == len(vae_decoder_param_shapes()):
            out.update({"encoder." + k: v for k, v in self._dec_sd.items()})
        return out

    def _missing_decoder_keys(self):
        return [k for k in vae_decoder_param_shapes() if k not in self._dec_sd]

    @property
    def has_decoder(self):
        """True when all 140 decoder tensors are loaded and the config (if any) is the SD v1 decoder's."""
        return self._dec_config_error is None and not self._missing_decoder_keys()

    def to(self, device):
        device = torch.device(device)
        if device != self.device:
            self._drop_engine()
            self.device = device
        return self

    def eval(self):
        return self

    # ------------------------------------------------------------------ native engines
    def _drop_engine(self):
        """Destroys both engines (encoder and decoder)."""
        for attr, fn in (("_h", "nope_vae_destroy"), ("_dec_h", "nope_vae_decoder_destroy")):
            h = getattr(self, attr, None)
            if h is not None:
                try:
                    getattr(_lib.load(), fn)(h)
                except Exception:
                    pass
                setattr(self, attr, None)

    def __del__(self):
        self._drop_engine()

    def _engine(self):
        if self._h is not None:
            return self._h
        if self._sd is None:
            raise _lib.NopeError("VAE_StableDiffusion has no weights: pass pretrained_path or call load_state_dict")
        self._h = _lib.build_engine("vae", (self.device.index or 0,), self._sd.items())
        return self._h

    def _images(self, image):
        if self.device.type != "cuda":
            raise _lib.NopeError("VAE_StableDiffusion needs a CUDA device (no CPU path)")
        if not isinstance(image, torch.Tensor) or image.device.type != "cuda":
            raise _lib.NopeError("VAE_StableDiffusion encodes CUDA tensors only (no CPU path)")
        if image.dim() != 4 or tuple(image.shape[1:]) != (3, 256, 256) or image.shape[0] < 1:
            raise _lib.NopeError(f"the VAE encoder is built for [B, 3, 256, 256] inputs, got {tuple(image.shape)}")
        return image.to(device=self.device, dtype=torch.float32).contiguous()

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    @property
    def last_launch_count(self):
        return int(_lib.load().nope_vae_last_launch_count(self._h)) if self._h is not None else 0

    @torch.no_grad()
    def encode_image(self, image, mode=None):
        """AutoencoderKL.py:29-42 with mode "mode" (None means "mode"): the latent mean times 0.18215."""
        if mode not in (None, "mode"):
            raise NotImplementedError(f"encode_image mode {mode!r} (only 'mode' is supported)")
        x = self._images(image)
        out = torch.empty((x.shape[0], self.latent_dim, 32, 32), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().nope_vae_encode(self._engine(), _lib.ptr(x), x.shape[0], _lib.ptr(out),
                                                   self._stream()))
        return out

    @torch.no_grad()
    def encode_image_inplane(self, image, A):
        """image [B,3,256,256] -> [B,A,4,32,32]: the latents of the A in-plane rotated copies of every image
        (the FeatureExtractor.encode_image_inplane contract, DESIGN.md section 11), equal bit for bit to
        encode_image of inplane.rotate_images(image, A) flattened to [B*A, ...]."""
        from .inplane import _on_device, check_angles, inplane_table
        A = check_angles(A)
        x = self._images(image)
        out = torch.empty((x.shape[0], A, self.latent_dim, 32, 32), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().nope_vae_encode_inplane(
                self._engine(), _lib.ptr(x), x.shape[0], _lib.ptr(_on_device(inplane_table, A, self.device)), A,
                _lib.ptr(out), self._stream()))
        return out

    @torch.no_grad()
    def encode_image_rotated(self, image, image_idx, cossin):
        """image [B,3,256,256], pairs image_idx [P] and cossin [P, 2] -> [P,4,32,32] (the
        FeatureExtractor.encode_image_rotated contract, DESIGN.md section 14): the latent of image image_idx[p]
        rotated by cossin[p]; an index outside [0, B) encodes an all -1 crop."""
        if image_idx.dim() != 1 or tuple(cossin.shape) != (image_idx.shape[0], 2) or image_idx.shape[0] < 1:
            raise ValueError(f"image_idx [P] and cossin [P, 2] with P >= 1 expected, got {tuple(image_idx.shape)} and "
                             f"{tuple(cossin.shape)}")
        x = self._images(image)
        idx = image_idx.to(device=self.device, dtype=torch.int32).contiguous()
        cs = cossin.to(device=self.device, dtype=torch.float32).contiguous()
        P = idx.shape[0]
        out = torch.empty((P, self.latent_dim, 32, 32), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().nope_vae_encode_rotated(
                self._engine(), _lib.ptr(x), x.shape[0], _lib.ptr(idx), _lib.ptr(cs), P, _lib.ptr(out),
                self._stream()))
        return out

    @torch.no_grad()
    def run_block(self, name, x, want_pair=True):
        """Debug / parity: one module of the encoder engine, or of the decoder engine for a "decoder." name, on its
        own (nope_vae_run_block / nope_vae_decoder_run_block).  x [n, C, H, H] (CUDA) -> (out, pair): the fp32
        residual stream after the module and, when want_pair, hi + lo of its (hi, lo) copy, both fp32 NCHW.
        "encoder.conv_out" / "decoder.conv_out" give the latent / the image and no pair."""
        if not isinstance(x, torch.Tensor) or x.device.type != "cuda" or x.dim() != 4:
            raise _lib.NopeError("run_block takes [n, C, H, H] CUDA tensors")
        dec = name.startswith("decoder.")
        h = self._decoder() if dec else self._engine()
        x = x.to(device=self.device, dtype=torch.float32).contiguous()
        out = torch.empty((x.shape[0],) + _vae_block_out(name), device=self.device)
        pair = torch.empty_like(out) if want_pair else None
        fn = _lib.load().nope_vae_decoder_run_block if dec else _lib.load().nope_vae_run_block
        with torch.cuda.device(self.device):
            _lib.check(fn(h, name.encode(), _lib.ptr(x), x.shape[1], x.shape[2], x.shape[0], _lib.ptr(out),
                          _lib.ptr(pair), out.numel(), self._stream()))
        return out, pair

    # ------------------------------------------------------------------ decoder
    def _decoder(self):
        if self._dec_h is not None:
            return self._dec_h
        if self._dec_config_error is not None:
            raise ValueError(f"decode_latent: {self._dec_config_error}")
        missing = self._missing_decoder_keys()
        if missing:
            raise _lib.NopeError(f"decode_latent needs the AutoencoderKL decoder weights: {len(missing)} of the "
                                 f"{len(vae_decoder_param_shapes())} decoder tensors are missing, e.g. {missing[:5]}")
        self._dec_h = _lib.build_engine("vae_decoder", (self.device.index or 0,), self._dec_sd.items())
        return self._dec_h

    @property
    def last_decode_launch_count(self):
        return int(_lib.load().nope_vae_decoder_last_launch_count(self._dec_h)) if self._dec_h is not None else 0

    @torch.no_grad()
    def decode_latent(self, latent):
        """AutoencoderKL.py:44-47: latent [B,4,32,32] (CUDA) -> AutoencoderKL.decode(latent / 0.18215).sample,
        fp32 [B,3,256,256], not clamped.  The decoder engine is built on the first call."""
        if self.device.type != "cuda":
            raise _lib.NopeError("VAE_StableDiffusion needs a CUDA device (no CPU path)")
        if not isinstance(latent, torch.Tensor) or latent.device.type != "cuda":
            raise _lib.NopeError("VAE_StableDiffusion decodes CUDA tensors only (no CPU path)")
        if latent.dim() != 4 or tuple(latent.shape[1:]) != (self.latent_dim, 32, 32) or latent.shape[0] < 1:
            raise _lib.NopeError(f"the VAE decoder is built for [B, 4, 32, 32] latents, got {tuple(latent.shape)}")
        h = self._decoder()
        z = latent.to(device=self.device, dtype=torch.float32).contiguous()
        out = torch.empty((z.shape[0], 3, 256, 256), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().nope_vae_decoder_decode(h, _lib.ptr(z), z.shape[0], _lib.ptr(out),
                                                           self._stream()))
        return out


def build_vae_model(unet="ldm", vae_path=None, device="cuda:0", chunk=None, precision=None, vae_state_dict=None,
                    similarity_metric="l2"):
    """PoseConditional with the SD VAE encoder: unet="ldm" is configs/model/vae_cin_ldm.yaml (UNetModelPose),
    "base" is configs/model/vae_base.yaml (the default UNet at u_net_dim 192 on 4 latent channels).  The VAE
    weights come from `vae_path` (a diffusers directory) or `vae_state_dict`, or later through the
    PoseConditional's load_state_dict (a reference checkpoint's `u_net.encoder.encoder.*` entries)."""
    from .model import PoseConditional
    enc = VAE_StableDiffusion(pretrained_path=vae_path, latent_dim=4, name="VAE", device=device)
    if vae_state_dict is not None:
        enc.load_state_dict(vae_state_dict)
    if unet == "ldm":
        from .ldm import UNetModelPose
        net = UNetModelPose(encoder=enc, device=device, chunk=256 if chunk is None else chunk,
                            precision="fp16" if precision is None else precision)
    elif unet == "base":
        from .unet import UNet
        net = UNet(u_net_dim=192, rot_representation_dim=6, encoder=enc, pose_mlp_name="single_layer",
                   device=device, chunk=642 if chunk is None else chunk,
                   precision="fp16" if precision is None else precision)
    else:
        raise ValueError("unet must be 'ldm' (vae_cin_ldm.yaml) or 'base' (vae_base.yaml)")
    return PoseConditional(net, optim_config={"loss_type": "l1"},
                           testing_config={"similarity_metric": similarity_metric}, save_dir=None)
