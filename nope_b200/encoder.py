"""Template encoder: image [B,3,256,256] -> latent [B,8,32,32].

Two backends behind the reference's `FeatureExtractor` surface:
  * "b200" (default on a CUDA device): the native engine in libnope_b200.so
    (`nope_encoder_*`, csrc/encoder.cuh) -- the wgmma convolution kernel with
    split-precision fp16 (hi, lo) operands, fp32-accurate (SURVEY.md section 8 row f1);
  * "torch": the PyTorch/cuDNN module below in fp32 with TF32 off (row a3; slower: cuDNN has
    no tensor-core path at fp32 accuracy).  Used for CPU tests and as a
    cross-check; never picked silently on a GPU.

Mirrors reference `FeatureExtractor` (src/model/encoder/template.py:24-53): ResNet-50
without max-pool and with layer4 at stride 1 (src/model/encoder/resnet.py:93-152, so the
total stride is 8), eval-mode BatchNorm, then ReLU -> 1x1(2048->256) -> ReLU -> 1x1(256->D).
Parameter names equal the reference's `backbone.*` / `projector.*` keys so its
state_dict loads unchanged; the duplicate `encoder.{0,1}.*` aliases the reference
registers (template.py:40) are accepted and ignored.

`precision` picks the native engine's arithmetic (DESIGN.md section 22): "split" (default) is the fp32-accurate
split precision above; "fp16" is the opt-in fast mode with single fp16 weights and stored activations and fp32
accumulation, one tensor-core product per tap instead of three.  "fp16" has no torch-backend or CPU path.
"""
import torch
from torch import nn
import torch.nn.functional as F

from . import _lib

# FeatureExtractor / VAE_StableDiffusion `precision` -> the engines' "precision" option
ENCODER_PRECISIONS = {"split": 0, "fp16": 1}


def check_precision(precision):
    """Returns the engine option value of an encoder `precision`; ValueError for anything else."""
    if not isinstance(precision, str) or precision not in ENCODER_PRECISIONS:
        raise ValueError(f"encoder precision must be one of {sorted(ENCODER_PRECISIONS)}, got {precision!r}")
    return ENCODER_PRECISIONS[precision]


def precision_option(kind, precision):
    """The build_engine `configure` step that sets the "precision" option of a `kind` engine ("encoder" or "vae"),
    or None for the default split precision (the engine's own default, so that mode makes no extra call)."""
    value = check_precision(precision)
    if value == 0:
        return None
    return lambda lib, h: _lib.check(getattr(lib, f"nope_{kind}_set_option")(h, b"precision", value))


def native_encode(kind, engine, device, image, D, name, A=None, pairs=None):
    """One encode by the native `kind` engine ("encoder" or "vae"), which `engine()` returns built, on `device`:
    images [B,3,256,256] -> D-channel latents [B,D,32,32] (nope_<kind>_encode); with A (checked), the latents of the
    A in-plane rotated copies of every image, [B,A,D,32,32] (_encode_inplane); with pairs = (image_idx [P], cossin
    [P, 2]), the latent of image image_idx[p] rotated by cossin[p], [P,D,32,32] (_encode_rotated).  Images of another
    shape raise NopeError naming the `name` encoder; malformed pairs raise ValueError."""
    if image.dim() != 4 or tuple(image.shape[1:]) != (3, 256, 256) or image.shape[0] < 1:
        raise _lib.NopeError(f"the {name} encoder is built for [B, 3, 256, 256] inputs, got {tuple(image.shape)}")
    x = image.to(device=device, dtype=torch.float32).contiguous()
    B = x.shape[0]
    fn, args, lead = "encode", (), (B,)
    if A is not None:
        from .inplane import _on_device, inplane_table
        fn, args, lead = "encode_inplane", (_lib.ptr(_on_device(inplane_table, A, device)), A), (B, A)
    elif pairs is not None:
        image_idx, cossin = pairs
        if image_idx.dim() != 1 or tuple(cossin.shape) != (image_idx.shape[0], 2) or image_idx.shape[0] < 1:
            raise ValueError(f"image_idx [P] and cossin [P, 2] with P >= 1 expected, got {tuple(image_idx.shape)} and "
                             f"{tuple(cossin.shape)}")
        idx = image_idx.to(device=device, dtype=torch.int32).contiguous()
        cs = cossin.to(device=device, dtype=torch.float32).contiguous()
        fn, args, lead = "encode_rotated", (_lib.ptr(idx), _lib.ptr(cs), idx.shape[0]), (idx.shape[0],)
    out = torch.empty(lead + (D, 32, 32), device=device, dtype=torch.float32)
    with torch.cuda.device(device):
        _lib.check(getattr(_lib.load(), f"nope_{kind}_{fn}")(engine(), _lib.ptr(x), B, *args, _lib.ptr(out),
                                                            _lib.stream(device)))
    return out


def native_run_block(kind, h, device, name, x, out_chw, want_pair=None):
    """One module `name` of the built native `kind` engine `h` on its own (nope_<kind>_run_block): x [n, C, H, H] ->
    out [n, *out_chw], fp32 NCHW.  want_pair None is the template encoder, whose call has no (hi, lo) output; else
    -> (out, pair), pair the hi + lo copy when want_pair, else None."""
    x = x.to(device=device, dtype=torch.float32).contiguous()
    out = torch.empty((x.shape[0],) + out_chw, device=device)
    pair = torch.empty_like(out) if want_pair else None
    outs = (_lib.ptr(out),) if want_pair is None else (_lib.ptr(out), _lib.ptr(pair))
    with torch.cuda.device(device):
        _lib.check(getattr(_lib.load(), f"nope_{kind}_run_block")(h, name.encode(), _lib.ptr(x), x.shape[1],
                                                                 x.shape[2], x.shape[0], *outs, out.numel(),
                                                                 _lib.stream(device)))
    return out if want_pair is None else (out, pair)


class _Bottleneck(nn.Module):
    # resnet.py:55-91
    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, stride=stride, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.downsample = downsample

    def forward(self, x):
        out = F.relu(self.bn1(self.conv1(x)))
        out = F.relu(self.bn2(self.conv2(out)))
        out = self.bn3(self.conv3(out))
        if self.downsample is not None:
            x = self.downsample(x)
        return F.relu(out + x)


class _Backbone(nn.Module):
    # resnet.py:93-152 with use_avg_pooling_and_fc=False (no max-pool, no avgpool/fc in forward)
    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 64, 7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.inplanes = 64
        self.layer1 = self._make_layer(64, 3, 1)
        self.layer2 = self._make_layer(128, 4, 2)
        self.layer3 = self._make_layer(256, 6, 2)
        self.layer4 = self._make_layer(512, 3, 1)
        self.fc = nn.Linear(2048, 1)   # present in the reference state_dict, unused

    def _make_layer(self, planes, blocks, stride):
        down = None
        if stride != 1 or self.inplanes != planes * 4:
            down = nn.Sequential(nn.Conv2d(self.inplanes, planes * 4, 1, stride=stride, bias=False),
                                 nn.BatchNorm2d(planes * 4))
        layers = [_Bottleneck(self.inplanes, planes, stride, down)]
        self.inplanes = planes * 4
        layers += [_Bottleneck(self.inplanes, planes) for _ in range(1, blocks)]
        return nn.Sequential(*layers)

    def forward(self, x):
        x = F.relu(self.bn1(self.conv1(x)))
        return self.layer4(self.layer3(self.layer2(self.layer1(x))))


def _encoder_block_out(name, D):
    """(C, H, W) of a native-engine module's output (FeatureExtractor.run_block); (1, 1, 1) for an unknown name,
    which the engine refuses."""
    if name == "stem":
        return (64, 128, 128)
    if name == "projector":
        return (D, 32, 32)
    for li, (planes, blocks, side) in enumerate([(64, 3, 128), (128, 4, 64), (256, 6, 32), (512, 3, 32)], start=1):
        if name in [f"backbone.layer{li}.{b}" for b in range(blocks)]:
            return (planes * 4, side, side)
    return (1, 1, 1)


class FeatureExtractor(nn.Module):
    """Same constructor/attributes as the reference (template.py:25-45)."""

    def __init__(self, descriptor_size=8, threshold=0.2, normalize=False, backend="auto", precision="split",
                 **kwargs):
        super().__init__()
        if backend not in ("auto", "b200", "torch"):
            raise ValueError("backend must be 'auto', 'b200' or 'torch'")
        self.backend = backend
        self._native = _lib.Engine("encoder")
        self._native_device = None
        check_precision(precision)
        if precision != "split" and backend == "torch":
            raise _lib.NopeError(f"precision={precision!r} is a mode of the native engine; the torch backend has "
                                 "none (no fallback)")
        self.precision = precision
        self.latent_dim = descriptor_size
        self.normalize = normalize
        self.threshold = threshold
        self.name = "template"
        self.backbone = _Backbone()
        self.projector = nn.Sequential(
            nn.ReLU(inplace=False), nn.Conv2d(2048, 256, 1, bias=False),
            nn.ReLU(inplace=False), nn.Conv2d(256, descriptor_size, 1, bias=False))
        self.eval()

    def load_state_dict(self, state_dict, strict=True):
        own = {k: v for k, v in state_dict.items() if not k.startswith("encoder.")}
        self._drop_engine()
        return super().load_state_dict(own, strict=strict)

    # ------------------------------------------------------------------ native engine
    @property
    def _h(self):
        """the native engine's handle, None while there is none"""
        return self._native.h

    def _drop_engine(self):
        self._native.destroy()

    def _engine(self, device):
        """Builds the native engine from this module's current parameters (once per device)."""
        if self._native.h is None or self._native_device != device:
            tensors = [(k, v) for k, v in self.state_dict().items()
                       if not (k.endswith("num_batches_tracked") or k.startswith("backbone.fc."))]
            self._native.build((self.latent_dim, device.index or 0), tensors,
                               precision_option("encoder", self.precision))
            self._native_device = device
        return self._native.h

    def _use_native(self, device):
        if self.backend == "torch":
            return False
        if device.type != "cuda":
            if self.backend == "b200":
                raise _lib.NopeError("backend='b200' needs a CUDA device (no CPU fallback)")
            if self.precision != "split":
                raise _lib.NopeError(f"precision={self.precision!r} needs the native engine on a CUDA device "
                                     "(no CPU fallback)")
            return False          # 'auto' on CPU tensors: the torch module (CPU tests only)
        return True

    @torch.no_grad()
    def encode_image(self, image, mode=None):
        """template.py:47-53.  fp32 with TF32 off by default, so the latent matches the
        reference's fp32 path; `mode` is accepted and ignored as in the reference."""
        p = next(self.parameters())
        if self._use_native(p.device):
            out = native_encode("encoder", lambda: self._engine(p.device), p.device, image, self.latent_dim, "native")
            return F.normalize(out, dim=1) if self.normalize else out
        image = image.to(device=p.device, dtype=p.dtype)
        prev = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = False
        try:
            feat = self.projector(self.backbone(image))
        finally:
            torch.backends.cudnn.allow_tf32 = prev
        if self.normalize:
            feat = F.normalize(feat, dim=1)
        return feat.float()

    @torch.no_grad()
    def run_block(self, name, x):
        """Debug / parity: one module of the native engine on its own (nope_encoder_run_block).  name "stem"
        (x = images [n, 3, 256, 256]), "backbone.layer<l>.<b>" or "projector"; x [n, C, H, H] (CUDA) -> the module's
        output, fp32 NCHW: hi + lo of its (hi, lo) pair, the projector's fp32 output.  n <= 32."""
        p = next(self.parameters())
        if not self._use_native(p.device):
            raise _lib.NopeError("run_block needs the native engine on a CUDA device")
        if x.dim() != 4:
            raise _lib.NopeError(f"run_block takes [n, C, H, H] inputs, got {tuple(x.shape)}")
        return native_run_block("encoder", self._engine(p.device), p.device, name, x,
                                _encoder_block_out(name, self.latent_dim))

    @torch.no_grad()
    def encode_image_inplane(self, image, A):
        """image [B,3,256,256] -> [B,A,D,32,32]: the latents of the A in-plane rotated copies of every image
        (nope_b200.inplane, DESIGN.md section 11), equal to encode_image of inplane.rotate_images(image, A) flattened
        to [B*A, ...], without forming that batch.  Native engine only: the torch backend raises NopeError."""
        from .inplane import check_angles
        A = check_angles(A)
        p = next(self.parameters())
        if not self._use_native(p.device):
            raise _lib.NopeError("encode_image_inplane needs the native engine on a CUDA device "
                                 "(no torch-backend path)")
        out = native_encode("encoder", lambda: self._engine(p.device), p.device, image, self.latent_dim, "native", A=A)
        return F.normalize(out, dim=2) if self.normalize else out

    @torch.no_grad()
    def encode_image_rotated(self, image, image_idx, cossin):
        """image [B,3,256,256], pairs image_idx [P] (int) and cossin [P, 2] (float32 (cos, sin)) -> [P,D,32,32]: the
        latent of image image_idx[p] rotated by cossin[p] (the section 11 image convention, DESIGN.md section 14),
        equal to encode_image of the materialised rotated pairs, without forming them.  An index outside [0, B)
        encodes an all -1 crop.  Native engine only: the torch backend raises NopeError."""
        p = next(self.parameters())
        if not self._use_native(p.device):
            raise _lib.NopeError("encode_image_rotated needs the native engine on a CUDA device "
                                 "(no torch-backend path)")
        out = native_encode("encoder", lambda: self._engine(p.device), p.device, image, self.latent_dim, "native",
                            pairs=(image_idx, cossin))
        return F.normalize(out, dim=1) if self.normalize else out
