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
"""
import ctypes as C

import torch
from torch import nn
import torch.nn.functional as F

from . import _lib


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


class FeatureExtractor(nn.Module):
    """Same constructor/attributes as the reference (template.py:25-45)."""

    def __init__(self, descriptor_size=8, threshold=0.2, normalize=False, backend="auto", **kwargs):
        super().__init__()
        if backend not in ("auto", "b200", "torch"):
            raise ValueError("backend must be 'auto', 'b200' or 'torch'")
        self.backend = backend
        self._h = None
        self._h_device = None
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
    def _drop_engine(self):
        if self._h is not None:
            try:
                _lib.load().nope_encoder_destroy(self._h)
            except Exception:
                pass
            self._h = None

    def __del__(self):
        self._drop_engine()

    def _engine(self, device):
        """Builds the native engine from this module's current parameters (once per device)."""
        if self._h is not None and self._h_device == device:
            return self._h
        self._drop_engine()
        lib = _lib.load()
        h = C.c_void_p()
        _lib.check(lib.nope_encoder_create(C.byref(h), self.latent_dim, device.index or 0))
        for k, v in self.state_dict().items():
            if k.endswith("num_batches_tracked") or k.startswith("backbone.fc."):
                continue
            t = v.detach().to("cpu", torch.float32).contiguous()
            shape = (C.c_int64 * t.dim())(*t.shape)
            _lib.check(lib.nope_encoder_load_tensor(h, k.encode(), C.c_void_p(t.data_ptr()), shape, t.dim()))
        _lib.check(lib.nope_encoder_finalize(h))
        self._h, self._h_device = h, device
        return h

    def _use_native(self, device):
        if self.backend == "torch":
            return False
        if device.type != "cuda":
            if self.backend == "b200":
                raise _lib.NopeError("backend='b200' needs a CUDA device (no CPU fallback)")
            return False          # 'auto' on CPU tensors: the torch module (CPU tests only)
        return True

    @torch.no_grad()
    def encode_image(self, image, mode=None):
        """template.py:47-53.  fp32 with TF32 off by default, so the latent matches the
        reference's fp32 path; `mode` is accepted and ignored as in the reference."""
        p = next(self.parameters())
        if self._use_native(p.device):
            if image.shape[-2:] != (256, 256):
                raise _lib.NopeError("the native encoder is built for 256x256 inputs")
            x = image.to(device=p.device, dtype=torch.float32).contiguous()
            out = torch.empty((x.shape[0], self.latent_dim, 32, 32), device=p.device, dtype=torch.float32)
            with torch.cuda.device(p.device):
                _lib.check(_lib.load().nope_encoder_encode(
                    self._engine(p.device), _lib.ptr(x), x.shape[0], _lib.ptr(out),
                    C.c_void_p(torch.cuda.current_stream(p.device).cuda_stream)))
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
