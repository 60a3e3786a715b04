"""Torch emulation of the encoders' single-fp16 mode (precision "fp16", DESIGN.md section 22) for the error budget.

Test tooling, never imported by the product.  It restates the template encoder (oracle/unet_oracle.encode_image) and
the SD VAE encoder (oracle/vae_oracle.encode) module by module, in the engines' form and with a rounding hook at every
tensor the engine stores as fp16 in that mode:

  template encoder  BatchNorm folded into the weights in float64, weights rounded to fp32 then fp16 (the stem's stay
                    fp32); every stored activation (stem, conv1 / conv2 / downsample / conv3 outputs, projector.1)
                    rounded to fp16; the bias, the residual add and the accumulation in `dtype`; the projector's
                    output stays unrounded
  VAE encoder       conv / linear weights rounded to fp16 (conv_in's stay fp32; conv_out + quant_conv folded in
                    float64 first); the fp16 copies the convolutions read -- the GroupNorm + SiLU output, the
                    attention output, the residual stream's copy for the identity add, the 1x1 shortcut and the
                    downsample -- rounded to fp16; the fp32 stream, the GroupNorm statistics, conv1's output, q / k /
                    v and the attention core unrounded

`rnd=False` with dtype float64 is the oracle restated (the self-check of tests/test_encoder_precision_cpu.py).
Each module function takes the module's input as the engines' run_block stage it (fp32 NCHW) and returns what
run_block returns in that mode: the encoder's fp16 output (the projector's fp32 output), the VAE's fp32 stream (the
latent for encoder.conv_out)."""
import torch
import torch.nn.functional as F

ENC_MODULES = (["stem"] + [f"backbone.layer{l}.{b}" for l, n in ((1, 3), (2, 4), (3, 6), (4, 3)) for b in range(n)]
               + ["projector"])
VAE_MODULES = (["encoder.conv_in"]
               + [m for i in range(4) for m in [f"encoder.down_blocks.{i}.resnets.{j}" for j in range(2)]
                  + ([f"encoder.down_blocks.{i}.downsamplers.0"] if i < 3 else [])]
               + ["encoder.mid_block.resnets.0", "encoder.mid_block.attentions.0", "encoder.mid_block.resnets.1",
                  "encoder.conv_out"])
_ATTN = "encoder.mid_block.attentions.0."


def _r16(t):
    """round to fp16 and back (through fp32 first, as the engines' hosts and kernels do)"""
    return t.float().half().to(t.dtype)


class _Rounding:
    def __init__(self, rnd, dtype):
        self.rnd, self.dtype = rnd, dtype

    def act(self, t):
        return _r16(t) if self.rnd else t

    def w(self, t64):
        """a float64 weight as the engine packs it: (float) then fp16 in this mode"""
        t = t64.to(torch.float32) if self.rnd else t64
        return (_r16(t) if self.rnd else t).to(self.dtype)

    def w32(self, t64):
        """a weight the engine keeps in fp32"""
        return (t64.to(torch.float32) if self.rnd else t64).to(self.dtype)


# ------------------------------------------------------------------ template encoder
def _fold(sd, wkey, bnkey):
    W = sd[wkey].double()
    if bnkey is None:
        return W, torch.zeros(W.shape[0], dtype=torch.float64)
    s = sd[bnkey + ".weight"].double() / torch.sqrt(sd[bnkey + ".running_var"].double() + 1e-5)
    return W * s[:, None, None, None], sd[bnkey + ".bias"].double() - sd[bnkey + ".running_mean"].double() * s


class TemplateEncoder:
    """The template encoder's fp16 mode (rnd=True) on a state_dict of `backbone.*` / `projector.*` keys."""

    def __init__(self, sd, rnd=True, dtype=torch.float32):
        self.R = _Rounding(rnd, dtype)
        self.dtype = dtype
        self.sd = {k: v.detach().cpu() for k, v in sd.items()}
        self._w = {}

    def _conv(self, name, wkey, bnkey, stem=False):
        if name not in self._w:
            W, b = _fold(self.sd, wkey, bnkey)
            self._w[name] = ((self.R.w32 if stem else self.R.w)(W), self.R.w32(b))
        return self._w[name]

    def module(self, name, x):
        x = x.to(self.dtype)
        R = self.R
        if name == "stem":
            w, b = self._conv("stem", "backbone.conv1.weight", "backbone.bn1", stem=True)
            return R.act(F.relu(F.conv2d(x, w, b, stride=2, padding=3)))
        x = R.act(x)                                            # run_block stages fp16
        if name == "projector":
            w1, _ = self._conv("p1", "projector.1.weight", None)
            w3, _ = self._conv("p3", "projector.3.weight", None)
            return F.conv2d(R.act(F.relu(F.conv2d(F.relu(x), w1))), w3)
        p = name
        stride = 2 if p.endswith(".0") and p.split(".")[1] in ("layer2", "layer3") else 1
        w1, b1 = self._conv(p + ".conv1", p + ".conv1.weight", p + ".bn1")
        w2, b2 = self._conv(p + ".conv2", p + ".conv2.weight", p + ".bn2")
        w3, b3 = self._conv(p + ".conv3", p + ".conv3.weight", p + ".bn3")
        a = R.act(F.relu(F.conv2d(x, w1, b1)))
        a = R.act(F.relu(F.conv2d(a, w2, b2, stride=stride, padding=1)))
        res = x
        if p + ".downsample.0.weight" in self.sd:
            wd, bd = self._conv(p + ".down", p + ".downsample.0.weight", p + ".downsample.1")
            res = R.act(F.conv2d(x, wd, bd, stride=stride))
        return R.act(F.relu(F.conv2d(a, w3, b3) + res))

    def encode(self, images, taps=None):
        h = images
        for m in ENC_MODULES:
            out = self.module(m, h)
            if taps is not None:
                taps[m] = (h, out)
            h = out
        return h


# ------------------------------------------------------------------ SD VAE encoder
class VaeEncoder:
    """The SD VAE encoder's fp16 mode (rnd=True) on an AutoencoderKL state_dict (either attention naming)."""

    def __init__(self, sd, rnd=True, dtype=torch.float32):
        from oracle import vae_oracle
        self.R = _Rounding(rnd, dtype)
        self.dtype = dtype
        self.sd = vae_oracle.canonical({k: v.detach().cpu() for k, v in sd.items()})   # float64
        self.scale = vae_oracle.SCALE

    def _p(self, k):
        return self.sd[k].to(self.dtype) if not self.R.rnd else self.sd[k].float().to(self.dtype)

    def _gn(self, x, p):
        # statistics of the fp32 tensor (float64 sums in the engine), applied in `dtype`
        return F.group_norm(x, 32, self._p(p + ".weight"), self._p(p + ".bias"), 1e-6)

    def _resnet(self, x, p):
        R, sd = self.R, self.sd
        h = R.act(F.silu(self._gn(x, p + ".norm1")))
        t = F.conv2d(h, R.w(sd[p + ".conv1.weight"]), self._p(p + ".conv1.bias"), padding=1)
        h = R.act(F.silu(self._gn(t, p + ".norm2")))
        if p + ".conv_shortcut.weight" in sd:
            b = R.w32(sd[p + ".conv2.bias"] + sd[p + ".conv_shortcut.bias"])
            return (F.conv2d(h, R.w(sd[p + ".conv2.weight"]), None, padding=1)
                    + F.conv2d(R.act(x), R.w(sd[p + ".conv_shortcut.weight"])) + b[:, None, None])
        return F.conv2d(h, R.w(sd[p + ".conv2.weight"]), self._p(p + ".conv2.bias"), padding=1) + R.act(x)

    def _attention(self, x):
        R, sd, a = self.R, self.sd, _ATTN
        B, C, H, W = x.shape
        t = R.act(self._gn(x, a + "group_norm")).reshape(B, C, H * W).transpose(1, 2)
        q, k, v = (F.linear(t, R.w(sd[a + n + ".weight"]), self._p(a + n + ".bias")) for n in ("query", "key", "value"))
        s = torch.matmul(q, k.transpose(1, 2)) * (1.0 / C ** 0.5)
        s = torch.exp(s - s.max(dim=-1, keepdim=True).values)
        o = R.act(torch.matmul(s / s.sum(dim=-1, keepdim=True), v))
        o = F.linear(o, R.w(sd[a + "proj_attn.weight"]), self._p(a + "proj_attn.bias"))
        return o.transpose(1, 2).reshape(B, C, H, W) + R.act(x)

    def _conv_out(self, x):
        R, sd = self.R, self.sd
        h = R.act(F.silu(self._gn(x, "encoder.conv_norm_out")))
        Q = sd["quant_conv.weight"][:4, :, 0, 0]
        Wf = torch.einsum("oj,jcyx->ocyx", Q, sd["encoder.conv_out.weight"]) * self.scale
        bf = (sd["quant_conv.bias"][:4] + Q @ sd["encoder.conv_out.bias"]) * self.scale
        return F.conv2d(h, R.w(Wf), R.w32(bf), padding=1)

    def module(self, name, x):
        x = x.to(self.dtype)
        sd, R = self.sd, self.R
        if name == "encoder.conv_in":
            return F.conv2d(x, R.w32(sd["encoder.conv_in.weight"]), self._p("encoder.conv_in.bias"), padding=1)
        if name == "encoder.conv_out":
            return self._conv_out(x)
        if name == _ATTN[:-1]:
            return self._attention(x)
        if name.endswith("downsamplers.0"):
            return F.conv2d(F.pad(R.act(x), (0, 1, 0, 1)), R.w(sd[name + ".conv.weight"]),
                            self._p(name + ".conv.bias"), stride=2)
        return self._resnet(x, name)

    def encode(self, images, taps=None):
        h = images
        for m in VAE_MODULES:
            out = self.module(m, h)
            if taps is not None:
                taps[m] = (h, out)
            h = out
        return h


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


def worst_image_rel_l2(out, ref):
    d = (out.double() - ref.double()).flatten(1).norm(dim=1)
    return float((d / ref.double().flatten(1).norm(dim=1)).max())


def predict(n_images=4, seed=70):
    """The error budget on the seeded weights: per-module worst-image rel-L2 of the fp16 mode fed the float64
    oracle's module inputs, and the end-to-end latent rel-L2, for both encoders -> dict."""
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from oracle import unet_oracle, vae_oracle, weights
    from nope_b200.synth_weights import make_vae_state_dict
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_vae_gpu import _crop_like, _uniform
    x = torch.cat([_uniform(seed, n_images - n_images // 2), _crop_like(seed, n_images // 2)])
    out = {}
    full = weights.make_full_state_dict(seed=0)
    enc_sd = {k[len("encoder."):]: v for k, v in full.items()
              if k.startswith("encoder.backbone.") or k.startswith("encoder.projector.")}
    for tag, emu, ref_fn, sd in (
            ("encoder", TemplateEncoder(enc_sd), lambda t, taps: unet_oracle.encode_image(
                {k: v.double() for k, v in enc_sd.items()}, t, taps=taps), enc_sd),
            ("vae", VaeEncoder(make_vae_state_dict(seed=0)),
             lambda t, taps: vae_oracle.encode(make_vae_state_dict(seed=0), t, taps=taps), None)):
        taps = {}
        ref = ref_fn(x.double(), taps)
        mods = ENC_MODULES if tag == "encoder" else VAE_MODULES
        per = {m: worst_image_rel_l2(emu.module(m, taps[m][0].float()), taps[m][1]) for m in mods}
        out[tag] = {"modules": per, "latent": rel_l2(emu.encode(x.float()), ref),
                    "latent_worst_image": worst_image_rel_l2(emu.encode(x.float()), ref)}
    return out


if __name__ == "__main__":
    import json
    torch.set_num_threads(8)
    print(json.dumps(predict(), indent=1))
