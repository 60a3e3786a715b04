"""Time the encoders' split and fp16 precision modes (DESIGN.md section 22) in ONE process, the modes alternated in
every repetition:
  encoder          the template encoder, ms per crop at B = 32 (one full chunk)
  vae              the SD VAE encoder, ms per crop at B = 16 (one full chunk)
  cudnn_fp16       eager PyTorch / cuDNN fp16, channels-last, of the same ResNet + projector at B = 32 (on-box baseline)
  inplane          predict_pose_inplane, fp16 UNet, level 2 (N = 642), A = 36, Q in --queries, with each encoder mode
  ldm_inplane      the LDM variant's predict_pose_inplane at Q = 1, A = 36, N = 642, with each VAE mode
Device events around whole calls after a warm-up of every shape; ms is the median over --reps repetitions with the
min / max beside it.  Seeded weights and inputs.  Prints one JSON line per case with the card name and power limit.
    python tools/encoder_precision_time.py --reps 3 --out /tmp/encoder_precision.json
A development aid, not the bench."""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from nope_b200 import synth_weights as weights
from nope_b200.encoder import FeatureExtractor
from nope_b200.model import build_model
from nope_b200.poses import icosphere_object_rotations, relative_rotation_6d
from nope_b200.vae import VAE_StableDiffusion, build_vae_model

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from multi_query_time import card, timed_ms          # noqa: E402

MODES = ("split", "fp16")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--angles", type=int, default=36)
    ap.add_argument("--reps", type=int, default=3, help="alternating repetitions of every case")
    ap.add_argument("--iters", type=int, default=5, help="calls per timed window of the encoder cases")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("encoder_precision_time.py needs a CUDA device")
    info = card()
    A = args.angles
    full = weights.make_full_state_dict(seed=0)
    enc_sd = {k[len("encoder."):]: v for k, v in full.items()
              if k.startswith("encoder.backbone.") or k.startswith("encoder.projector.")}
    vae_sd = weights.make_vae_state_dict(seed=0)
    model = build_model(device="cuda:0").load_state_dict(full).eval()
    encs = {}
    for m in MODES:
        fe = FeatureExtractor(descriptor_size=8, precision=m).cuda()
        fe.load_state_dict(enc_sd)
        encs[m] = fe
    vaes = {m: VAE_StableDiffusion(device="cuda:0", name="VAE", precision=m).load_state_dict(vae_sd) for m in MODES}
    ldm = build_vae_model("ldm", device="cuda:0")
    sd = dict(weights.make_ldm_state_dict(seed=0))
    sd.update({"encoder.encoder." + k: v for k, v in vae_sd.items()})
    ldm.load_state_dict(sd).eval()
    cudnn = FeatureExtractor(descriptor_size=8, backend="torch").cuda()
    cudnn.load_state_dict(enc_sd)
    cudnn = cudnn.half().to(memory_format=torch.channels_last)

    g = torch.Generator().manual_seed(0)
    img32 = (torch.rand(32, 3, 256, 256, generator=g) * 2 - 1).cuda()
    img16 = img32[:16].contiguous()
    img32_cl = img32.half().to(memory_format=torch.channels_last)
    ref = (torch.rand(1, 3, 256, 256, generator=g) * 2 - 1).cuda()
    qry = (torch.rand(max(args.queries), 3, 256, 256, generator=g) * 2 - 1).cuda()
    R2 = icosphere_object_rotations(2)
    rel = relative_rotation_6d(R2, R2[7])[None].cuda()

    def inplane(net, enc, Q):
        def fn():
            net.u_net.encoder = enc
            return net.predict_pose_inplane(qry[:Q], ref, rel, None, k=5, angles=A)
        return fn

    cases = {}
    for m in MODES:
        cases[("encoder", m, 32)] = (lambda e=encs[m]: e.encode_image(img32), args.iters, 32)
        cases[("vae", m, 16)] = (lambda v=vaes[m]: v.encode_image(img16), args.iters, 16)
        for Q in args.queries:
            cases[("inplane", m, Q)] = (inplane(model, encs[m], Q), 1, Q)
        cases[("ldm_inplane", m, 1)] = (inplane(ldm, vaes[m], 1), 1, 1)
    with torch.no_grad():
        cases[("cudnn_fp16", "fp16 channels-last", 32)] = (lambda: cudnn.projector(cudnn.backbone(img32_cl)),
                                                           args.iters, 32)
        for fn, _, _ in cases.values():
            fn()
            fn()
        samples = {key: [] for key in cases}
        for _ in range(args.reps):
            for m in MODES:                      # split, fp16, split, fp16, ... across the repetitions
                for key, (fn, iters, _) in cases.items():
                    if key[1] == m or (m == MODES[0] and key[0] == "cudnn_fp16"):
                        samples[key].append(timed_ms(fn, iters))
    model.u_net.encoder = encs["split"]
    ldm.u_net.encoder = vaes["split"]

    lines = []
    for (name, mode, n), ms in samples.items():
        med = statistics.median(ms)
        line = {"case": name, "mode": mode, "batch_or_Q": n, "ms_per_call": round(med, 3), "ms_min": round(min(ms), 3),
                "ms_max": round(max(ms), 3), "reps": len(ms)}
        if name in ("encoder", "vae", "cudnn_fp16"):
            line["ms_per_crop"] = round(med / n, 4)
        else:
            line.update({"A": A, "N": 642})
        lines.append({**line, **info})
    for name, n in [("encoder", 32), ("vae", 16)] + [("inplane", Q) for Q in args.queries] + [("ldm_inplane", 1)]:
        s, h = statistics.median(samples[(name, "split", n)]), statistics.median(samples[(name, "fp16", n)])
        lines.append({"case": name + " speed-up", "batch_or_Q": n, "split_ms": round(s, 3), "fp16_ms": round(h, 3),
                      "speedup": round(s / h, 3), **info})
    torch.cuda.synchronize()
    for line in lines:
        print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
