"""Time the SD VAE encoder (nope_b200.vae, DESIGN.md section 16) in ONE process:
  engine      VAE_StableDiffusion.encode_image at B in --batches: ms per image, algorithmic TFLOP/s (the oracle's
              hooked count, 272.7 GFLOP per image) and executed TFLOP/s (three split-precision products per tensor-core
              convolution, conv_out's four channels padded to 64, the fp32 conv_in and attention core once);
  eager       the functional oracle (oracle/vae_oracle.py) on the same GPU at B = --eager-batch, fp32 with TF32 off
              and float64: the eager PyTorch baseline;
  ldm         PoseConditional (vae_cin_ldm.yaml) predict_pose from images against UNetModelPose.predict_pose from
              precomputed latents, --poses poses, Q query images of one reference.
    python tools/vae_time.py --out /tmp/vae.json
Device events around whole calls, warm-up of every shape; ms is the median over --reps repetitions with the min / max
beside it.  Prints the card name and power limit with the numbers.  Seeded weights.  A development aid, not the
bench."""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from nope_b200.poses import icosphere_object_rotations, synthetic_pose_batch
from nope_b200.synth_weights import make_ldm_state_dict, make_vae_state_dict
from nope_b200.vae import VAE_StableDiffusion, build_vae_model
from oracle import vae_oracle

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from multi_query_time import card, timed_ms          # noqa: E402


def flops():
    """(algorithmic, executed) FLOP per image"""
    c = vae_oracle.flops_per_image()
    alg = sum(c.values())
    conv_in = 2 * 256 * 256 * 128 * 27
    conv_out, quant = 2 * 1024 * 8 * 512 * 9, 2 * 1024 * 8 * 8
    conv_out_exec = 2 * 1024 * 64 * 512 * 9            # quant_conv folded in, 4 channels padded to one 64-wide tile
    tensor_core = c["conv"] - conv_in - conv_out - quant + conv_out_exec + c["linear"]
    return alg, 3 * tensor_core + conv_in + c["attention"]


def stats(xs):
    return {"ms": statistics.median(xs), "min": min(xs), "max": max(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 16, 64])
    ap.add_argument("--eager-batch", type=int, default=16)
    ap.add_argument("--poses", type=int, default=642)
    ap.add_argument("--queries", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vae_time.py needs a CUDA device")
    info = card()
    rows = []

    def emit(row):
        row.update(info)
        rows.append(row)
        print(json.dumps(row), flush=True)

    sd = make_vae_state_dict(seed=0)
    vae = VAE_StableDiffusion(device="cuda:0").load_state_dict(sd)
    g = torch.Generator().manual_seed(0)
    x = (torch.rand(max(args.batches + [args.eager_batch]), 3, 256, 256, generator=g) * 2 - 1).cuda()
    alg, exe = flops()
    for B in args.batches:
        vae.encode_image(x[:B])
        ms = [timed_ms(lambda: vae.encode_image(x[:B]), 2) for _ in range(args.reps)]
        st = stats(ms)
        emit({"case": "engine", "B": B, **st, "ms_per_image": st["ms"] / B,
              "algorithmic_tflops": alg * B / st["ms"] / 1e9, "executed_tflops": exe * B / st["ms"] / 1e9,
              "launches": vae.last_launch_count})

    Be = args.eager_batch
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for dt in (torch.float32, torch.float64):
            sdd = vae_oracle.canonical(sd, "cuda", dt)
            vae_oracle.encode(sdd, x[:Be], dtype=dt)
            ms = [timed_ms(lambda: vae_oracle.encode(sdd, x[:Be], dtype=dt), 1) for _ in range(max(2, args.reps // 2))]
            st = stats(ms)
            emit({"case": f"eager oracle {str(dt).split('.')[-1]} (TF32 off)", "B": Be, **st,
                  "ms_per_image": st["ms"] / Be, "algorithmic_tflops": alg * Be / st["ms"] / 1e9})
            del sdd
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    torch.cuda.empty_cache()

    model = build_vae_model("ldm", device="cuda:0")
    full = dict(make_ldm_state_dict(seed=0))
    full.update({"encoder.encoder." + k: v for k, v in sd.items()})
    model.load_state_dict(full).eval()
    u = model.u_net
    N = args.poses
    rel = synthetic_pose_batch(N, 1)[0].cuda()
    tp = torch.from_numpy(icosphere_object_rotations(2)).cuda() if N == 642 else None
    ref = x[:1]
    for Q in args.queries:
        q = x[1:1 + Q] if Q > 1 else x[1:2]
        zq, zr = u.encoder.encode_image(q), u.encoder.encode_image(ref)
        cases = {"images": lambda: model.predict_pose(q, ref, rel, tp, k=5),
                 "latents": lambda: u.predict_pose(zq, zr, rel, tp, k=5)}
        for f in cases.values():
            f()
        ms = {k: [] for k in cases}
        for _ in range(args.reps):
            for k, f in cases.items():
                ms[k].append(timed_ms(f, 1))
        for k in cases:
            emit({"case": f"ldm predict_pose from {k}", "Q": Q, "poses": N, **stats(ms[k])})
    if args.out:
        with open(args.out, "w") as f:
            f.writelines(json.dumps(r) + "\n" for r in rows)


if __name__ == "__main__":
    main()
