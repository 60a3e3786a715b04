"""Time the SD VAE decoder (VAE_StableDiffusion.decode_latent, DESIGN.md section 17) in ONE process:
  engine      decode_latent at B in --batches: ms per image, algorithmic TFLOP/s (the oracle's hooked count, 622.2
              GFLOP per image) and executed TFLOP/s (three split-precision products per tensor-core convolution, the
              upsample convolutions folded to 2x2, conv_out's three channels padded to 64, the fp32 conv_in and
              attention core once);
  eager       the functional oracle (tests/vae_decoder_oracle.py) on the same GPU at B = --eager-batch, fp32 with TF32
              off and float64: the eager PyTorch baseline;
  templates   PoseConditional (vae_cin_ldm.yaml) generate_templates over --poses poses of one reference, with the
              decoder's weights loaded (latents and images) and without them (latents only).
    python tools/vae_decode_time.py --out /tmp/vae_decode.json
Device events around whole calls, warm-up of every shape; ms is the median over --reps repetitions with the min / max
beside it.  Prints the card name and power limit with the numbers.  Seeded weights.  A development aid, not the
bench."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(1, os.path.join(ROOT, "tests"))
import torch

from nope_b200.poses import synthetic_pose_batch
from nope_b200.synth_weights import make_ldm_state_dict, make_vae_state_dict
from nope_b200.vae import VAE_StableDiffusion, build_vae_model
import vae_decoder_oracle as D                      # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from multi_query_time import card, timed_ms          # noqa: E402


def flops():
    """(algorithmic, executed) FLOP per image"""
    c = D.flops_per_image()
    alg = sum(c.values())
    conv_in, post_quant = 2 * 32 * 32 * 512 * 4 * 9, 2 * 32 * 32 * 4 * 4
    conv_out, conv_out_exec = 2 * 65536 * 3 * 128 * 9, 2 * 65536 * 64 * 128 * 9    # 3 channels padded to one tile
    ups = 2 * 9 * (64 * 64 * 512 * 512 + 128 * 128 * 512 * 512 + 256 * 256 * 256 * 256)
    tensor_core = c["conv"] - conv_in - post_quant - conv_out - ups + ups * 4 // 9 + conv_out_exec + c["linear"]
    return alg, 3 * tensor_core + conv_in + post_quant + c["attention"]


def stats(xs):
    return {"ms": statistics.median(xs), "min": min(xs), "max": max(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8, 16, 64])
    ap.add_argument("--eager-batch", type=int, default=8)
    ap.add_argument("--poses", type=int, default=642)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vae_decode_time.py needs a CUDA device")
    info = card()
    rows = []

    def emit(row):
        row.update(info)
        rows.append(row)
        print(json.dumps(row), flush=True)

    sd = make_vae_state_dict(seed=0, decoder=True)
    vae = VAE_StableDiffusion(device="cuda:0").load_state_dict(sd)
    g = torch.Generator().manual_seed(0)
    x = (torch.rand(16, 3, 256, 256, generator=g) * 2 - 1).cuda()
    z16 = vae.encode_image(x)
    z = z16.repeat((max(args.batches + [args.eager_batch]) + 15) // 16, 1, 1, 1)
    alg, exe = flops()
    emit({"case": "flop per image", "algorithmic_gflop": alg / 1e9, "executed_gflop": exe / 1e9})
    for B in args.batches:
        vae.decode_latent(z[:B])
        ms = [timed_ms(lambda: vae.decode_latent(z[:B]), 2) for _ in range(args.reps)]
        st = stats(ms)
        emit({"case": "engine", "B": B, **st, "ms_per_image": st["ms"] / B,
              "algorithmic_tflops": alg * B / st["ms"] / 1e9, "executed_tflops": exe * B / st["ms"] / 1e9,
              "launches": vae.last_decode_launch_count})

    Be = args.eager_batch
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for dt in (torch.float32, torch.float64):
            sdd = D.canonical(sd, "cuda", dt)
            D.decode(sdd, z[:Be], dtype=dt)
            ms = [timed_ms(lambda: D.decode(sdd, z[:Be], dtype=dt), 1) for _ in range(max(2, args.reps // 2))]
            st = stats(ms)
            emit({"case": f"eager oracle {str(dt).split('.')[-1]} (TF32 off)", "B": Be, **st,
                  "ms_per_image": st["ms"] / Be, "algorithmic_tflops": alg * Be / st["ms"] / 1e9})
            del sdd
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    del vae
    torch.cuda.empty_cache()

    N = args.poses
    rel = synthetic_pose_batch(N, 1)[0].cuda()
    ref = x[:1]
    enc_only = {k: v for k, v in sd.items() if not (k.startswith("decoder.") or k.startswith("post_quant_conv."))}
    for name, vsd in (("with decoder", sd), ("without decoder", enc_only)):
        model = build_vae_model("ldm", device="cuda:0")
        full = dict(make_ldm_state_dict(seed=0))
        full.update({"encoder.encoder." + k: v for k, v in vsd.items()})
        model.load_state_dict(full).eval()
        model.generate_templates(ref, rel)
        ms = [timed_ms(lambda: model.generate_templates(ref, rel), 1) for _ in range(args.reps)]
        emit({"case": f"ldm generate_templates {name}", "poses": N, **stats(ms)})
        del model
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            f.writelines(json.dumps(r) + "\n" for r in rows)


if __name__ == "__main__":
    main()
