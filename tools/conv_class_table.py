"""Per-class convolution table from a NOPE_PROF_DUMP file, e.g.
    NOPE_PROF_DUMP=/tmp/prof.csv python tools/time_sweep.py fp16 --profile
    python tools/conv_class_table.py /tmp/prof.csv
The dump holds one block per profiled sweep (each opens with a `# launch,...` header line); every block is one
pass.  Per class and pass: ms, algorithmic TFLOP/s (algorithmic FLOPs over CUDA-event time) and the K-steps of
64 channels each tile walks; the table gives the range over the passes.  Classes: 3x3 convolutions by
resolution, the to_qkv 1x1 (the launch right before to_out, the only 1x1 with K = 128), every other 1x1,
the unshuffle 1x1 and the folded upsample convolutions."""
import argparse
import sys

MODES = {0: "3x3", 1: "1x1", 2: "unshuffle 1x1", 3: "folded upsample 3x3"}
HEADS_HIDDEN = 128      # to_out's K (4 heads x 32): no other convolution of the UNet has 128 input channels


def read_passes(path):
    passes, cur = [], None
    with open(path) as f:
        for line in f:
            line = line.strip()
            if not line:
                continue
            if line.startswith("#"):
                cur = []
                passes.append(cur)
                continue
            i, ms, ex, alg, res, mode, cout, k = line.split(",")
            cur.append(dict(ms=float(ms), ex=float(ex), alg=float(alg), res=int(res), mode=int(mode),
                            cout=int(cout), k=int(k)))
    return [p for p in passes if p]


def classify(launches):
    names = []
    for j, L in enumerate(launches):
        nxt = launches[j + 1] if j + 1 < len(launches) else None
        if L["mode"] == 0:
            names.append(f"3x3 at {L['res']}^2")
        elif L["mode"] == 1 and L["k"] == HEADS_HIDDEN:
            names.append("1x1 to_out")
        elif L["mode"] == 1 and nxt is not None and nxt["mode"] == 1 and nxt["k"] == HEADS_HIDDEN:
            names.append("1x1 to_qkv")
        elif L["mode"] == 1:
            names.append("1x1 (other)")
        else:
            names.append(MODES[L["mode"]])
    return names


def ksteps(L):
    # executed K-steps per tile: the split-precision modes run 2x / 3x the fp16 mode's K loop
    return round(L["ex"] / L["alg"] * L["k"] / 64) if L["alg"] > 0 else 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("dump")
    ap.add_argument("--hyps", type=int, default=0, help="hypotheses per profiled sweep: adds a GFLOP/hyp column")
    args = ap.parse_args()
    passes = read_passes(args.dump)
    if not passes:
        sys.exit(f"{args.dump}: no profiled pass")
    order, stats = [], {}
    for launches in passes:
        per = {}
        for name, L in zip(classify(launches), launches):
            d = per.setdefault(name, dict(ms=0.0, alg=0.0, n=0, ks=[]))
            d["ms"] += L["ms"]
            d["alg"] += L["alg"]
            d["n"] += 1
            d["ks"].append(ksteps(L))
            if name not in order:
                order.append(name)
        for name, d in per.items():
            stats.setdefault(name, []).append(d)
    key = {n: (0, -int(n.split()[2].split("^")[0])) if n.startswith("3x3 at") else (1, n) for n in order}
    order.sort(key=lambda n: key[n])
    hdr = ["class", "launches", "GFLOP/step"] + (["GFLOP/hyp"] if args.hyps else []) + \
          ["ms/step", "TFLOP/s", "K-steps per tile"]
    rows = []
    tot_ms = [0.0] * len(passes)
    tot_alg = 0.0
    for n in order:
        ds = stats[n]
        ms = [d["ms"] for d in ds]
        tf = [d["alg"] / d["ms"] for d in ds if d["ms"] > 0]      # GFLOP / ms = TFLOP/s
        ks = ds[0]["ks"]
        for i, d in enumerate(ds):
            tot_ms[i] += d["ms"]
        tot_alg += ds[0]["alg"]
        r = [n, str(ds[0]["n"]), f"{ds[0]['alg']:.1f}"]
        if args.hyps:
            r.append(f"{ds[0]['alg'] / args.hyps:.3f}")
        r += [f"{min(ms):.2f}-{max(ms):.2f}", f"{min(tf):.0f}-{max(tf):.0f}", f"{min(ks)}-{max(ks)}"]
        rows.append(r)
    r = ["all", str(sum(stats[n][0]["n"] for n in order)), f"{tot_alg:.1f}"]
    if args.hyps:
        r.append(f"{tot_alg / args.hyps:.3f}")
    r += [f"{min(tot_ms):.2f}-{max(tot_ms):.2f}", f"{tot_alg / max(tot_ms):.0f}-{tot_alg / min(tot_ms):.0f}", ""]
    rows.append(r)
    print(f"{len(passes)} pass(es) from {args.dump}")
    print("| " + " | ".join(hdr) + " |")
    print("|" + "---|" * len(hdr))
    for r in rows:
        print("| " + " | ".join(r) + " |")


if __name__ == "__main__":
    main()
