"""GPU: the lock-step GroupNorm-fused epilogue (EPI 3, chosen once per process by NOPE_GN_EPI=3) at every tile
width it is built for -- BN 192 (three math warpgroups, the third one epilogue only), 128 and 64 -- run through the
sweep's fused layer (ops.conv_gn_fused) in a child process, against the reference and tolerance of the role-split
epilogue (test_fused_gpu).  The last case of each width runs at least three tiles per CTA (asserted from the shape)
over 5 N-tiles.  5 does not divide the 66 clusters, so a CTA's tiles fall on different N-tiles and the channel-parameter
cache must reload bias / gamma / beta between them; the staging hand-over between a CTA's tiles runs too.  Errors are
the worst rel-L2 over (image, N-tile) blocks."""
import json
import os
import subprocess
import sys

import pytest
import torch

from _util import h, log, min_many_tile_pairs, pair_tiles, pick_bn, rel_l2, rounds, worst_block_rel_l2
from test_fused_gpu import TOL, _reference

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
# (n, C0, Cout, S, G, chan_bias, residual), 3x3 + SiLU, fp16 operands: BN = pick_bn(Cout)
CASES = [(3, 192, 192, 32, 8, True, True), (5, 128, 128, 16, 8, False, True), (9, 64, 64, 8, 8, True, False)]
# 5 N-tiles of 192 / 128 / 64 channels; groups of 96 / 128 / 32 channels tile the N-tiles
MANY_TILES = [(11, 64, 960, 32, 10, True, True), (11, 64, 640, 32, 5, False, True), (11, 64, 320, 32, 10, True, False)]
CASES = CASES + MANY_TILES


def run_cases():
    """-> [(worst (image, N-tile) rel-L2 against the fp64 reference, that block, output)] for every case, in this
    process's epilogue."""
    from nope_b200 import ops
    dev = torch.device("cuda:0")
    D = lambda t: None if t is None else t.to(dev)
    res = []
    for i, (n, C0, Cout, S, G, pb, rs) in enumerate(CASES):
        g = torch.Generator().manual_seed(7 * i + 4)
        x0 = h(torch.randn(n, C0, S, S, generator=g) * 1.2 + 0.2)
        w = h(torch.randn(Cout, C0, 3, 3, generator=g) / (C0 * 9) ** 0.5)
        b = 0.1 * torch.randn(Cout, generator=g)
        gamma = 1 + 0.2 * torch.randn(Cout, generator=g)
        beta = 0.2 * torch.randn(Cout, generator=g)
        cb = h(torch.randn(n, Cout, generator=g)) if pb else None
        r = h(torch.randn(n, Cout, S, S, generator=g)) if rs else None
        d64 = lambda t: None if t is None else t.to(dev, torch.float64)
        ref = _reference("3x3", d64(x0), None, d64(w), d64(b), d64(gamma), d64(beta), G, True, d64(cb), d64(r), 0)
        out = ops.conv_gn_fused(D(x0), D(w), D(b), D(gamma), D(beta), groups=G, silu=True, mode="3x3",
                                chan_bias=D(cb), residual=D(r))
        e, blk = worst_block_rel_l2(out, ref, pick_bn(Cout))
        res.append((e, blk, out.cpu()))
    return res


CHILD = """
import json, sys
import torch
sys.path[:0] = [{root!r}, {here!r}]
import test_conv_gn_epi3_gpu as t
res = t.run_cases()
torch.save([o for _, _, o in res], {path!r})
print(json.dumps([(e, blk) for e, blk, _ in res]))
"""


def test_conv_gn_lockstep_epilogue_all_widths(tmp_path):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    for case in MANY_TILES:
        n, _, Cout, S = case[:4]
        assert pair_tiles(n, S, S, Cout, pick_bn(Cout)) >= min_many_tile_pairs(0), case
    path = str(tmp_path / "epi3.pt")
    env = dict(os.environ, NOPE_GN_EPI="3")
    r = subprocess.run([sys.executable, "-c", CHILD.format(root=ROOT, here=HERE, path=path)], env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    errs = json.loads(r.stdout.strip().splitlines()[-1])
    epi3 = torch.load(path)
    # this process runs the default role-split epilogue (EPI 4): outputs that differ in bits show that the
    # child ran the other epilogue
    epi4 = [o for _, _, o in run_cases()]
    for case, (e, blk), a, b in zip(CASES, errs, epi3, epi4):
        pairs = pair_tiles(case[0], case[3], case[3], case[2], pick_bn(case[2]))
        log("conv_gn_epi3", case=list(case), pair_tiles=pairs, rounds=rounds(pairs, 0), n_tiles=case[2] // pick_bn(case[2]),
            worst_block_rel_l2=e, worst_block=blk, bits_differ_from_epi4=not torch.equal(a, b),
            rel_l2_vs_epi4=rel_l2(a, b))
    for case, (e, blk) in zip(CASES, errs):
        assert e < TOL[0], (case, "worst (image, N-tile)", blk, e)
