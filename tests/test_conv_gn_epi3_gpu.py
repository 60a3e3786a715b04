"""GPU: the lock-step GroupNorm-fused epilogue (EPI 3, chosen once per process by NOPE_GN_EPI=3) at every tile
width it is built for -- BN 192 (three math warpgroups, the third one epilogue only), 128 and 64 -- run through the
sweep's fused layer (ops.conv_gn_fused) in a child process, against the reference and tolerance of the role-split
epilogue (test_fused_gpu)."""
import json
import os
import subprocess
import sys

import pytest
import torch

from _util import h, log, rel_l2
from test_fused_gpu import TOL, _reference

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
# (n, C0, Cout, S, G, chan_bias, residual), 3x3 + SiLU, fp16 operands: BN = Cout
CASES = [(3, 192, 192, 32, 8, True, True), (5, 128, 128, 16, 8, False, True), (9, 64, 64, 8, 8, True, False)]


def run_cases():
    """-> [(rel-L2 against the fp64 reference, output)] for every case, in this process's epilogue."""
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
        ref = _reference("3x3", x0.double(), None, w.double(), b.double(), gamma.double(), beta.double(), G, True,
                         None if cb is None else cb.double(), None if r is None else r.double(), 0)
        out = ops.conv_gn_fused(D(x0), D(w), D(b), D(gamma), D(beta), groups=G, silu=True, mode="3x3",
                                chan_bias=D(cb), residual=D(r)).cpu()
        res.append((rel_l2(out, ref), out))
    return res


CHILD = """
import json, sys
import torch
sys.path[:0] = [{root!r}, {here!r}]
import test_conv_gn_epi3_gpu as t
res = t.run_cases()
torch.save([o for _, o in res], {path!r})
print(json.dumps([e for e, _ in res]))
"""


def test_conv_gn_lockstep_epilogue_all_widths(tmp_path):
    path = str(tmp_path / "epi3.pt")
    env = dict(os.environ, NOPE_GN_EPI="3")
    r = subprocess.run([sys.executable, "-c", CHILD.format(root=ROOT, here=HERE, path=path)], env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    errs = json.loads(r.stdout.strip().splitlines()[-1])
    epi3 = torch.load(path)
    # this process runs the default role-split epilogue (EPI 4): outputs that differ in bits show that the
    # child ran the other epilogue
    epi4 = [o for _, o in run_cases()]
    for case, e, a, b in zip(CASES, errs, epi3, epi4):
        log("conv_gn_epi3", case=list(case), rel_l2=e, bits_differ_from_epi4=not torch.equal(a, b),
            rel_l2_vs_epi4=rel_l2(a, b))
    for case, e in zip(CASES, errs):
        assert e < TOL[0], (case, e)
