"""GPU: the lock-step GroupNorm-fused epilogue (EPI 3, chosen once per process by NOPE_GN_EPI=3) at every tile
width it is built for -- BN 192 (three math warpgroups, the third one epilogue only), 128 and 64 -- run in a child
process against the same reference as the role-split epilogue."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CASES = [(3, 192, 192, 32, 8), (5, 128, 128, 16, 8), (9, 64, 64, 8, 8)]   # (n, C0, Cout, S, G): BN = Cout

CHILD = r"""
import json, sys
import torch
import torch.nn.functional as F
sys.path[:0] = [ROOT, HERE]
from _util import rel_l2
from test_ops_gpu import conv_reference, make_conv_case
from nope_b200 import ops
dev = torch.device("cuda:0")
res = []
for n, C0, Cout, S, G in CASES:
    x0, _, w, b = make_conv_case(n, C0, 0, Cout, S, "3x3", seed=4)
    g = torch.Generator().manual_seed(S + Cout)
    gamma = 1 + 0.2 * torch.randn(Cout, generator=g)
    beta = 0.2 * torch.randn(Cout, generator=g)
    ref = F.silu(F.group_norm(conv_reference(x0, None, w, b, "3x3"), G, gamma, beta, eps=1e-5))
    out = ops.conv_gn(x0.to(dev), w.to(dev), b.to(dev), gamma.to(dev), beta.to(dev), G, silu=True,
                      mode="3x3", impl="tcgen05_2cta")
    res.append(rel_l2(out, ref))
print(json.dumps(res))
"""


def test_conv_gn_lockstep_epilogue_all_widths():
    env = dict(os.environ, NOPE_GN_EPI="3")
    code = f"ROOT = {ROOT!r}\nHERE = {HERE!r}\nCASES = {CASES!r}\n" + CHILD
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    errs = json.loads(r.stdout.strip().splitlines()[-1])
    for case, e in zip(CASES, errs):
        assert e < 2e-3, (case, e)
