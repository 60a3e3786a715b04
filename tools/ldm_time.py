"""Quick timing of the LDM-variant sweep (not the bench): N hypotheses of one reference latent."""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from nope_b200.ldm import UNetModelPose
from nope_b200.synth_weights import make_ldm_state_dict

N = int(sys.argv[1]) if len(sys.argv) > 1 else 128
m = UNetModelPose(device="cuda:0", chunk=N)
t0 = time.time()
m.load_state_dict(make_ldm_state_dict(seed=0))
print(f"load {time.time() - t0:.1f}s", flush=True)
g = torch.Generator().manual_seed(0)
ref = torch.randn(1, 4, 32, 32, generator=g).cuda()
qry = torch.randn(1, 4, 32, 32, generator=g).cuda()
poses = torch.randn(1, N, 6, generator=g).cuda()
for _ in range(2):
    m.sweep(ref, poses, qry, want_emb=False, k=5)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
reps = 3
for _ in range(reps):
    out = m.sweep(ref, poses, qry, want_emb=False, k=5)
e1.record()
torch.cuda.synchronize()
if os.environ.get("NOPE_PROFILE"):
    torch.cuda.profiler.start()
    m.sweep(ref, poses, qry, want_emb=False, k=5)
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
ms = e0.elapsed_time(e1) / reps
print(f"LDM sweep N={N}: {ms:.2f} ms/sweep, {N / ms * 1e3:.0f} hyp/s, "
      f"{m.last_launch_count} launches, mem {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB torch", flush=True)
