"""Per-layer comparison of the GPU sweep against the oracle for a given UNet width."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from oracle import unet_oracle as orc
from nope_b200 import synth_weights as weights
from nope_b200.encoder import FeatureExtractor
from nope_b200.unet import UNet

dim = int(sys.argv[1]) if len(sys.argv) > 1 else 64
names = sys.argv[2].split(",") if len(sys.argv) > 2 else None
sd = weights.make_unet_state_dict(seed=3, u_net_dim=dim)
unet = UNet(u_net_dim=dim, rot_representation_dim=6, encoder=FeatureExtractor(descriptor_size=8),
            pose_mlp_name="single_layer", device="cuda:0")
unet.load_state_dict(sd)
g = torch.Generator().manual_seed(dim)
rf = torch.randn(1, 8, 32, 32, generator=g) * 1.5
poses = torch.randn(3, 6, generator=g)
taps = {}
with torch.no_grad():
    orc.unet_forward(sd, rf.expand(3, -1, -1, -1), poses, taps=taps)
for name in names or ["init_conv", "downs.0.0", "downs.0.1", "downs.0.2", "downs.0.3", "downs.1.0", "downs.1.2",
                      "downs.1.3", "downs.2.3", "downs.3.3", "mid.0", "mid.1", "ups.0.0", "ups.0.2", "ups.0.3",
                      "ups.1.3", "ups.2.3", "ups.3.3", "final_res_block", "final_conv.0"]:
    got = unet.debug_tap(rf, poses, name).cpu()
    ref = taps[name]
    print(f"dim={dim} {name:18s} rel_l2 {float((got - ref).norm() / ref.norm()):.3e}", flush=True)
