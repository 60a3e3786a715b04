"""TEST INFRASTRUCTURE ONLY -- CPU fp32 restatement of the reference hot path.

This is the parity oracle for nope_b200.  Only tests/, __graft_entry__.smoke()
and bench.py's cpu_baseline / --impl reference legs may import it; the product
path (nope_b200/) never does and fails loudly without its CUDA library.

Every function restates one reference function with plain torch CPU ops on a
state_dict (no nn.Module graph), citing the reference file:line it follows
(paths relative to the reference root).  Pinned by oracle/make_golden.py, which
runs the *unmodified* reference modules in the build container on seeded
weights/inputs and (a) asserts this restatement equals them, (b) writes the
golden fixtures in tests/golden/.  The reference ships no tests or golden
vectors of its own for this path (SURVEY.md section 4), so those generated
fixtures are the pin.
"""
import torch
import torch.nn.functional as F

HEADS = 4
DIM_HEAD = 32


# ----------------------------------------------------------------------------
# building blocks
# ----------------------------------------------------------------------------
def block(sd, p, x, groups=8):
    """Block.forward: conv3x3 -> GroupNorm -> SiLU  (model_utils.py:237-253)."""
    x = F.conv2d(x, sd[f"{p}.proj.weight"], sd[f"{p}.proj.bias"], padding=1)
    x = F.group_norm(x, groups, sd[f"{p}.norm.weight"], sd[f"{p}.norm.bias"], eps=1e-5)
    return F.silu(x)


def resnet_block(sd, p, x, emb=None):
    """ResnetBlock.forward (model_utils.py:271-279): the pose projection is added
    AFTER block1's SiLU; res_conv is a 1x1 when Cin != Cout."""
    h = block(sd, f"{p}.block1", x)
    if emb is not None and f"{p}.mlp.1.weight" in sd:
        t = F.linear(F.silu(emb), sd[f"{p}.mlp.1.weight"], sd[f"{p}.mlp.1.bias"])
        h = t[:, :, None, None] + h
    h = block(sd, f"{p}.block2", h)
    if f"{p}.res_conv.weight" in sd:
        x = F.conv2d(x, sd[f"{p}.res_conv.weight"], sd[f"{p}.res_conv.bias"])
    return h + x


def linear_attention(sd, p, x):
    """Residual(PreNorm(LinearAttention)) (model_utils.py:393-418, 226-234, 198-204)."""
    b, c, h, w = x.shape
    n = h * w
    y = F.group_norm(x, 1, sd[f"{p}.fn.norm.weight"], sd[f"{p}.fn.norm.bias"], eps=1e-5)
    qkv = F.conv2d(y, sd[f"{p}.fn.fn.to_qkv.weight"])            # no bias
    q, k, v = [t.reshape(b, HEADS, DIM_HEAD, n) for t in qkv.chunk(3, dim=1)]
    q = q.softmax(dim=-2) * DIM_HEAD ** -0.5                       # over d, then scale
    k = k.softmax(dim=-1)                                          # over n
    context = torch.einsum("bhdn,bhen->bhde", k, v)
    out = torch.einsum("bhde,bhdn->bhen", context, q).reshape(b, HEADS * DIM_HEAD, h, w)
    out = F.conv2d(out, sd[f"{p}.fn.fn.to_out.0.weight"], sd[f"{p}.fn.fn.to_out.0.bias"])
    out = F.group_norm(out, 1, sd[f"{p}.fn.fn.to_out.1.weight"],
                       sd[f"{p}.fn.fn.to_out.1.bias"], eps=1e-5)
    return out + x


def attention(sd, p, x):
    """Residual(PreNorm(Attention)) at the bottleneck (model_utils.py:367-390)."""
    b, c, h, w = x.shape
    n = h * w
    y = F.group_norm(x, 1, sd[f"{p}.fn.norm.weight"], sd[f"{p}.fn.norm.bias"], eps=1e-5)
    qkv = F.conv2d(y, sd[f"{p}.fn.fn.to_qkv.weight"])
    q, k, v = [t.reshape(b, HEADS, DIM_HEAD, n) for t in qkv.chunk(3, dim=1)]
    q = q * DIM_HEAD ** -0.5
    sim = torch.einsum("bhdi,bhdj->bhij", q, k)
    sim = sim - sim.amax(dim=-1, keepdim=True)
    attn = sim.softmax(dim=-1)
    out = torch.einsum("bhij,bhdj->bhid", attn, v)                 # b h n d
    out = out.permute(0, 1, 3, 2).reshape(b, HEADS * DIM_HEAD, h, w)  # b (h d) x y
    out = F.conv2d(out, sd[f"{p}.fn.fn.to_out.weight"], sd[f"{p}.fn.fn.to_out.bias"])
    return out + x


def hard_downsample(sd, p, x):
    """HardDownsample (model_utils.py:168-172): 'b c (h p1) (w p2) -> b (c p1 p2) h w' + 1x1."""
    b, c, hh, ww = x.shape
    x = x.reshape(b, c, hh // 2, 2, ww // 2, 2).permute(0, 1, 3, 5, 2, 4)
    x = x.reshape(b, c * 4, hh // 2, ww // 2)
    return F.conv2d(x, sd[f"{p}.1.weight"], sd[f"{p}.1.bias"])


def hard_upsample(sd, p, x):
    """HardUpsample (model_utils.py:161-165): nearest x2 + conv3x3."""
    x = F.interpolate(x, scale_factor=2, mode="nearest")
    return F.conv2d(x, sd[f"{p}.1.weight"], sd[f"{p}.1.bias"], padding=1)


# ----------------------------------------------------------------------------
# UNet.forward (u_net.py:160-198)
# ----------------------------------------------------------------------------
def unet_forward(sd, x, pose, taps=None):
    """x [B,C,32,32] fp32, pose [B,6] -> [B,C,32,32].  `taps`, if a dict, receives
    named intermediate activations for per-layer parity tests."""
    def tap(name, t):
        if taps is not None:
            taps[name] = t
    n_levels = 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("downs."))
    x = F.conv2d(x, sd["init_conv.weight"], sd["init_conv.bias"], padding=1)
    r = x.clone()
    tap("init_conv", x)
    c = F.linear(pose, sd["pose_mlp.0.weight"], sd["pose_mlp.0.bias"])   # u_net.py:63-66
    hs = []
    for i in range(n_levels):
        x = resnet_block(sd, f"downs.{i}.0", x, c)
        tap(f"downs.{i}.0", x)
        hs.append(x)
        x = resnet_block(sd, f"downs.{i}.1", x, c)
        tap(f"downs.{i}.1", x)
        x = linear_attention(sd, f"downs.{i}.2", x)
        tap(f"downs.{i}.2", x)
        hs.append(x)
        if f"downs.{i}.3.1.weight" in sd:
            x = hard_downsample(sd, f"downs.{i}.3", x)
        else:
            x = F.conv2d(x, sd[f"downs.{i}.3.weight"], sd[f"downs.{i}.3.bias"], padding=1)
        tap(f"downs.{i}.3", x)
    # the mid block runs twice with shared weights (u_net.py:177-183)
    for rep in range(2):
        x = resnet_block(sd, "mid_block1", x, c)
        x = attention(sd, "mid_attn", x)
        x = resnet_block(sd, "mid_block2", x, c)
        tap(f"mid.{rep}", x)
    for i in range(n_levels):
        x = torch.cat((x, hs.pop()), dim=1)
        x = resnet_block(sd, f"ups.{i}.0", x, c)
        tap(f"ups.{i}.0", x)
        x = torch.cat((x, hs.pop()), dim=1)
        x = resnet_block(sd, f"ups.{i}.1", x, c)
        x = linear_attention(sd, f"ups.{i}.2", x)
        tap(f"ups.{i}.2", x)
        if f"ups.{i}.3.1.weight" in sd:
            x = hard_upsample(sd, f"ups.{i}.3", x)
        else:
            x = F.conv2d(x, sd[f"ups.{i}.3.weight"], sd[f"ups.{i}.3.bias"], padding=1)
        tap(f"ups.{i}.3", x)
    x = torch.cat((x, r), dim=1)
    x = resnet_block(sd, "final_res_block", x, c)
    tap("final_res_block", x)
    x = resnet_block(sd, "final_conv.0", x, None)      # no pose here (nn.Sequential call)
    tap("final_conv.0", x)
    return F.conv2d(x, sd["final_conv.1.weight"], sd["final_conv.1.bias"])


# ----------------------------------------------------------------------------
# FeatureExtractor.encode_image (template.py:47-53; resnet.py:55-91,135-152)
# ----------------------------------------------------------------------------
def _bn(sd, p, x):
    return F.batch_norm(x, sd[f"{p}.running_mean"], sd[f"{p}.running_var"],
                        sd[f"{p}.weight"], sd[f"{p}.bias"], training=False, eps=1e-5)


def _bottleneck(sd, p, x, stride):
    out = F.relu(_bn(sd, f"{p}.bn1", F.conv2d(x, sd[f"{p}.conv1.weight"])))
    out = F.relu(_bn(sd, f"{p}.bn2", F.conv2d(out, sd[f"{p}.conv2.weight"],
                                               stride=stride, padding=1)))
    out = _bn(sd, f"{p}.bn3", F.conv2d(out, sd[f"{p}.conv3.weight"]))
    if f"{p}.downsample.0.weight" in sd:
        x = _bn(sd, f"{p}.downsample.1",
                F.conv2d(x, sd[f"{p}.downsample.0.weight"], stride=stride))
    return F.relu(out + x)


def encode_image(sd, image, prefix="", taps=None):
    """ResNet-50 without max-pool, layer4 stride 1 (=> /8), eval-mode BN, then
    ReLU -> 1x1(2048->256) -> ReLU -> 1x1(256->D); normalize=False
    (configs/model/template_base.yaml:12).  taps, if a dict, receives (input, output) of every module the native
    engine runs on its own (nope_encoder_run_block) under its name: "stem" (conv1 + bn1 + ReLU),
    "backbone.layer<l>.<b>" and "projector"."""
    sdp = {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)} if prefix else sd

    def module(name, fn, h):
        out = fn(h)
        if taps is not None:
            taps[name] = (h, out)
        return out

    x = module("stem", lambda t: F.relu(_bn(sdp, "backbone.bn1", F.conv2d(t, sdp["backbone.conv1.weight"], stride=2,
                                                                           padding=3))), image)
    for li, (blocks, stride) in enumerate([(3, 1), (4, 2), (6, 2), (3, 1)], start=1):
        for b in range(blocks):
            p = f"backbone.layer{li}.{b}"
            x = module(p, lambda t: _bottleneck(sdp, p, t, stride if b == 0 else 1), x)
    return module("projector", lambda t: F.conv2d(F.relu(F.conv2d(F.relu(t), sdp["projector.1.weight"])),
                                                  sdp["projector.3.weight"]), x)


# ----------------------------------------------------------------------------
# retrieval (model.py:254-266) and the sweep (model.py:193-252, 113-124)
# ----------------------------------------------------------------------------
def l2_similarity(query_feat, template_feat):
    """similarity[b,n] = -sum_hw sqrt(sum_c (q-t)^4)   (model.py:260-262;
    same formula restated in loss.py:129-132)."""
    d = (query_feat[:, None] - template_feat) ** 2
    d = torch.norm(d, dim=2)
    return -d.sum(dim=3).sum(dim=2)


def cosine_similarity(query_feat, template_feat, eps=1e-8):
    """Extension (not in the reference, SURVEY.md F3 / section 8c): cosine of the
    flattened C*H*W descriptors, F.cosine_similarity semantics."""
    b, n = template_feat.shape[:2]
    q = query_feat.reshape(b, 1, -1).expand(b, n, -1)
    return F.cosine_similarity(q, template_feat.reshape(b, n, -1), dim=-1, eps=eps)


def cosine_occlusion_similarity(query_feat, template_feat, threshold=0.2, eps=1e-8):
    """Extension (SURVEY.md section 8c / row f4): the two modules the reference's encoder declares but
    never calls -- `sim_distance = nn.CosineSimilarity(dim=1)` (per-pixel cosine over channels,
    src/model/encoder/template.py:45) followed by `OcclusionAwareSimilarity(threshold)` (similarities
    <= threshold set to zero, src/model/encoder/base_template.py:67-75) -- averaged over the pixels."""
    b, n = template_feat.shape[:2]
    q = query_feat[:, None].expand_as(template_feat)
    s = F.cosine_similarity(q, template_feat, dim=2, eps=eps)          # [B, N, H, W]
    s = torch.where(s <= threshold, torch.zeros_like(s), s)
    return s.flatten(2).mean(dim=2)


def topk_lowest_index(similarity, k):
    """torch.topk's tie order is unspecified; the contract here is descending
    score, ties broken by the LOWEST index (SURVEY.md section 7 'Tie-breaking')."""
    b, n = similarity.shape
    idx = torch.arange(n).expand(b, n)
    # stable sort on -score keeps index order among equals
    order = torch.sort(-similarity, dim=1, stable=True).indices
    return order[:, :k]


def generate_templates(unet_sd, reference_feat, all_relativeR, chunk=16):
    """[B,C,32,32], [B,N,6] -> [B,N,C,32,32]; the reference loops over N at batch B
    (model.py:212-222); batching along dim 0 is arithmetically identical."""
    b, n = all_relativeR.shape[:2]
    out = []
    x = reference_feat[:, None].expand(b, n, *reference_feat.shape[1:]).reshape(
        b * n, *reference_feat.shape[1:])
    p = all_relativeR.reshape(b * n, -1)
    for s in range(0, b * n, chunk):
        out.append(unet_forward(unet_sd, x[s:s + chunk], p[s:s + chunk]))
    return torch.cat(out).reshape(b, n, *reference_feat.shape[1:])


def predict_pose(full_sd, query, reference, all_relativeR, template_poses=None,
                 k=5, metric="l2"):
    """eval_geodesic without logging (model.py:313-357): encode, sweep, score, top-k,
    pose lookup."""
    enc_sd = {kk[len("encoder."):]: v for kk, v in full_sd.items() if kk.startswith("encoder.")}
    unet_sd = {kk: v for kk, v in full_sd.items() if not kk.startswith("encoder.")}
    with torch.no_grad():
        qf = encode_image(enc_sd, query)
        rf = encode_image(enc_sd, reference)
        emb = generate_templates(unet_sd, rf, all_relativeR)
        sim = l2_similarity(qf, emb) if metric == "l2" else cosine_similarity(qf, emb)
        idx = topk_lowest_index(sim, min(k, sim.shape[1]))
    poses = template_poses[idx] if template_poses is not None else None
    return poses, idx, sim, emb, qf, rf
