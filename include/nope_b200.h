/* nope_b200 -- C ABI of the H100-native NOPE inference hot path.
 *
 * The reference (nv-nguyen/nope) is pure Python/PyTorch and has no FFI of its own;
 * each entry point below names the reference function it replaces (paths relative to
 * the reference root).  All pointers are raw device pointers unless marked HOST; no
 * torch types cross this boundary.  Every function returns 0 on success and a negative
 * value on failure; nope_last_error() then returns a description (thread-local).
 * `stream` is a cudaStream_t passed as void* (NULL = default stream).
 *
 * Layout conventions at the boundary follow the reference's tensors:
 *   latent features   fp32 NCHW [B, C, 32, 32]           (encoder output, u_net input)
 *   poses             fp32 [B, N, 6]                     (6-D rotations, all_relativeR)
 *   embeddings        fp32 [B, N, C, 32, 32]             (pred_feat_templates)
 *   similarity        fp32 [B, N]; nearest_idx int64 [B, k]
 * Inside the library activations are NHWC fp16 and weights are repacked K-major fp16.
 *
 * ABI version 2 (round 2): nope_unet_set_option / get_option, caller-owned workspace
 * (nope_unet_workspace_bytes / nope_unet_set_workspace), nope_unet_profile_read reports executed and
 * algorithmic FLOPs, nope_op_conv_gn_fused, nope_topk_merge, nope_score_topk metric 2.
 * Later additions under version 2 include nope_encoder_set_option and nope_vae_set_option.
 */
#ifndef NOPE_B200_H
#define NOPE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct nope_unet nope_unet_t;

#define NOPE_METRIC_L2 0      /* reference "l2": -(sum_hw sqrt(sum_c (q-t)^4)), model.py:260-262 */
#define NOPE_METRIC_COSINE 1  /* extension: cosine of flattened descriptors (not in the reference) */
/* extension: occlusion-aware cosine -- the per-pixel cosine over channels (the encoder's
 * `sim_distance = nn.CosineSimilarity(dim=1)`, src/model/encoder/template.py:45) with similarities <=
 * threshold set to zero (`OcclusionAwareSimilarity`, src/model/encoder/base_template.py:67-75; threshold
 * 0.2 in configs/model/template_base.yaml), averaged over the 32x32 pixels */
#define NOPE_METRIC_COSINE_OCC 2

/* Thread-local message of the last failing call on this thread. */
const char* nope_last_error(void);

/* Library/ABI version and the SM architecture the kernels were built for ("sm_90a"). */
int nope_abi_version(void);
const char* nope_build_arch(void);

/* ---- engine lifetime ------------------------------------------------------------
 * Replaces construction of src/model/u_net/denoising_diffusion_pytorch/u_net.py:27-158
 * (UNet.__init__ with use_hard_up_down=True, dim_mults=(1,2,4,8), 8 groups,
 * pose_mlp_name="single_layer").  u_net_dim must be a multiple of 64; latent_ch <= 8;
 * latent_hw is the latent side (32 for 256x256 images). */
int nope_unet_create(nope_unet_t** out, int u_net_dim, int latent_ch, int latent_hw, int device);
void nope_unet_destroy(nope_unet_t* u);

/* Hand one tensor of the reference state_dict to the engine, by its reference key
 * (e.g. "downs.0.0.block1.proj.weight"; SURVEY.md 8b).  `data` is a HOST fp32 pointer,
 * contiguous, with `ndim` sizes in `shape`.  Unknown keys are rejected; encoder.* keys
 * are not accepted here (they go to nope_encoder_load_tensor below).
 * Replaces nn.Module.load_state_dict for the UNet; the shape-filtered partial load of
 * src/utils/weight.py:6-37 (skip keys whose shape does not match) is done by the Python mirror
 * (nope_b200.unet.load_checkpoint), this call rejects a mismatching shape. */
int nope_unet_load_tensor(nope_unet_t* u, const char* key, const float* data,
                          const int64_t* shape, int ndim);

/* Checks that every tensor was provided, repacks weights (OIHW fp32 -> K-major fp16,
 * pose projections concatenated into one GEMM) and uploads them. */
int nope_unet_finalize(nope_unet_t* u);

/* Tunables: hypotheses per chunk (workspace = ~4.7 MB per hypothesis at u_net_dim 192), and the
 * convolution implementation: 2 = wgmma, clustered kernel with the fused epilogues (the only one;
 * anything else is an error). */
int nope_unet_set_chunk(nope_unet_t* u, int hyps_per_chunk);
int nope_unet_set_conv_impl(nope_unet_t* u, int impl);
/* Named options:
 *   "precision" (before nope_unet_finalize): 0 = fp16 operands (default; embeddings ~1.3e-3 rel-L2 of the
 *       fp32 reference, u_net.py:160-198), 1 = exact weights: every weight is an fp16 pair W_hi + W_lo and
 *       each convolution accumulates A W_hi + A W_lo (2x the tensor-core work), 2 = split precision:
 *       exact weights and activations carried as fp16 pairs, A_hi W_hi + A_hi W_lo + A_lo W_hi (3x;
 *       the "parity" mode that meets the 1e-3 embedding tolerance with margin), 3 = bf16 operands and
 *       activations (BASELINE configs[2]; 8-bit mantissa: embeddings ~1e-2 of the fp32 reference),
 *       4 = split precision with single-fp16 tensors inside the ResnetBlocks (block2 convolutions run two
 *       products instead of three; embeddings ~5e-4: the fastest mode inside the 1e-3 tolerance);
 *   "conv_impl": as nope_unet_set_conv_impl;
 *   "attn_impl": LinearAttention core, 0 = wgmma kernel at 32x32 / 16x16 (CUDA cores below 128 tokens),
 *       1 = CUDA-core kernel everywhere. */
int nope_unet_set_option(nope_unet_t* u, const char* name, int value);
int nope_unet_get_option(const nope_unet_t* u, const char* name, int* value);

/* Workspace ownership.  By default the engine owns one device slab and grows it on demand (a growth
 * synchronises the device and calls cudaMalloc).  A host framework that wants every byte to come from
 * its own allocator asks for the size and hands a buffer over; the sweep then never allocates and
 * fails if the buffer is too small.  hyps = min(chunk, B*N) hypotheses per chunk, refs = B,
 * scores = B*Q*N, the number of scored (reference, query, pose) triples (0 when no query is scored).  The buffer must stay alive while the engine uses it. */
int64_t nope_unet_workspace_bytes(nope_unet_t* u, int hyps, int refs, int scores);
int nope_unet_set_workspace(nope_unet_t* u, void* device_ptr, int64_t bytes, int hyps, int refs, int scores);

/* ---- the hot path -----------------------------------------------------------------
 * Sweep over the pose grid.  Replaces the Python loop of
 * PoseConditional.generate_templates (src/model/model.py:193-252) around
 * UNet.forward (u_net.py:160-198) and, when query_feat != NULL, the scoring and top-k of
 * PoseConditional.retrieval (model.py:254-266) fused onto the last layer.
 *   ref_feat   [B, C, hw, hw] fp32   encode_image(reference)
 *   poses      [B, N, 6] fp32        all_relativeR
 *   query_feat [B, C, hw, hw] fp32 or NULL
 *   out_emb    [B, N, C, hw, hw] fp32 or NULL (skip materialising the templates)
 *   out_sim    [B, N] fp32 or NULL   (requires query_feat)
 *   out_topv / out_topi  [B, k] fp32 / int64 or NULL; descending score, ties broken by
 *              the lowest index; indices are offset by idx_base (global index of this
 *              shard's first pose).  k = 0 skips the ranking.
 * Kernels are enqueued on `stream`; the call does not synchronise. */
int nope_unet_sweep(nope_unet_t* u, const float* ref_feat, const float* poses, int B, int N,
                    const float* query_feat, float* out_emb, float* out_sim, int k,
                    float* out_topv, int64_t* out_topi, int64_t idx_base, void* stream);

/* One sweep per reference, Q queries per reference: the templates depend on the reference and the pose grid
 * only, so several queries of one object (video frames, detections of several instances) share one sweep and
 * are all scored in its last layer.  Arguments as nope_unet_sweep, plus Q >= 1, with
 *   query_feat [B, Q, C, hw, hw] fp32
 *   out_sim    [B, Q, N] fp32 or NULL
 *   out_topv / out_topi  [B, Q, k]
 * sim[b, q] is bit-identical to a Q = 1 sweep of query q alone; nope_unet_sweep is the Q = 1 case.  A
 * caller-owned workspace must be sized for scores = B*Q*N. */
int nope_unet_sweep_multi(nope_unet_t* u, const float* ref_feat, const float* poses, int B, int N,
                          const float* query_feat, int Q, float* out_emb, float* out_sim, int k,
                          float* out_topv, int64_t* out_topi, int64_t idx_base, void* stream);

/* Similarity metric of the scoring fused onto the sweep's last layer (NOPE_METRIC_*; default l2, the only
 * one the reference implements, model.py:254-266).  occlusion_threshold is used by NOPE_METRIC_COSINE_OCC. */
int nope_unet_set_metric(nope_unet_t* u, int metric, float occlusion_threshold);

/* Number of kernels the last nope_unet_sweep call enqueued (for bench.py's gpu_launches). */
int64_t nope_unet_last_launch_count(const nope_unet_t* u);

/* Profiling hook for bench.py's roofline: when enabled, every tensor-core convolution
 * launch of subsequent sweeps is bracketed by CUDA events on the launching stream.
 * nope_unet_profile_read synchronises the device and returns the summed launch time
 * (ms), the summed EXECUTED FLOPs (2*M*N*K' per launch, K' counting the extra split-precision
 * K-segments), the summed ALGORITHMIC FLOPs (2*M*N*K of the layer, what the reference computes),
 * the launch count and the best single-launch executed TFLOP/s.  Enabling/disabling clears the
 * recorded events. */
int nope_unet_profile(nope_unet_t* u, int enable);
int nope_unet_profile_read(nope_unet_t* u, double* conv_ms, double* conv_flops, double* conv_alg_flops,
                           int64_t* conv_launches, double* max_launch_tflops);

/* ---- template encoder ----------------------------------------------------------------
 * FeatureExtractor.encode_image (src/model/encoder/template.py:47-53): ResNet-50 without
 * max-pool and with layer4 at stride 1 (src/model/encoder/resnet.py:93-152), eval-mode
 * BatchNorm folded into the convolutions, projector ReLU-1x1-ReLU-1x1, normalize=False.
 * Runs on the wgmma convolution kernel with split-precision (fp16 hi+lo) operands, so the
 * latents match the reference's fp32 path to 5e-5 rel-L2 (measured; tests assert 1.5e-4;
 * cuDNN TF32 / fp16 are 2-3e-3 off).  Keys are the reference's
 * `backbone.*` / `projector.*` names (HOST fp32 pointers, shape-checked); 256x256 inputs. */
typedef struct nope_encoder nope_encoder_t;
int nope_encoder_create(nope_encoder_t** out, int descriptor_size, int device);
void nope_encoder_destroy(nope_encoder_t* e);
int nope_encoder_load_tensor(nope_encoder_t* e, const char* key, const float* data,
                             const int64_t* shape, int ndim);
int nope_encoder_finalize(nope_encoder_t* e);
/* Named options, before nope_encoder_finalize only (the weight packing depends on them):
 *   "precision": 0 = split precision (default; the fp32-accurate latents above), 1 = fp16: one fp16 weight per tap
 *       (BatchNorm folded in float64, then rounded once), one fp16 copy of every stored activation, fp32 accumulation,
 *       one K-segment per tap instead of three (DESIGN.md section 22).  Every encode and run_block call honours it.
 * An unknown name or value, or a call after finalize, is refused before any CUDA call. */
int nope_encoder_set_option(nope_encoder_t* e, const char* name, int value);
/* images [B, 3, 256, 256] fp32 NCHW (device) -> out [B, D, 32, 32] fp32 NCHW (device).
 * Any B >= 1: the engine walks the batch 32 images at a time (workspace ~80 MB per image of a chunk). */
int nope_encoder_encode(nope_encoder_t* e, const float* images, int B, float* out, void* stream);
int64_t nope_encoder_last_launch_count(const nope_encoder_t* e);
/* Debug / parity: run ONE module of the encoder in isolation, the launches encode makes for it.
 *   name "stem" (x = images [n, 3, 256, 256]), "backbone.layer<l>.<b>" (a bottleneck) or "projector";
 *   x [n, C, H, H] fp32 NCHW (device), C and H the module's input shape, 1 <= n <= 32 -> out fp32 NCHW (device):
 *   hi + lo of the module's (hi, lo) output, the projector's fp32 output [n, D, 32, 32].  An unknown name, a C or H
 *   that does not fit it, n out of range or an out_capacity_floats below the output's size fail.
 * Synchronises the stream. */
int nope_encoder_run_block(nope_encoder_t* e, const char* name, const float* x, int C, int H, int n, float* out,
                           int64_t out_capacity_floats, void* stream);

/* In-plane rotation search (DESIGN.md section 11).  cossin [A, 2] fp32 holds (cos, sin) of the angles
 * alpha_a = a * 360 / A.  Rotated copy a of an image is I_a(x, y) = I(c + R2(alpha_a) ((x, y) - c)) in pixel-index
 * coordinates (x right, y down), c = ((W - 1) / 2, (H - 1) / 2), R2 = [[cos, -sin], [sin, cos]], bilinear, taps
 * outside the image read -1.  Products and sums are rounded one by one (no FMA) in a fixed order.  A match of copy a
 * with a template of pose T means the query pose Rz(alpha_a) T.  Both calls require B >= 1 and 1 <= A <= 360 and
 * refuse before any CUDA call.
 * nope_inplane_rotate: images [B, 3, H, W] fp32 (device) -> out [B, A, 3, H, W] fp32 (device); H, W >= 1.
 * nope_encoder_encode_inplane: images [B, 3, 256, 256] -> out [B, A, D, 32, 32], equal to nope_encoder_encode of
 * the rotated batch [B * A, 3, 256, 256] without forming it: the (image, angle) pairs go 32 at a time through a
 * staging buffer the engine allocates on its first call (25 MB). */
int nope_inplane_rotate(const float* images, int B, int H, int W, const float* cossin, int A, float* out,
                        void* stream);
int nope_encoder_encode_inplane(nope_encoder_t* e, const float* images, int B, const float* cossin, int A,
                                float* out, void* stream);

/* Rotated copies of arbitrary (image, roll) pairs (DESIGN.md section 14), with the arithmetic of
 * nope_inplane_rotate: pair p rotates image image_idx[p] (int32) by (cossin[2p], cossin[2p + 1]), so a pair holding
 * angle-table entry a equals copy a bit for bit.  An image index outside [0, B) gives a copy that is -1 everywhere.
 * Both calls require B >= 1 and 1 <= P < 2^30 and refuse before any CUDA call.
 * nope_inplane_rotate_pairs: images [B, 3, H, W] fp32 (device) -> out [P, 3, H, W]; H, W >= 1.
 * nope_encoder_encode_rotated: images [B, 3, 256, 256] -> out [P, D, 32, 32], equal to nope_encoder_encode of the
 * rotated pairs [P, 3, 256, 256]: they go 32 at a time, in pair order, through the staging buffer of
 * nope_encoder_encode_inplane. */
int nope_inplane_rotate_pairs(const float* images, int B, int H, int W, const int32_t* image_idx,
                              const float* cossin, int P, float* out, void* stream);
int nope_encoder_encode_rotated(nope_encoder_t* e, const float* images, int B, const int32_t* image_idx,
                                const float* cossin, int P, float* out, void* stream);

/* Stable Diffusion VAE encoder (DESIGN.md section 16): AutoencoderKL.encode(x).latent_dist.mode() * 0.18215 of the
 * SD v1 configuration (block_out_channels 128, 256, 512, 512; two resnets per block; GroupNorm(32, eps 1e-6); one
 * 512-channel attention head; latent_channels 4), the encoder of the LDM variant and of vae_base.yaml.
 * Convolutions run on the wgmma kernel with split-precision (fp16 hi + lo) operands; the attention core in fp32.
 * nope_vae_load_tensor takes the diffusers state_dict names with the 0.14-era attention projections
 * (`encoder.mid_block.attentions.0.{query,key,value,proj_attn}`), HOST fp32 pointers, shape-checked; every key of
 * the schema is required by nope_vae_finalize, which also allocates the workspace (16 images, ~3.2 GB).
 * Encode calls: images [B, 3, 256, 256] fp32 NCHW (device) in [-1, 1]; any B >= 1, 16 images at a time, and a latent
 * does not depend on the batch it was encoded in.  nope_vae_encode -> out [B, 4, 32, 32];
 * nope_vae_encode_inplane (1 <= A <= 360, cossin [A, 2]) -> out [B, A, 4, 32, 32] and nope_vae_encode_rotated
 * (1 <= P < 2^30, image_idx [P] int32, cossin [P, 2]) -> out [P, 4, 32, 32] rotate exactly as
 * nope_encoder_encode_inplane / nope_encoder_encode_rotated and equal nope_vae_encode of the rotated batch.  Bad
 * arguments are refused before any CUDA call; no call synchronises the host. */
typedef struct nope_vae nope_vae_t;
int nope_vae_create(nope_vae_t** out, int device);
void nope_vae_destroy(nope_vae_t* v);
int nope_vae_load_tensor(nope_vae_t* v, const char* key, const float* data, const int64_t* shape, int ndim);
int nope_vae_finalize(nope_vae_t* v);
/* "precision" as nope_encoder_set_option (0 = split, the default; 1 = fp16 operands and stored activations, with the
 * fp32 residual stream, float64 GroupNorm statistics, fp32 attention core and fp32 conv_out kept), before
 * nope_vae_finalize only; refusals as there. */
int nope_vae_set_option(nope_vae_t* v, const char* name, int value);
int nope_vae_encode(nope_vae_t* v, const float* images, int B, float* out, void* stream);
int nope_vae_encode_inplane(nope_vae_t* v, const float* images, int B, const float* cossin, int A, float* out,
                            void* stream);
int nope_vae_encode_rotated(nope_vae_t* v, const float* images, int B, const int32_t* image_idx, const float* cossin,
                            int P, float* out, void* stream);
int64_t nope_vae_last_launch_count(const nope_vae_t* v);
/* Debug / parity: run ONE module of the encoder in isolation, through the member functions encode calls.
 *   name "encoder.conv_in" (x = images [n, 3, 256, 256]), "encoder.down_blocks.<i>.resnets.<j>",
 *   "encoder.down_blocks.<i>.downsamplers.0", "encoder.mid_block.resnets.<j>", "encoder.mid_block.attentions.0" or
 *   "encoder.conv_out" (conv_norm_out + SiLU + conv_out + quant_conv mean x 0.18215 -> [n, 4, 32, 32]);
 *   x [n, C, H, H] fp32 NCHW (device), the module's input shape, 1 <= n <= 16 -> out: the fp32 residual stream after
 *   the module, out_pair (nullable; not for conv_out): hi + lo of its (hi, lo) copy, both fp32 NCHW (device).
 * Synchronises the stream. */
int nope_vae_run_block(nope_vae_t* v, const char* name, const float* x, int C, int H, int n, float* out,
                       float* out_pair, int64_t out_capacity_floats, void* stream);

/* Stable Diffusion VAE decoder (DESIGN.md section 17): AutoencoderKL.decode(z / 0.18215).sample of the SD v1
 * configuration (post_quant_conv 1x1; conv_in 3x3 4 -> 512; mid block as the encoder's; four UpDecoderBlock2D of three
 * resnets with 512, 512, 256, 128 channels, blocks 0-2 ending in nearest x2 + 3x3 conv; GroupNorm(32, eps 1e-6),
 * SiLU, conv_out 3x3 128 -> 3), with the encoder's split-precision scheme.  A handle of its own: it takes the 140
 * `decoder.*` / `post_quant_conv.*` tensors (0.14-era attention names under `decoder.mid_block.attentions.0.`), HOST
 * fp32 pointers, shape-checked; every key is required by nope_vae_decoder_finalize, which also allocates the workspace
 * (8 images, ~3.2 GB).  nope_vae_decoder_decode: latents [B, 4, 32, 32] fp32 (device) -> out [B, 3, 256, 256] fp32
 * NCHW, unclamped; any B >= 1, 8 latents at a time, and an image does not depend on the batch it was decoded in.
 * Bad arguments are refused before any CUDA call; no call synchronises the host. */
typedef struct nope_vae_decoder nope_vae_decoder_t;
int nope_vae_decoder_create(nope_vae_decoder_t** out, int device);
void nope_vae_decoder_destroy(nope_vae_decoder_t* d);
int nope_vae_decoder_load_tensor(nope_vae_decoder_t* d, const char* key, const float* data, const int64_t* shape,
                                 int ndim);
int nope_vae_decoder_finalize(nope_vae_decoder_t* d);
int nope_vae_decoder_decode(nope_vae_decoder_t* d, const float* latents, int B, float* out, void* stream);
int64_t nope_vae_decoder_last_launch_count(const nope_vae_decoder_t* d);
/* Debug / parity: as nope_vae_run_block, for the modules of decode: "decoder.conv_in" (post_quant_conv with
 * 1 / 0.18215, then conv_in; x = latents [n, 4, 32, 32]), "decoder.mid_block.resnets.<j>",
 * "decoder.mid_block.attentions.0", "decoder.up_blocks.<i>.resnets.<j>", "decoder.up_blocks.<i>.upsamplers.0" and
 * "decoder.conv_out" (conv_norm_out + SiLU + conv_out -> [n, 3, 256, 256]); 1 <= n <= 8. */
int nope_vae_decoder_run_block(nope_vae_decoder_t* d, const char* name, const float* x, int C, int H, int n,
                               float* out, float* out_pair, int64_t out_capacity_floats, void* stream);

/* T-LESS evaluation (DESIGN.md section 12): a depth rasterizer standing in for pyrender's DEPTH_ONLY render and the
 * VSD error of src/poses/vsd.py:92-135 (visibility mode "bop19", src/poses/vsd_utils.py).  Both calls refuse bad
 * arguments before any CUDA call and do not synchronise.
 * nope_render_depth: vertices [V, 3] fp32 (model frame, mm), faces [F, 3] int32, poses [P, 4, 4] fp32 row-major (model
 * -> OpenCV camera, mm) -> out [P, H, W] fp32 camera-Z depth, 0 where nothing is hit.  Pixel (r, c) samples the image
 * point (c + 1/2, r + 1/2), u = fx X / Z + cx, v = fy Y / Z + cy.  Coverage is exact (8 sub-pixel bits, int64 edge
 * functions, top-left rule, no culling); the output does not depend on face order or winding.  Faces with an index
 * outside [0, V), a vertex at Z < znear or a projected coordinate beyond 2^20 px are skipped, as are degenerate ones.
 * Requires V, F >= 1, 1 <= P <= 65535, 1 <= H, W <= 8192, znear > 0.
 * nope_vsd_error: depth_test [F, H, W] fp64 (the sensor depth, mm), depth_gt [F, H, W] fp32 (the model rendered at the
 * ground-truth pose), depth_est [F, P, H, W] fp32 (at P estimated poses), K [F, 4] fp64 (fx, fy, cx, cy) -> out [F, P]
 * fp64, (cost + |union| - |inter|) / |union|, 1 where the union is empty.  delta (visibility tolerance, compared in
 * fp32 as numpy compares a float32 array with a Python number) >= 0; tau (misalignment tolerance) > 0; cost_type
 * NOPE_VSD_STEP or NOPE_VSD_TLINEAR.  Requires 1 <= F, P <= 65535, 1 <= H, W <= 8192. */
#define NOPE_VSD_STEP 0      /* cost 1 where |dist_gt - dist_est| >= tau */
#define NOPE_VSD_TLINEAR 1   /* cost min(|dist_gt - dist_est| / tau, 1) */
int nope_render_depth(const float* vertices, int V, const int32_t* faces, int F, const float* poses, int P, float fx,
                      float fy, float cx, float cy, float znear, int H, int W, float* out, void* stream);
int nope_vsd_error(const double* depth_test, const float* depth_gt, const float* depth_est, int F, int P, int H, int W,
                   const double* K, double delta, double tau, int cost_type, double* out, void* stream);

/* Translation from the object mask (DESIGN.md section 18).
 * nope_fit_translation: for F frames and P rotation hypotheses per frame, fit the translation so that the silhouette
 * of the mesh (vertices [V, 3] fp32, faces [NF, 3] int32, as nope_render_depth) lines up with the frame's mask:
 * R [F, P, 9] fp64 row-major and t_init [F, P, 3] fp64 (model -> OpenCV camera, mm), masks [F, H, W] uint8 (nonzero =
 * object), all on the device; K HOST [F, 4] fp64 (fx, fy, cx, cy; finite, fx and fy non-zero), staged in stream order.
 * Each of the `iters` updates renders [R | t] rounded to fp32 with nope_render_depth's rasterizer, scales t's distance
 * by sqrt of the ratio of the silhouette's to the mask's box area and moves the origin so that the box centres meet;
 * an empty silhouette leaves t unchanged.  -> t_out [F, P, 3] fp64, iou [F, P] fp64 = |S n M| / |S u M| of the
 * silhouette S at t_out (0 when S is empty); both NaN for every hypothesis of a frame whose mask is empty.
 * stats_out [F, P, 6] int32 (n_S, |S n M|, row0, row1, col0, col1 of S at t_out; an empty box is (INT_MAX, -1)) may be
 * null.  depth [F P, H, W] fp32 is the caller's workspace; on return it holds nope_render_depth's image at the last
 * rendered translation of each hypothesis.  Requires V, NF >= 1, 1 <= F, P <= 65535, 1 <= H, W <= 8192, iters >= 0,
 * znear finite and > 0.  Refuses bad arguments before any CUDA call; all iterations are enqueued without
 * synchronising the host.  The result does not depend on the batch or on scheduling. */
int nope_fit_translation(const float* vertices, int V, const int32_t* faces, int NF, const double* R,
                         const double* t_init, const uint8_t* masks, const double* K, int F, int P, int H, int W,
                         float znear, int iters, float* depth, double* t_out, double* iou, int32_t* stats_out,
                         void* stream);

/* Pose refinement from the sensor depth (DESIGN.md section 19).
 * nope_refine_depth: projective point-to-plane ICP of P pose hypotheses per frame for F frames against the frame's
 * sensor depth.  Mesh as nope_render_depth; R [F, P, 9] fp64 row-major and t_init [F, P, 3] fp64 (model -> OpenCV
 * camera, mm), depth_sensor [F, H, W] fp64 (mm, 0 = no reading), masks [F, H, W] uint8 (nonzero = object; null: every
 * pixel counts), all on the device; K HOST [F, 4] fp64 (fx, fy, cx, cy; finite, fx and fy non-zero), staged in stream
 * order; rho the largest vertex norm of the mesh (finite, > 0); tau HOST [iters + 1] fp64 the pairing tolerances (mm,
 * each finite and > 0).  Iteration i renders [R | t] rounded to fp32 with nope_render_depth's rasterizer, pairs every
 * interior pixel whose render and its four neighbours are hit, inside the mask, with a sensor reading S and
 * |S - D| <= tau[i], and applies one damped Gauss-Newton step of the point-to-plane distances (rotation about t).
 * -> R_out [F, P, 9], t_out [F, P, 3] fp64 after `iters` steps; fit_out [F, P, 4] fp64 = (n_in, n_valid, rms, score)
 * at the returned pose and tau[iters]: the pairs, the mask pixels with a reading, tau sqrt(sum e^2 / n_in) in mm (NaN
 * when n_in = 0) and n_in / n_valid (NaN when n_valid = 0).  sums_out [F, P, 29] int64 (the fixed-point sums of the
 * last render, units of 2^-32: J J^T upper triangle, J e, e^2, n_in) may be null.  depth [F P, H, W] fp32 is the
 * caller's workspace; on return it holds nope_render_depth's image at the returned pose.  Requires V, NF >= 1,
 * 1 <= F, P <= 65535, 1 <= H, W <= 8192, 0 <= iters <= 1024, znear finite and > 0.  Refuses bad arguments before any
 * CUDA call; all iterations are enqueued without synchronising the host.  The result does not depend on the batch or
 * on scheduling. */
int nope_refine_depth(const float* vertices, int V, const int32_t* faces, int NF, const double* R, const double* t_init,
                      const double* depth_sensor, const uint8_t* masks, const double* K, int F, int P, int H, int W,
                      double rho, const double* tau, int iters, float znear, float* depth, double* R_out,
                      double* t_out, double* fit_out, int64_t* sums_out, void* stream);

/* Pose refinement from the object mask's contour (DESIGN.md section 20).
 * nope_mask_sdf: the signed distance field sdf_out [F, H, W] fp64 of masks [F, H, W] uint8 (nonzero = object), both
 * on the device: sqrt(d2_out) - 1/2 off the object and 1/2 - sqrt(d2_in) on it, with d2_out (d2_in) the exact squared
 * distance in px to the nearest object (background) pixel of the frame; NaN everywhere for a mask that is empty or
 * covers the whole frame.  Requires 1 <= F <= 65535, 1 <= H, W <= 8192.
 * nope_refine_contour: damped Gauss-Newton alignment of the rendered silhouette's contour with the mask, for P pose
 * hypotheses per frame and F frames.  Mesh, R, t_init, K, rho, znear, iters, the workspace depth and sums_out as
 * nope_refine_depth; masks [F, H, W] uint8 on the device; tau HOST [iters + 1] fp64 the pairing tolerances as
 * fractions of the mask's box size sqrt(w h) (each finite and > 0).  Iteration i renders [R | t] rounded to fp32,
 * pairs every interior contour pixel of the render (hit, a 4-neighbour not hit) whose residual phi + 1/2 lies within
 * tau[i] sqrt(w h) px with the mask through its signed distance field phi, and applies one step of the six pose
 * parameters (rotation about t).  A frame whose mask is empty or full keeps every pose.
 * -> R_out [F, P, 9], t_out [F, P, 3] fp64 after `iters` steps; fit_out [F, P, 4] fp64 = (n_in, n_contour, rms, iou)
 * at the returned pose: the pairs at tau[iters], the contour pixels of the render, the RMS residual in px (NaN when
 * n_in = 0) and the silhouette IoU with the mask; rms and iou are NaN for a frame whose mask is empty or full.
 * Refuses bad arguments before any CUDA call; all iterations are enqueued without synchronising the host.  The result
 * does not depend on the batch or on scheduling. */
int nope_mask_sdf(const uint8_t* masks, int F, int H, int W, double* sdf_out, void* stream);
int nope_refine_contour(const float* vertices, int V, const int32_t* faces, int NF, const double* R,
                        const double* t_init, const uint8_t* masks, const double* K, int F, int P, int H, int W,
                        double rho, const double* tau, int iters, float znear, float* depth, double* R_out,
                        double* t_out, double* fit_out, int64_t* sums_out, void* stream);

/* BOP 2019 errors (DESIGN.md section 15).
 * nope_vsd_error_taus: nope_vsd_error at T misalignment tolerances in one pass (the distance images, visibility
 * masks and counts are shared): taus HOST [T] fp64, each finite and > 0, 1 <= T <= 16; K HOST [F, 4] fp64, finite,
 * fx and fy non-zero -> out [F, P, T] fp64; out[f, p, j] equals nope_vsd_error at tau = taus[j] bit for bit.
 * nope_pose_errors: MSSD (mm) and MSPD (px) of P estimated poses per row, minimised over S symmetry transforms:
 * points [V, 3] fp32 (model frame, mm), sym [S, 12], gt [F, 12] and est [F, P, 12] fp64 row-major 3x4 (R | t),
 * K HOST [F, 4] fp64 (fx, fy, cx, cy; finite, fx and fy non-zero) -> out_mssd, out_mspd [F, P] fp64.
 * MSSD = min_s max_x |(R_e x + t_e) - (R_g (R_s x + t_s) + t_g)|, MSPD the same between the projections
 * u = fx X / Z + cx, v = fy Y / Z + cy; a symmetry under which a point has Z <= 0 for either pose counts +inf.
 * Requires V, S >= 1, S <= 2^24, 1 <= F, P <= 65535.  The result does not depend on the launch shape.
 * Both calls refuse bad arguments before any CUDA call, stage K in stream order and do not synchronise. */
int nope_vsd_error_taus(const double* depth_test, const float* depth_gt, const float* depth_est, int F, int P, int H,
                        int W, const double* K, double delta, int cost_type, const double* taus, int T, double* out,
                        void* stream);
int nope_pose_errors(const float* points, int V, const double* sym, int S, const double* gt, const double* est,
                     const double* K, int F, int P, double* out_mssd, double* out_mspd, void* stream);

/* Full-frame crops (DESIGN.md section 13): the virtual-bounding-box crop of src/poses/utils.py:204-272 with the
 * dataloaders' pipeline around it, bit for bit -- PIL's paste onto black through the mask, cv2.warpPerspective
 * (bilinear, constant border 0), ToTensor and x*2-1.
 * frames [F, H, W, C] uint8, C = 3 (RGB) or 4 (RGBA: channel 3 is the mask, and masks must be null); masks [B, H, W]
 * uint8, one per crop, or null (255 everywhere); frame_idx [B] int32, or null when F == B; inv_maps [B, 9] fp64, the
 * destination -> source map (cv2.invert of crop_frame's M, DECOMP_LU) -> out [B, 3, S, S] fp32 in [-1, 1].  A frame
 * index outside [0, F) gives an all -1 crop and reads nothing.  All pointers are device pointers.  Requires F >= 1,
 * 1 <= B <= 65535, 1 <= H, W <= 16384, 1 <= S <= 4096; refuses bad arguments before any CUDA call and does not
 * synchronise. */
int nope_crop_frames(const uint8_t* frames, int F, int H, int W, int C, const uint8_t* masks, const int32_t* frame_idx,
                     const double* inv_maps, int B, int S, float* out, void* stream);

/* Score materialised templates against a query and rank them: the arithmetic of
 * PoseConditional.retrieval (model.py:254-266) after encode_image.
 *   query_feat [B, C, HW] fp32, emb [B, N, C, HW] fp32 -> sim [B, N], topv/topi [B, k]. */
int nope_score_topk(const float* query_feat, const float* emb, int B, int N, int C, int HW,
                    int metric, float occlusion_threshold, int k, float* out_sim, float* out_topv,
                    int64_t* out_topi, int64_t idx_base, void* stream);
/* The same with the reference's broadcasting of query_feat against template_feat (model.py:260-262):
 *   query_feat [B, Q, C, HW] fp32, emb [Bt, N, C, HW] fp32 with Bt = 1 (one template set for every query)
 *   or Bt = B (templates of row b for the Q queries of row b) -> sim [B, Q, N], topv/topi [B, Q, k].
 * No [B*Q, N, C, HW] difference tensor is formed: each template is read once and scored against its queries.
 * nope_score_topk is the Q = 1, Bt = B case. */
int nope_score_topk_multi(const float* query_feat, const float* emb, int B, int Q, int Bt, int N, int C, int HW,
                          int metric, float occlusion_threshold, int k, float* out_sim, float* out_topv,
                          int64_t* out_topi, int64_t idx_base, void* stream);

/* Rank an existing similarity matrix sim [B, N] (used to merge per-GPU shards): top-k per row, descending score,
 * ties (+0 == -0, inf == inf) -> lowest index, NaN after every number and NaNs by index.  Every ranking call below
 * uses this order. */
int nope_topk(float* sim, int B, int N, int k, float* out_topv, int64_t* out_topi,
              int64_t idx_base, void* stream);

/* Distinct pose hypotheses (DESIGN.md section 21): greedy non-maximum suppression of every row of sim [R, N] in the
 * order of nope_topk, modulo each row's symmetry group.  Row r's rotations are rot [G_r, N, 3, 3] fp64 at r / Q (at 0
 * when G_r = 1), object -> camera.  Entries i, j are within theta when c(i, j) >= c_thr = 1 + 2 cos(theta), where c
 * is the largest trace over the group: M_d = D_d Rot_j^T Rot_i, c = max_d tr M_d, or with an axis a,
 * max_d a^T M_d a + sqrt((tr M_d - a^T M_d a)^2 + s^2), s = a . (M32 - M23, M13 - M31, M21 - M12).  The best entry
 * left is taken (ties -> lowest index; -inf and NaN never), everything within theta of it is dropped, k times ->
 * idx_out [R, k] int64, score_out [R, k] fp32, (-1, -inf) where no entry is left.
 * HOST arrays: sym_disc [sum n_disc, 3, 3] fp64 (group g's n_disc[g] rotations in turn, the identity first),
 * n_disc [G] int32 (1..32), axis [G, 3] fp64 (a unit vector, or zeros for none), group [R] int32 (0..G-1).
 * Requires 1 <= k <= 64, -1 <= c_thr <= 3, G_r == 1 or G_r * Q == R.  No host synchronisation. */
int nope_distinct_topk(const float* sim, int R, int N, const double* rot, int G_r, int Q, const double* sym_disc,
                       const int32_t* n_disc, const double* axis, int G, const int32_t* group, int k, double c_thr,
                       int64_t* idx_out, float* score_out, void* stream);

/* Coarse-to-fine pose search (DESIGN.md section 9).  A cell table cells [n_coarse, F] int32 lists, for every
 * pose of a coarse grid, the poses of the next finer grid whose nearest coarse pose it is (ascending, -1 padded,
 * F = the largest cell); cells are disjoint.  Rows r = b * Q + q pair reference b with its query q.
 * nope_pose_cells_expand: the row's keep coarse indices top_idx [R, keep] (int64; entries outside
 * [0, n_coarse) and repeats are skipped) -> out_cand [R, M] int32, the union of their cells in top_idx order
 * (ascending inside a cell, -1 after the last candidate), and out_poses [R, M, 6], those poses gathered from
 * poses [B, n_fine, 6] of reference r / Q.  A padding slot gets the row's first candidate pose.
 * Requires 1 <= keep <= 64, M >= keep * F and R == B * Q.
 * nope_pose_cells_rank: sim [R, M] scored at cand [R, M] -> top-k over the scored candidates (descending, ties ->
 * lowest fine index, NaN last; ranks beyond the candidate count get -inf / -1) as fine indices, and optionally
 * out_sim [R, n_fine]: -inf, with the scored entries scattered in.  Requires 1 <= k <= 64. */
int nope_pose_cells_expand(const int64_t* top_idx, int R, int keep, const int32_t* cells, int n_coarse, int F,
                           const float* poses, int B, int Q, int n_fine, int M,
                           int32_t* out_cand, float* out_poses, void* stream);
int nope_pose_cells_rank(const float* sim, const int32_t* cand, int R, int M, int n_fine, int k,
                         float* out_sim, float* out_topv, int64_t* out_topi, void* stream);

/* Off-grid pose refinement (DESIGN.md section 10).  A candidate is (D, seed): D a 3x3 rotation (float32,
 * row-major), seed an index of the grid all_relativeR [B, N, 6]; its relative rotation is D * S_seed (S_seed: rows
 * 1-2 the grid's 6-D pose, row 3 their cross product).  Rows r = b * Q + q pair reference b with its query q.
 * Products and sums are rounded one by one (no FMA) in a fixed order, so results are bit-reproducible.
 * nope_pose_refine_propose: centres D [R, keep, 9] / seed [R, keep] int32 and stencil [27, 9] (rotation 0 the
 * identity) -> M = keep * 27 candidates per row, slot c * 27 + j = (L_j * D_c, seed_c): out_D [R, M, 9],
 * out_seed [R, M], out_rel [R, M, 9] (D * S_seed) and out_poses [R, M, 6] (its rows 1-2, the sweep's input).
 * A centre whose seed lies outside [0, N) yields 27 padding slots: seed -1, otherwise a copy of the row's first
 * valid candidate.  Requires 1 <= keep <= 64 and R == B * Q.
 * nope_pose_refine_select: sim [R, M] scored at those candidates -> k entries per row, greedily: the highest
 * score first (ties -> lowest slot, NaN after every number), skipping padding and any candidate whose
 * trace(rel_a rel_b^T) exceeds trace_threshold against an entry already chosen.  out_D / out_rel (optional) [R, k, 9], out_seed [R, k],
 * out_score [R, k]; ranks with no candidate left get -inf, seed -1 and zero matrices.
 * Requires 1 <= k <= 64, k <= M <= 64 * 27. */
int nope_pose_refine_propose(const float* D, const int32_t* seed, int R, int keep, const float* all_relativeR,
                             int B, int Q, int N, const float* stencil, float* out_D, int32_t* out_seed,
                             float* out_rel, float* out_poses, void* stream);
int nope_pose_refine_select(const float* sim, const float* cand_D, const int32_t* cand_seed, const float* cand_rel,
                            int R, int M, int k, float trace_threshold, float* out_D, int32_t* out_seed,
                            float* out_score, float* out_rel, void* stream);

/* Joint roll and viewpoint refinement (DESIGN.md section 14).  A candidate is (D, seed, rho), rho = (cos, sin) an
 * fp32 roll: the pose Rz(rho) * D * template_poses[seed], scored as the relative rotation D * S_seed against the
 * query crop rotated by rho.  Same rounding discipline as above.
 * nope_pose_refine_inplane_propose: centres D [R, keep, 9], seed [R, keep] int32, cossin [R, keep, 2]; stencil
 * [9, 9] (rotation 0 the identity) and the roll step (roll_cos, roll_sin).  Pose slots c * 9 + j are those of
 * nope_pose_refine_propose with this stencil (out_D, out_seed, out_rel [R, keep * 9, ...], out_poses [R, keep * 9,
 * 6]); angle slots c * 3 + l (out_cossin [R, keep * 3, 2]) are rho_c for l = 0 (copied bit for bit), rho_c
 * composed with (roll_cos, roll_sin) for l = 1 and with (roll_cos, -roll_sin) for l = 2.  A centre whose seed lies
 * outside [0, N) gives padding pose slots (seed -1) and three copies of the first valid centre's rho.  Requires
 * 1 <= keep <= 16 and R == B * Q.
 * nope_pose_refine_inplane_select: sim [R, keep * 3, keep * 9] scored at the pairs (angle slot a, pose slot p) ->
 * k entries per row, greedily: the highest score first (ties -> lowest a * keep * 9 + p, NaN after every number),
 * skipping pairs with a padding pose slot or angle slot, and any pair whose trace(E E_b^T), E = Rz(rho_a) * rel_p,
 * exceeds trace_threshold against a pair already chosen.  out_D / out_rel (optional) [R, k, 9], out_seed [R, k],
 * out_cossin [R, k, 2], out_aslot [R, k] (the angle slot), out_score [R, k]; ranks with no pair left get -inf,
 * seed and aslot -1 and zeros.  Requires 1 <= keep <= 16, 1 <= k <= 64 and k <= 27 * keep^2.
 * Neither call synchronises; both refuse bad arguments before any CUDA call. */
int nope_pose_refine_inplane_propose(const float* D, const int32_t* seed, const float* cossin, int R, int keep,
                                     const float* all_relativeR, int B, int Q, int N, const float* stencil,
                                     float roll_cos, float roll_sin, float* out_D, int32_t* out_seed, float* out_rel,
                                     float* out_poses, float* out_cossin, void* stream);
int nope_pose_refine_inplane_select(const float* sim, const float* cand_D, const int32_t* cand_seed,
                                    const float* cand_rel, const float* cand_cossin, int R, int keep, int k,
                                    float trace_threshold, float* out_D, int32_t* out_seed, float* out_cossin,
                                    int32_t* out_aslot, float* out_score, float* out_rel, void* stream);

/* Multi-GPU merge (SURVEY.md 8e): each rank sweeps a contiguous slice of the pose grid and contributes
 * ONE packed record to a single all-gather:
 *   [ topv: B*k f32 | 1 pad float if B*k is odd | topi: B*k int64 (GLOBAL indices, -1 = padding) |
 *     similarity slice: B * n_local f32 (optional) | pad to a multiple of 4 floats ]
 * nope_topk_pack_floats gives the record length in floats (n_local_max = ceil(N / world)); records sit back to back
 * in the gathered buffer, so the length keeps every record's int64 block 8-byte aligned.
 * nope_topk_merge turns the `world` gathered records (each pack_floats long) into the global top-k
 * per batch row (descending, ties -> lowest index, NaN last; identical on every rank) and, when has_sim, the
 * full similarity rows [B, N].  Rank r owns poses [r*per, min(N, (r+1)*per)). */
int64_t nope_topk_pack_floats(int B, int k, int n_local_max, int want_sim);
int nope_topk_merge(const float* gathered, int world, int64_t pack_floats, int B, int k, int N, int per,
                    int has_sim, float* out_sim, float* out_topv, int64_t* out_topi, void* stream);

/* ---- per-op entry points (parity tests drive single layers through these) -----------
 * All tensors fp32 NCHW device pointers; conversion to the internal NHWC fp16 layout
 * happens inside.  These calls synchronise the stream before returning.
 * conv: mode 0 = 3x3 pad 1 (model_utils.py:240), 1 = 1x1 (model_utils.py:269),
 *       2 = pixel-unshuffle(2)+1x1 (HardDownsample, model_utils.py:168-172; input is
 *       [n, C0, 2H, 2W], weight [Cout, 4*C0]), 3 = nearest-x2 upsample + 3x3 (HardUpsample,
 *       model_utils.py:161-165; input is [n, C0, H/2, W/2], weight [Cout, C0, 3, 3], folded
 *       inside into four 2x2 parity kernels).  x1 (optional) is concatenated after x0 along
 *       channels (u_net.py:186).  impl must be 2, as in nope_unet_set_conv_impl. */
int nope_op_conv(int impl, int mode, const float* x0, int C0, const float* x1, int C1,
                 const float* weight, const float* bias, float* out, int n_img, int H, int W,
                 int Cout, void* stream);
/* Block.forward (model_utils.py:248-252): [SiLU](GroupNorm_G(conv(x) + bias)), normalised on the host
 * from nothing but the per-(32 pixels, 8 channels) partial sums the plain convolution epilogue writes
 * (the statistics the LDM engine's GroupNorms use).  mode 0..2 as nope_op_conv, impl must be 2. */
int nope_op_conv_gn(int impl, int mode, const float* x0, int C0, const float* x1, int C1,
                    const float* weight, const float* bias, const float* gamma, const float* beta,
                    int G, int silu, float* out, int n_img, int H, int W, int Cout, void* stream);
/* The sweep's fused layer: out = [SiLU](GroupNorm_G(conv(x) + bias)) + chan_bias[n, c] +
 * residual[n / res_div] with everything after the convolution applied in its epilogue
 * (ResnetBlock.forward, model_utils.py:271-279; G = 0: no normalisation).  mode 0..2 as nope_op_conv.
 * precision as nope_unet_set_option.  chan_bias [n, Cout], residual [ceil(n / res_div), Cout, H, W]
 * (res_div 0: one residual image per input image), emit_out (optional) [n, 2] receives the sum and the
 * sum of squares of the stored output (the GroupNorm(1) statistics handed to a following pre-norm). */
int nope_op_conv_gn_fused(int mode, int precision, const float* x0, int C0, const float* x1, int C1,
                          const float* weight, const float* bias, const float* gamma, const float* beta,
                          int G, int silu, const float* chan_bias, const float* residual, int res_div,
                          float* out, float* emit_out, int n_img, int H, int W, int Cout, void* stream);
/* LinearAttention core on qkv [n, 384, H, W] -> [n, 128, H, W] (model_utils.py:403-417).
 * impl 0: wgmma kernel (both contractions on tensor cores, H*W a multiple of 128), 1: CUDA cores. */
int nope_op_linear_attention(int impl, const float* qkv, float* out, int n_img, int H, int W, void* stream);
/* Attention core on qkv [n, 384, H, W] -> [n, 128, H, W], H*W <= 32 (model_utils.py:376-388) */
int nope_op_attention(const float* qkv, float* out, int n_img, int H, int W, void* stream);
/* nearest x2 upsample (model_utils.py:161-163) */
int nope_op_upsample2x(const float* x, float* out, int n_img, int C, int H, int W, void* stream);

/* Debug: run the sweep for B=1 and copy the activation named `tap` (oracle tap names,
 * e.g. "downs.0.0", "mid.1", "ups.2.3", "final_conv.0") to out as fp32 NCHW [N, C, H, W]. */
int nope_unet_debug_tap(nope_unet_t* u, const float* ref_feat, const float* poses, int N,
                        const char* tap, float* out, int64_t out_capacity_floats,
                        int* out_C, int* out_H, void* stream);

/* ---- LDM variant (SURVEY.md 8 f2) ------------------------------------------------------
 * UNetModelPose (src/model/u_net/ldm/adapt_openaimodel.py:14-158 over ldm/openaimodel.py:428-760
 * and ldm/attention.py:149-277; configs/model/vae_cin_ldm.yaml): ResBlocks + SpatialTransformers
 * (self-attention on wgmma, the one-token pose cross-attention folded to a per-hypothesis
 * channel vector, GEGLU feed-forward), strided-conv down / nearest-x2+conv up, emb = 0.
 * Supported configuration: channel_mult (1, 2, 4), 2 ResBlocks per level, attention at every
 * level, num_head_channels 32, transformer_depth 1, injecting_condition_twice false,
 * pose_mlp "single_layer", model_channels a multiple of 256, 32x32 latents.
 * Keys are the reference's state_dict names (628 tensors for model_channels 256; the unused
 * time_embed.* entries are accepted); HOST fp32 pointers, shape-checked.  The VAE encoder
 * (diffusers AutoencoderKL, not part of the reference tree) is out of scope: the sweep takes
 * latents.  Arguments of nope_ldm_sweep are those of nope_unet_sweep with
 * ref_feat / query_feat = [B, latent_ch, 32, 32] latents. */
typedef struct nope_ldm nope_ldm_t;
int nope_ldm_create(nope_ldm_t** out, int model_channels, int context_dim, int latent_ch,
                    int latent_hw, int device);
void nope_ldm_destroy(nope_ldm_t* m);
int nope_ldm_load_tensor(nope_ldm_t* m, const char* key, const float* data, const int64_t* shape,
                         int ndim);
int nope_ldm_finalize(nope_ldm_t* m);
int nope_ldm_set_chunk(nope_ldm_t* m, int hyps_per_chunk);       /* ~15.6 MB workspace / hypothesis (model_channels 256) */
/* conv_impl: 2 = clustered wgmma kernel (the only one; anything else is an error);
 * attn_impl: 0 = wgmma attention (default), 1 = CUDA-core twin (bring-up). */
int nope_ldm_set_impl(nope_ldm_t* m, int conv_impl, int attn_impl);
/* Named options: "hoist" (default 1: the pose-independent prefix -- input conv, first ResBlock,
 * first transformer up to its self-attention -- runs once per reference instead of once per
 * hypothesis); before nope_ldm_finalize only: "precision"
 * (default 0: fp16 weights; 1: exact weights -- packed rows hold [W_hi | W_lo] and every GEMM
 * accumulates A W_hi + A W_lo, 2x the MMA work; embeddings 1.1e-3 -> below the 1e-3 bar against
 * the fp32 reference).  Any other name is an error. */
int nope_ldm_set_option(nope_ldm_t* m, const char* name, int value);
int nope_ldm_sweep(nope_ldm_t* m, const float* ref_latent, const float* poses, int B, int N,
                   const float* query_latent, float* out_emb, float* out_sim, int k,
                   float* out_topv, int64_t* out_topi, int64_t idx_base, void* stream);
/* Q queries per reference, as nope_unet_sweep_multi: query_latent [B, Q, latent_ch, 32, 32], out_sim [B, Q, N],
 * out_topv / out_topi [B, Q, k]; nope_ldm_sweep is the Q = 1 case. */
int nope_ldm_sweep_multi(nope_ldm_t* m, const float* ref_latent, const float* poses, int B, int N,
                         const float* query_latent, int Q, float* out_emb, float* out_sim, int k,
                         float* out_topv, int64_t* out_topi, int64_t idx_base, void* stream);
int64_t nope_ldm_last_launch_count(const nope_ldm_t* m);
/* Profiling hook (bench.py roofline), as nope_unet_profile: CUDA events around every tensor-core
 * GEMM / convolution launch (index 0) and every attention launch (index 1) of later sweeps.
 * nope_ldm_profile_read fills ms[2], flops[2] (algorithmic, 2*M*N*K resp. 4*n^2*C per image),
 * launches[2] and synchronises the device. */
int nope_ldm_profile(nope_ldm_t* m, int enable);
int nope_ldm_profile_read(nope_ldm_t* m, double* ms, double* flops, int64_t* launches);
/* Debug: as nope_unet_debug_tap; tap names follow the reference's module paths
 * ("input_blocks.4.0" = ResBlock output, "input_blocks.4" = block output, "middle_block.1",
 * "output_blocks.2.1", "output_blocks.2", ...). */
int nope_ldm_debug_tap(nope_ldm_t* m, const float* ref_latent, const float* poses, int N,
                       const char* tap, float* out, int64_t out_capacity_floats, int* out_C,
                       int* out_H, void* stream);
/* Debug / parity: run ONE module in isolation on fp32 NCHW device inputs.
 *   name "<prefix>.0" of a ResBlock, "<prefix>.1" of a SpatialTransformer (poses [n, 6] needed),
 *   "input_blocks.<i>.0.op" (Downsample), "output_blocks.<i>.2.conv" (Upsample; S = input side).
 *   x0 [n, C0, S, S], x1 (optional, concatenated after x0) [n, C1, S, S] -> out fp32 NCHW.
 * Synchronises the stream. */
int nope_ldm_run_block(nope_ldm_t* m, const char* name, const float* x0, int C0, const float* x1,
                       int C1, int S, int n, const float* poses, float* out, void* stream);
/* Multi-head self-attention core (ldm/attention.py:177-194, heads of 32 channels):
 * qkv [n_img, n_tok, 3C] fp32 (q | k | v) -> out [n_img, n_tok, C] fp32.  impl as attn_impl. */
int nope_op_mh_attention(int impl, const float* qkv, float* out, int n_img, int n_tok, int C,
                         void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NOPE_B200_H */
