// nope_b200 -- scoring and ranking: the standalone score of materialised templates, and every kernel that ranks
// scores -- top-k, the coarse-to-fine, off-grid and joint roll refinement steps, and the multi-GPU merge.  Every
// greedy selection runs select_rounds, so the ranking order, the "no candidate" sentinel and the top-k limit live
// here once.
#pragma once
#include "common.cuh"

namespace nope {

// The most entries any ranking call selects per row (k, and keep of the coarse-to-fine and off-grid searches):
// select_rounds records every pick in shared memory.  nope_b200/_lib.py MAX_TOPK mirrors it.
constexpr int kMaxTopK = 64;
constexpr int kNoPick = 0x7fffffff;    // "no candidate": a ranking index above every index a row can hold

// Similarity metrics (include/nope_b200.h): 0 the reference's "l2" (model.py:260-262); 1 cosine of the
// flattened C*H*W descriptors (extension, F.cosine_similarity semantics, eps 1e-8); 2 occlusion-aware
// cosine: the per-pixel cosine over channels (the encoder's `sim_distance = nn.CosineSimilarity(dim=1)`,
// template.py:45) with similarities <= threshold zeroed (`OcclusionAwareSimilarity`,
// base_template.py:67-75), averaged over the pixels.
__device__ __forceinline__ float finish_score(int metric, float a, float b, float c, int hw) {
  if (metric == 0) return -a;
  if (metric == 1) return a / (fmaxf(sqrtf(b), 1e-8f) * fmaxf(sqrtf(c), 1e-8f));
  return a / (float)hw;
}

// finish_score over the n visible pixels of hw (DESIGN.md section 27): "l2" -(a f) with f = hw / n rounded once
// (f = 1 with every pixel visible), cosine from its sums over the visible pixels, the occlusion-aware cosine a / n;
// NaN when no pixel is visible.
__device__ __forceinline__ float finish_visible(int metric, float a, float b, float c, int n, int hw) {
  if (n == 0) return __int_as_float(0x7fc00000);
  if (metric == 0) return -(a * __fdiv_rn((float)hw, (float)n));
  if (metric == 1) return finish_score(1, a, b, c, hw);
  return a / (float)n;
}

// Standalone score of materialised embeddings (PoseConditional.retrieval, model.py:254-266):
// emb fp32 [Bt, N, Cl, hw], query rows fp32 [Bt * rows, Cl, hw] -> sim [Bt * rows, N]: query row r is scored
// against the templates of batch r / rows (the reference's broadcasting of query_feat against template_feat).
// metric 0: reference "l2"; 1: cosine over the flattened descriptor; 2: occlusion-aware cosine (extensions).
// One CTA per template (b, n) loops over its query rows: the template is read from DRAM once, and every row's
// sum runs in the same order whatever the number of rows.
// Grouped form (a template bank, DESIGN.md section 25): with slots [G] and row_off [G + 1] (device, both non-null),
// blockIdx.y is a group g that reads template batch slots[g] and scores query rows [row_off[g], row_off[g + 1]);
// `rows` is then unused.  With null pointers group b is template batch b and rows [b * rows, (b + 1) * rows).
// With kVis, query row r scores only the pixels its visible map vis [rows, hw] marks non-zero (finish_visible).
template <bool kVis = false>
__global__ void __launch_bounds__(256)
score_kernel(const float* __restrict__ query, const float* __restrict__ emb,
             float* __restrict__ sim, int N, int Cl, int hw, int metric, float occ_thr, int rows = 1,
             const int* __restrict__ slots = nullptr, const int* __restrict__ row_off = nullptr,
             const uint8_t* __restrict__ vis = nullptr) {
  __shared__ float s_a[2][8], s_b[2][8], s_c[2][8];     // double-buffered across rows
  __shared__ int s_n[2][8];
  const int n = blockIdx.x, b = blockIdx.y;
  const long long tb = slots ? slots[b] : b;
  const long long r0 = row_off ? row_off[b] : (long long)b * rows;
  const int nrows = row_off ? row_off[b + 1] - row_off[b] : rows;
  const float* e = emb + (tb * N + n) * Cl * hw;
  for (int j = 0; j < nrows; ++j) {
    const long long r = r0 + j;
    const float* q = query + r * Cl * hw;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    int nv = 0;
    for (int p = threadIdx.x; p < hw; p += blockDim.x) {
      if (kVis) {
        if (!vis[r * hw + p]) continue;
        ++nv;
      }
      if (metric == 0) {
        float s4 = 0.f;
        for (int c = 0; c < Cl; ++c) {
          const float d = q[c * hw + p] - e[c * hw + p];
          const float d2 = d * d;
          s4 = fmaf(d2, d2, s4);
        }
        a0 += sqrtf(s4);
      } else if (metric == 1) {
        for (int c = 0; c < Cl; ++c) {
          const float x = q[c * hw + p], y = e[c * hw + p];
          a0 = fmaf(x, y, a0);
          a1 = fmaf(x, x, a1);
          a2 = fmaf(y, y, a2);
        }
      } else {
        float qe = 0.f, qq = 0.f, ee = 0.f;
        for (int c = 0; c < Cl; ++c) {
          const float x = q[c * hw + p], y = e[c * hw + p];
          qe = fmaf(x, y, qe);
          qq = fmaf(x, x, qq);
          ee = fmaf(y, y, ee);
        }
        const float sc = qe / (fmaxf(sqrtf(qq), 1e-8f) * fmaxf(sqrtf(ee), 1e-8f));
        a0 += sc > occ_thr ? sc : 0.f;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a0 += __shfl_xor_sync(0xffffffffu, a0, o);
      a1 += __shfl_xor_sync(0xffffffffu, a1, o);
      a2 += __shfl_xor_sync(0xffffffffu, a2, o);
      if (kVis) nv += __shfl_xor_sync(0xffffffffu, nv, o);
    }
    const int buf = j & 1;
    if ((threadIdx.x & 31) == 0) {
      s_a[buf][threadIdx.x >> 5] = a0;
      s_b[buf][threadIdx.x >> 5] = a1;
      s_c[buf][threadIdx.x >> 5] = a2;
      if (kVis) s_n[buf][threadIdx.x >> 5] = nv;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float t0 = 0.f, t1 = 0.f, t2 = 0.f;
      int tn = 0;
      for (int i = 0; i < (int)(blockDim.x >> 5); ++i) {
        t0 += s_a[buf][i]; t1 += s_b[buf][i]; t2 += s_c[buf][i];
        if (kVis) tn += s_n[buf][i];
      }
      sim[r * N + n] = kVis ? finish_visible(metric, t0, t1, t2, tn, hw) : finish_score(metric, t0, t1, t2, hw);
    }
  }
}

// ----------------------------------------------------------------------------
// The order of every ranking kernel: candidate (v, i) ranks before (bv, bi) when v is a number and bv is NaN, or
// both are numbers and v > bv, or v == bv (+0 == -0, inf == inf) and i < bi, or both are NaN and i < bi.  It is
// the order of a stable sort of -score, which the oracles use: descending score, ties -> lowest index, NaN last.
// A total order over distinct indices, so no NaN can stick as a running best or share a rank.
// ----------------------------------------------------------------------------
template <typename I>
__device__ __forceinline__ bool ranks_before(float v, I i, float bv, I bi) {
  const bool vn = isnan(v), bn = isnan(bv);
  if (vn || bn) return !vn || (bn && i < bi);
  return v > bv || (v == bv && i < bi);
}

// Offers candidate (v, i) to a running best (bv, bi) that starts as "no candidate", (-inf, kNoPick).
__device__ __forceinline__ void offer(float v, int i, float& bv, int& bi) {
  if (bi == kNoPick || ranks_before(v, i, bv, bi)) { bv = v; bi = i; }
}

// ----------------------------------------------------------------------------
// CTA-wide arg-max of the per-thread candidates (bv, bi) in the order of ranks_before.  s_v / s_i hold one slot per
// warp.  The result is valid in thread 0 only; the caller synchronises before it reuses s_v / s_i.
// ----------------------------------------------------------------------------
__device__ __forceinline__ void cta_argmax(float& bv, int& bi, float* s_v, int* s_i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (oi != kNoPick) offer(ov, oi, bv, bi);
  }
  if ((threadIdx.x & 31) == 0) { s_v[threadIdx.x >> 5] = bv; s_i[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
      if (s_i[w] != kNoPick) offer(s_v[w], s_i[w], bv, bi);
  }
}

// Shared memory of select_rounds in a CTA of kThreads threads.
template <int kThreads>
struct SelectSmem {
  float v[kThreads / 32];              // cta_argmax's per-warp candidates
  int i[kThreads / 32];
  int pick[kMaxTopK];                  // the pick of every round so far
  float value;                         // the last pick's score
};

// ----------------------------------------------------------------------------
// The greedy selection of every ranking kernel but the merge: k <= kMaxTopK rounds, each of which takes the best
// candidate left in the order of ranks_before.  A pick is the index a candidate ranks by.  The policy `sel` holds what
// differs between the kernels; every thread calls each of its members:
//   sel.scan(t, picks, bv, bi)  offers (offer) this thread's live candidates of round t; picks[0 .. t) are the
//                               earlier picks, so the scan drops what they exclude;
//   sel.take(t, pick, value)    writes rank t;
//   sel.empty(u)                writes rank u when no candidate is left.
// Candidates are only ever removed, so once a round finds none every later round would find none either: the
// remaining ranks are filled with sel.empty at once.
// ----------------------------------------------------------------------------
template <class Sel, int kThreads>
__device__ __forceinline__ void select_rounds(const Sel& sel, int k, SelectSmem<kThreads>& sm) {
  for (int t = 0; t < k; ++t) {
    float bv = -INFINITY;
    int bi = kNoPick;
    sel.scan(t, sm.pick, bv, bi);
    cta_argmax(bv, bi, sm.v, sm.i);
    if (threadIdx.x == 0) { sm.pick[t] = bi; sm.value = bv; }
    __syncthreads();
    const int pick = sm.pick[t];
    if (pick == kNoPick) {
      for (int u = t; u < k; ++u) sel.empty(u);
      return;
    }
    sel.take(t, pick, sm.value);
  }
}

// What a pick of the top-k, cells rank and distinct selections writes: its score and index (+ idx_base); -inf / -1
// for an empty rank.
struct TopkOut {
  float* val;                          // the row's [k] outputs
  long long* idx;
  long long idx_base;

  __device__ __forceinline__ void take(int t, int pick, float value) const {
    if (threadIdx.x == 0) { val[t] = value; idx[t] = (long long)pick + idx_base; }
  }
  __device__ __forceinline__ void empty(int u) const {
    if (threadIdx.x == 0) { val[u] = -INFINITY; idx[u] = -1; }
  }
};

// Top-k of a row against the list of earlier picks (N is unbounded for nope_topk, so a mask would not fit).  Slot m
// ranks by m, or with kCand by the fine pose index cand[m], where cand[m] < 0 is padding.
template <bool kCand>
struct ChosenListSel : TopkOut {
  const float* row;                    // [M]
  const int* cand;                     // [M] with kCand
  int M;

  __device__ __forceinline__ void scan(int t, const int* picks, float& bv, int& bi) const {
    const float* v = row + threadIdx.x;          // walked with m: the loop reloads no row base
    for (int m = threadIdx.x; m < M; m += blockDim.x, v += blockDim.x) {
      const int c = kCand ? cand[m] : m;
      if (kCand && c < 0) continue;
      bool used = false;
#pragma unroll 8
      for (int i = 0; i < t; ++i) used |= (picks[i] == c);
      if (!used) offer(*v, c, bv, bi);
    }
  }
};

// ----------------------------------------------------------------------------
// sim = -(sum of slab partials) and top-k (model.py:265 topk(k=5)); descending score,
// ties -> lowest index, NaN last (ranks_before).  One CTA per row (b, q) of sim [B, Q, N]; partial is
// [B, N, Q, nslab, nparts].
// idx_base is added to the indices so a shard reports global pose indices.  With kVis the partials cover only the
// pixels the row's visible map vis [B * Q, hw] marks non-zero, and the row is finished over their count
// (finish_visible).
// ----------------------------------------------------------------------------
template <bool kVis = false>
__global__ void __launch_bounds__(256)
sim_topk_kernel(const float* __restrict__ partial, int nslab, float* __restrict__ sim, int N,
                int k, float* __restrict__ top_val, long long* __restrict__ top_idx,
                long long idx_base, int nparts = 1, int metric = 0, int hw = 1, int Q = 1,
                const uint8_t* __restrict__ vis = nullptr) {
  pdl_sync();
  __shared__ SelectSmem<256> sm;
  __shared__ int s_nv;
  const int b = blockIdx.x;              // row b * Q + q
  float* srow = sim + (long long)b * N;
  if (partial) {
    const int bb = b / Q, qi = b - bb * Q;
    int nv = 0;
    if (kVis) {                          // the row's visible pixels: an integer sum, so any order gives the same count
      if (threadIdx.x == 0) s_nv = 0;
      __syncthreads();
      for (int p = threadIdx.x; p < hw; p += blockDim.x) nv += vis[(long long)b * hw + p] != 0;
      atomicAdd(&s_nv, nv);
      __syncthreads();
      nv = s_nv;
    }
    for (int n = threadIdx.x; n < N; n += blockDim.x) {
      float t[3] = {0.f, 0.f, 0.f};
      const float* pp = partial + (((long long)bb * N + n) * Q + qi) * nslab * nparts;
      for (int s = 0; s < nslab; ++s)
        for (int q = 0; q < nparts; ++q) t[q] += pp[s * nparts + q];
      srow[n] = kVis ? finish_visible(metric, t[0], t[1], t[2], nv, hw) : finish_score(metric, t[0], t[1], t[2], hw);
    }
    __syncthreads();
  }
  if (k <= 0) return;
  const long long o = (long long)b * k;
  select_rounds(ChosenListSel<false>{{top_val + o, top_idx + o, idx_base}, srow, nullptr, N}, k, sm);
}

// ----------------------------------------------------------------------------
// Coarse-to-fine pose search (DESIGN.md section 9).  A cell table cells [n_coarse, F] lists, for every
// coarse pose, the fine poses nearest to it (ascending, -1 padded); cells are disjoint.
//
// Expand: one CTA per row r = (reference r / Q, query r % Q).  The row's `keep` coarse indices top_idx [R, keep]
// become the union of their cells, in top_idx order and ascending inside a cell: out_cand [R, M] (int32, -1 after
// the last candidate) and the candidates' poses out_poses [R, M, 6] gathered from poses [B, n_fine, 6].  Entries
// outside [0, n_coarse) and repeats of an earlier entry are skipped.  A padding slot carries the row's first
// candidate pose (fine pose 0 if the row has none), so every hypothesis of the launch is a valid rotation.
// ----------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
pose_cells_expand_kernel(const long long* __restrict__ top_idx, int keep, const int* __restrict__ cells,
                         int n_coarse, int F, const float* __restrict__ poses, int Q, int n_fine, int M,
                         int* __restrict__ out_cand, float* __restrict__ out_poses) {
  __shared__ int s_cell[kMaxTopK];         // coarse index of slot j, -1 when skipped
  __shared__ int s_off[kMaxTopK + 1];      // first candidate slot of slot j; s_off[keep] = candidate count
  const int r = blockIdx.x;
  const int b = r / Q;
  const long long* top = top_idx + (long long)r * keep;
  if (threadIdx.x < keep) {
    const int j = threadIdx.x;
    const long long c = top[j];
    bool ok = c >= 0 && c < n_coarse;
    for (int i = 0; i < j && ok; ++i) ok = top[i] != c;
    s_cell[j] = ok ? (int)c : -1;
    int n = 0;
    if (ok)
      while (n < F && cells[c * F + n] >= 0) ++n;
    s_off[j + 1] = n;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    s_off[0] = 0;
    for (int j = 1; j <= keep; ++j) s_off[j] += s_off[j - 1];
  }
  __syncthreads();
  const int total = s_off[keep];
  int first = 0;
  if (total > 0) {
    int j = 0;
    while (s_off[j + 1] == 0) ++j;
    first = cells[s_cell[j] * F];
  }
  const float* pb = poses + (long long)b * n_fine * 6;
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    int fine = -1;
    if (m < total) {
      int j = 0;
      while (s_off[j + 1] <= m) ++j;
      fine = cells[s_cell[j] * F + (m - s_off[j])];
    }
    out_cand[(long long)r * M + m] = fine;
    const float* src = pb + (long long)(fine >= 0 ? fine : first) * 6;
    float* dst = out_poses + ((long long)r * M + m) * 6;
#pragma unroll
    for (int e = 0; e < 6; ++e) dst[e] = src[e];
  }
}

// ----------------------------------------------------------------------------
// Rank one stage of the coarse-to-fine search: one CTA per row of sim [R, M] scored at the fine indices
// cand [R, M] (-1 = padding, not scored; valid entries distinct).  Top-k over the scored candidates only:
// descending score, ties -> lowest FINE index, NaN last; ranks beyond the candidate count get -inf / -1.  out_sim
// (optional) receives the row over the whole fine grid [R, n_fine]: -inf, then the scored entries scattered in.
// ----------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
pose_cells_rank_kernel(const float* __restrict__ sim, const int* __restrict__ cand, int M, int n_fine, int k,
                       float* __restrict__ out_sim, float* __restrict__ top_val, long long* __restrict__ top_idx) {
  __shared__ SelectSmem<256> sm;
  const int r = blockIdx.x;
  const float* srow = sim + (long long)r * M;
  const int* crow = cand + (long long)r * M;
  if (out_sim) {
    float* orow = out_sim + (long long)r * n_fine;
    for (int n = threadIdx.x; n < n_fine; n += blockDim.x) orow[n] = -INFINITY;
    __syncthreads();
    for (int m = threadIdx.x; m < M; m += blockDim.x) {
      const int c = crow[m];
      if (c >= 0) orow[c] = srow[m];
    }
  }
  const long long o = (long long)r * k;
  select_rounds(ChosenListSel<true>{{top_val + o, top_idx + o, 0}, srow, crow, M}, k, sm);
}

// ----------------------------------------------------------------------------
// Off-grid pose refinement (DESIGN.md section 10).  A candidate is (D, seed): D an accumulated 3x3 rotation
// (row-major), seed a grid index; its relative rotation is D * S_seed, where S_seed has rows 1-2 from the grid's
// 6-D pose and row 3 = row 1 x row 2.  Every product and sum is rounded on its own (__fmul_rn / __fadd_rn /
// __fsub_rn, no FMA contraction) in the order written here, which oracle/refine_oracle.py restates op by op:
// the kernels are bit-exact against it.  No sqrt or division: the stencil and the threshold come from the host.
// ----------------------------------------------------------------------------
constexpr int kRefineStencil = 27;                        // the 3x3x3 lattice, identity first
constexpr int kRefineMaxM = kMaxTopK * kRefineStencil;    // keep <= kMaxTopK centres per row

// c = a * b; c[i][j] = (a[i][0] b[0][j] + a[i][1] b[1][j]) + a[i][2] b[2][j]
__device__ __forceinline__ void mat3_mul_rn(const float* a, const float* b, float* c) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      c[i * 3 + j] = __fadd_rn(__fadd_rn(__fmul_rn(a[i * 3], b[j]), __fmul_rn(a[i * 3 + 1], b[3 + j])),
                               __fmul_rn(a[i * 3 + 2], b[6 + j]));
}

// e = Rz(c, s) * x: rows 1-2 mixed by the roll, row 3 copied
__device__ __forceinline__ void rz_mul_rn(float c, float s, const float* x, float* e) {
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    e[j] = __fsub_rn(__fmul_rn(c, x[j]), __fmul_rn(s, x[3 + j]));
    e[3 + j] = __fadd_rn(__fmul_rn(s, x[j]), __fmul_rn(c, x[3 + j]));
    e[6 + j] = x[6 + j];
  }
}

// Propose: one CTA per row r = (reference r / Q, query r % Q).  Centre c (D [R, keep, 9], seed [R, keep]) and
// stencil rotation j (stencil [27, 9], slot 0 the identity) give slot m = c * 27 + j: out_D = L_j * D_c,
// out_seed, out_rel = out_D * S_seed [R, M, 9] and out_poses = its rows 1-2 [R, M, 6], M = keep * 27.  A centre
// whose seed lies outside [0, N) yields 27 padding slots: seed -1 and a copy of the row's first valid candidate
// (slot 0 of its first valid centre; D = I at seed 0 when the row has none), so every hypothesis of the sweep
// is a valid rotation.
// The body of the propose kernels, for a stencil of kS rotations (27 here, 9 for the in-plane variant); returns the
// row's first valid centre (-1 when it has none).
template <int kS>
__device__ __forceinline__ int refine_propose_row(const float* __restrict__ D, const int* __restrict__ seed, int keep,
                                                  const float* __restrict__ rel6, int Q, int N,
                                                  const float* __restrict__ stencil, float* __restrict__ out_D,
                                                  int* __restrict__ out_seed, float* __restrict__ out_rel,
                                                  float* __restrict__ out_poses) {
  const int r = blockIdx.x;
  const int M = keep * kS;
  const float* Drow = D + (long long)r * keep * 9;
  const int* srow = seed + (long long)r * keep;
  const float* pb = rel6 + (long long)(r / Q) * N * 6;
  int first = -1;
  for (int c = 0; c < keep && first < 0; ++c)
    if (srow[c] >= 0 && srow[c] < N) first = c;
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    int c = m / kS, j = m - c * kS;
    int s = srow[c];
    const bool valid = s >= 0 && s < N;
    if (!valid) { c = first; j = 0; }
    float dn[9];
    if (c >= 0) {
      float dc[9], l[9];
      s = srow[c];
#pragma unroll
      for (int e = 0; e < 9; ++e) { dc[e] = Drow[c * 9 + e]; l[e] = stencil[j * 9 + e]; }
      mat3_mul_rn(l, dc, dn);
    } else {
      s = 0;
#pragma unroll
      for (int e = 0; e < 9; ++e) dn[e] = (e % 4 == 0) ? 1.0f : 0.0f;
    }
    float S[9], rel[9];
#pragma unroll
    for (int e = 0; e < 6; ++e) S[e] = pb[(long long)s * 6 + e];
    S[6] = __fsub_rn(__fmul_rn(S[1], S[5]), __fmul_rn(S[2], S[4]));
    S[7] = __fsub_rn(__fmul_rn(S[2], S[3]), __fmul_rn(S[0], S[5]));
    S[8] = __fsub_rn(__fmul_rn(S[0], S[4]), __fmul_rn(S[1], S[3]));
    mat3_mul_rn(dn, S, rel);
    const long long o = (long long)r * M + m;
    out_seed[o] = valid ? s : -1;
#pragma unroll
    for (int e = 0; e < 9; ++e) { out_D[o * 9 + e] = dn[e]; out_rel[o * 9 + e] = rel[e]; }
#pragma unroll
    for (int e = 0; e < 6; ++e) out_poses[o * 6 + e] = rel[e];
  }
  return first;
}

__global__ void __launch_bounds__(256)
pose_refine_propose_kernel(const float* __restrict__ D, const int* __restrict__ seed, int keep,
                           const float* __restrict__ rel6, int Q, int N, const float* __restrict__ stencil,
                           float* __restrict__ out_D, int* __restrict__ out_seed, float* __restrict__ out_rel,
                           float* __restrict__ out_poses) {
  refine_propose_row<kRefineStencil>(D, seed, keep, rel6, Q, N, stencil, out_D, out_seed, out_rel, out_poses);
}

// The policy of both refine selects.  Slot m is candidate m with E_m = rel_m, or with kRoll the pair of angle slot
// a = m / NP and pose slot p = m % NP with E_m = Rz(cs_a) * rel_p.  `dead` marks padding (set by the kernel), picks and
// what a pick suppresses; each round's scan suppresses what lies within thr of the last pick.
template <bool kRoll>
struct TraceSel {
  const float* row;                    // sim [M]
  const float* D;                      // cand_D [NP, 9]
  const int* seed;                     // cand_seed [NP]
  const float* rel;                    // cand_rel [NP, 9]
  const float* cs;                     // cand_cossin [M / NP, 2] with kRoll
  int NP, M;
  float thr;
  unsigned char* dead;                 // [M] in shared memory
  float* out_D;                        // the row's k outputs: out_cossin and out_aslot with kRoll, out_rel optional
  int* out_seed;
  float* out_cossin;
  int* out_aslot;
  float* out_score;
  float* out_rel;

  __device__ __forceinline__ void pose(int m, float* e) const {
    const int a = kRoll ? m / NP : 0;
    const float* x = rel + (m - a * NP) * 9;
    if (kRoll) rz_mul_rn(cs[a * 2], cs[a * 2 + 1], x, e);
    else
#pragma unroll
      for (int i = 0; i < 9; ++i) e[i] = x[i];
  }
  __device__ __forceinline__ void scan(int t, const int* picks, float& bv, int& bi) const {
    const int last = t > 0 ? picks[t - 1] : kNoPick;
    float eb[9];
    if (t > 0) pose(last, eb);
    for (int m = threadIdx.x; m < M; m += blockDim.x) {
      if (dead[m]) continue;
      if (t > 0) {
        float e[9];
        pose(m, e);
        float tr = __fmul_rn(e[0], eb[0]);
#pragma unroll
        for (int i = 1; i < 9; ++i) tr = __fadd_rn(tr, __fmul_rn(e[i], eb[i]));
        if (m == last || tr > thr) { dead[m] = 1; continue; }
      }
      offer(row[m], m, bv, bi);
    }
  }
  __device__ __forceinline__ void take(int t, int pick, float value) const {
    const int a = kRoll ? pick / NP : 0, p = pick - a * NP;
    if (threadIdx.x < 9) {
      out_D[t * 9 + threadIdx.x] = D[p * 9 + threadIdx.x];
      if (out_rel) out_rel[t * 9 + threadIdx.x] = rel[p * 9 + threadIdx.x];
    }
    if (kRoll && threadIdx.x < 2) out_cossin[t * 2 + threadIdx.x] = cs[a * 2 + threadIdx.x];
    if (threadIdx.x == 0) { out_score[t] = value; out_seed[t] = seed[p]; if (kRoll) out_aslot[t] = a; }
  }
  __device__ __forceinline__ void empty(int u) const {
    if (threadIdx.x < 9) {
      out_D[u * 9 + threadIdx.x] = 0.0f;
      if (out_rel) out_rel[u * 9 + threadIdx.x] = 0.0f;
    }
    if (kRoll && threadIdx.x < 2) out_cossin[u * 2 + threadIdx.x] = 0.0f;
    if (threadIdx.x == 0) { out_score[u] = -INFINITY; out_seed[u] = -1; if (kRoll) out_aslot[u] = -1; }
  }
};

// Select: one CTA per row of sim [R, M] scored at the candidates (cand_D / cand_rel [R, M, 9], cand_seed [R, M],
// -1 = padding, never chosen).  Greedy: the highest score first, ties -> lowest slot; a candidate whose
// trace(rel_a rel_b^T) (nine products summed in order) exceeds `thr` for an already chosen b is dropped.  Writes
// k entries of D / rel (optional) [R, k, 9], seed [R, k] and score [R, k]; ranks with no candidate left get
// -inf, seed -1 and zero matrices.
__global__ void __launch_bounds__(256)
pose_refine_select_kernel(const float* __restrict__ sim, const float* __restrict__ cand_D,
                          const int* __restrict__ cand_seed, const float* __restrict__ cand_rel, int M, int k,
                          float thr, float* __restrict__ out_D, int* __restrict__ out_seed,
                          float* __restrict__ out_score, float* __restrict__ out_rel) {
  __shared__ SelectSmem<256> sm;
  __shared__ unsigned char s_dead[kRefineMaxM];
  const long long r = blockIdx.x;
  for (int m = threadIdx.x; m < M; m += blockDim.x) s_dead[m] = cand_seed[r * M + m] < 0;
  __syncthreads();
  select_rounds(TraceSel<false>{sim + r * M, cand_D + r * M * 9, cand_seed + r * M, cand_rel + r * M * 9, nullptr, M, M,
                                thr, s_dead, out_D + r * k * 9, out_seed + r * k, nullptr, nullptr, out_score + r * k,
                                out_rel ? out_rel + r * k * 9 : nullptr},
                k, sm);
}

// ----------------------------------------------------------------------------
// Joint roll and viewpoint refinement (DESIGN.md section 14).  A candidate is (D, seed, rho): D and seed as in the
// off-grid refinement, rho = (cos, sin) a roll; it stands for the pose Rz(rho) * D * template_poses[seed] and is
// scored as the relative rotation D * S_seed against the query crop rotated by rho.  Each centre proposes 9 pose
// slots (an xy stencil about the camera's x and y axes, identity first) and 3 angle slots (rho, rho + phi,
// rho - phi); every (angle slot, pose slot) pair is a hypothesis.  Same rounding discipline as above:
// oracle/inplane_refine_oracle.py restates both kernels op by op.
// ----------------------------------------------------------------------------
constexpr int kInplaneXY = 9;                                           // pose slots per centre
constexpr int kInplaneRoll = 3;                                         // angle slots per centre
constexpr int kInplaneMaxKeep = 16;
constexpr int kInplaneMaxPairs = kInplaneXY * kInplaneRoll * kInplaneMaxKeep * kInplaneMaxKeep;

// Propose: one CTA per row.  Pose slots c * 9 + j exactly as pose_refine_propose_kernel with the 9-rotation
// stencil.  Angle slots c * 3 + l (out_cossin [R, keep * 3, 2]): l = 0 copies rho_c, l = 1 / 2 compose it with
// (roll_c, +roll_s) / (roll_c, -roll_s): (c c' - s s', s c' + c s').  A centre whose seed lies outside [0, N) gives
// three copies of the first valid centre's rho ((1, 0) when the row has none).
__global__ void __launch_bounds__(256)
pose_refine_inplane_propose_kernel(const float* __restrict__ D, const int* __restrict__ seed,
                                   const float* __restrict__ cossin, int keep, const float* __restrict__ rel6, int Q,
                                   int N, const float* __restrict__ stencil, float roll_c, float roll_s,
                                   float* __restrict__ out_D, int* __restrict__ out_seed, float* __restrict__ out_rel,
                                   float* __restrict__ out_poses, float* __restrict__ out_cossin) {
  const int first = refine_propose_row<kInplaneXY>(D, seed, keep, rel6, Q, N, stencil, out_D, out_seed, out_rel,
                                                   out_poses);
  const int r = blockIdx.x;
  const int* srow = seed + (long long)r * keep;
  const float* crow = cossin + (long long)r * keep * 2;
  float* orow = out_cossin + (long long)r * keep * kInplaneRoll * 2;
  for (int m = threadIdx.x; m < keep * kInplaneRoll; m += blockDim.x) {
    int c = m / kInplaneRoll, l = m - c * kInplaneRoll;
    const int s = srow[c];
    if (s < 0 || s >= N) { c = first; l = 0; }
    float oc = 1.0f, os = 0.0f;
    if (c >= 0) {
      const float ca = crow[2 * c], sa = crow[2 * c + 1];
      if (l == 0) {
        oc = ca;
        os = sa;
      } else {
        const float sb = l == 1 ? roll_s : -roll_s;
        oc = __fsub_rn(__fmul_rn(ca, roll_c), __fmul_rn(sa, sb));
        os = __fadd_rn(__fmul_rn(sa, roll_c), __fmul_rn(ca, sb));
      }
    }
    orow[2 * m] = oc;
    orow[2 * m + 1] = os;
  }
}

// Select: one CTA per row of sim [R, keep * 3, keep * 9], pair m = a * (keep * 9) + p of angle slot a and pose slot
// p.  A pair is padding when its pose slot or its angle slot's centre has seed -1.  Greedy: the highest score first,
// ties -> lowest m; a pair is dropped once trace(E_m E_b^T) > thr for a chosen b, E = Rz(rho_a) * rel_p (nine
// products summed in order).  Writes k entries of D / rel (optional) [R, k, 9], seed [R, k], cossin [R, k, 2],
// aslot [R, k] (the winner's angle slot) and score [R, k]; ranks with no pair left get -inf, seed and aslot -1 and
// zeros.
__global__ void __launch_bounds__(256)
pose_refine_inplane_select_kernel(const float* __restrict__ sim, const float* __restrict__ cand_D,
                                  const int* __restrict__ cand_seed, const float* __restrict__ cand_rel,
                                  const float* __restrict__ cand_cossin, int keep, int k, float thr,
                                  float* __restrict__ out_D, int* __restrict__ out_seed,
                                  float* __restrict__ out_cossin, int* __restrict__ out_aslot,
                                  float* __restrict__ out_score, float* __restrict__ out_rel) {
  __shared__ SelectSmem<256> sm;
  __shared__ unsigned char s_dead[kInplaneMaxPairs];
  const long long r = blockIdx.x;
  const int NP = keep * kInplaneXY, NA = keep * kInplaneRoll, M = NA * NP;
  const int* seedrow = cand_seed + r * NP;
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    const int a = m / NP, p = m - a * NP;
    s_dead[m] = seedrow[p] < 0 || seedrow[(a / kInplaneRoll) * kInplaneXY] < 0;
  }
  __syncthreads();
  select_rounds(TraceSel<true>{sim + r * M, cand_D + r * NP * 9, seedrow, cand_rel + r * NP * 9,
                               cand_cossin + r * NA * 2, NP, M, thr, s_dead, out_D + r * k * 9, out_seed + r * k,
                               out_cossin + r * k * 2, out_aslot + r * k, out_score + r * k,
                               out_rel ? out_rel + r * k * 9 : nullptr},
                k, sm);
}

// ----------------------------------------------------------------------------
// Multi-GPU merge (SURVEY.md 8e): every rank contributes ONE packed record to a single all-gather,
//   [ topv: B*k f32 | pad to even | topi: B*k i64 | sim slice: B*n_local f32 (optional) ]      (`pack` floats)
// with GLOBAL pose indices (idx -1 = padding).  This kernel turns the W gathered records into the
// global top-k per batch row (the order of ranks_before: descending score, ties -> lowest index, NaN last;
// deterministic, identical on every rank) and the full similarity rows.  One CTA per batch row; candidates
// W*k <= 1024.  rank r owns poses [r*per, min(N, (r+1)*per)).
// ----------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
topk_merge_kernel(const float* __restrict__ gathered, int world, long long pack, int B, int k, int N, int per,
                  int has_sim, float* __restrict__ out_sim, float* __restrict__ top_val,
                  long long* __restrict__ top_idx) {
  __shared__ float s_v[1024];
  __shared__ long long s_i[1024];
  const int b = blockIdx.x;
  const int kk = (B * k + 1) & ~1;                    // floats before the index block (8-byte aligned)
  const int ncand = world * k;
  for (int c = threadIdx.x; c < ncand; c += blockDim.x) {
    const int r = c / k, j = c - r * k;
    const float* rec = gathered + (long long)r * pack;
    const long long idx = reinterpret_cast<const long long*>(rec + kk)[b * k + j];
    s_i[c] = idx;
    s_v[c] = idx < 0 ? -INFINITY : rec[b * k + j];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < ncand; c += blockDim.x) {
    const float v = s_v[c];
    const long long i = s_i[c];
    if (i < 0) continue;
    int rank = 0;                                     // candidates that beat this one: a permutation of the valid ones
    for (int o = 0; o < ncand; ++o) {
      const long long io = s_i[o];
      if (io < 0 || o == c) continue;
      rank += ranks_before(s_v[o], io, v, i) ? 1 : 0;
    }
    if (rank < k) {
      top_val[(long long)b * k + rank] = v;
      top_idx[(long long)b * k + rank] = i;
    }
  }
  // fewer than k valid candidates (N < k cannot happen: the callers clamp k): nothing to pad
  if (has_sim && out_sim) {
    for (int n = threadIdx.x; n < N; n += blockDim.x) {
      const int r = n / per, j = n - r * per;
      const int lo = r * per, hi = min(N, lo + per);
      const float* rec = gathered + (long long)r * pack + kk + 2 * B * k;
      out_sim[(long long)b * N + n] = rec[(long long)b * (hi - lo) + j];
    }
  }
}

}  // namespace nope
