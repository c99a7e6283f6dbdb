// YOLOX head tail: box decode, SimOTA dynamic-k label assignment and the IoU / BCE losses with their gradients.
//
// Restates YOLOXHead.get_output_and_grid / get_assignments / get_in_boxes_info / dynamic_k_matching / get_losses
// (yolov7/modeling/head/yolox_head.py:226-245, 274-441, 450-669) as batched kernels without per-image host loops,
// host synchronisation or the [G, M, 80] temporary (the reference materialises up to 224 MB per image there).
//
// Arithmetic that decides an index (in-box tests, pairwise IoU, cost ordering) uses explicitly rounded fp32
// operations (__fmul_rn / __fadd_rn / __fdiv_rn) in the reference's evaluation order so that no FMA contraction can
// change a comparison.  Ties in cost are broken towards the lower anchor / lower gt index.
#include <algorithm>

#include "host_common.cuh"
#include "sm90.cuh"

using namespace yb;

namespace {

constexpr int kMaxLevels = 4;
constexpr int kMaxGt = 128;
constexpr int kTopK = 10;

struct Levels {
  int num;
  int h[kMaxLevels], w[kMaxLevels], stride[kMaxLevels], a_off[kMaxLevels + 1];
  int blk_off[kMaxLevels + 1];  // first block of each level when a level is cut into 128-anchor blocks
};

struct Anchor {
  float gx, gy, s;
  int level, pix;
};

__device__ __forceinline__ Anchor anchor_of(const Levels& L, int a) {
  int l = 0;
#pragma unroll
  for (int i = 1; i < kMaxLevels; ++i)
    if (i < L.num && a >= L.a_off[i]) l = i;
  const int r = a - L.a_off[l];
  Anchor an;
  an.level = l;
  an.pix = r;
  an.gx = static_cast<float>(r % L.w[l]);
  an.gy = static_cast<float>(r / L.w[l]);
  an.s = static_cast<float>(L.stride[l]);
  return an;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// ------------------------------------------------------------------------------------------------
// decode (in place on [B, A, 5+C] fp32): xy = (xy + grid) * s, wh = exp(wh) * s; eval additionally sigmoid(obj, cls)
//   yolox_head.py:226-245 (train), 197-224 + 247-272 (eval)
// ------------------------------------------------------------------------------------------------
__global__ void decode_kernel(float* __restrict__ out, int batch, int num_anchors, int ch, Levels L, int eval_mode, float4* __restrict__ raw_reg) {
  pdl_sync();
  const long long total = 1LL * batch * num_anchors;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int a = static_cast<int>(i % num_anchors);
    const Anchor an = anchor_of(L, a);
    float* o = out + i * ch;
    if (raw_reg) raw_reg[i] = make_float4(o[0], o[1], o[2], o[3]);  // origin_preds (yolox_head.py:195): the L1 branch compares the RAW outputs
    o[0] = __fmul_rn(__fadd_rn(o[0], an.gx), an.s);
    o[1] = __fmul_rn(__fadd_rn(o[1], an.gy), an.s);
    o[2] = __fmul_rn(expf(o[2]), an.s);
    o[3] = __fmul_rn(expf(o[3]), an.s);
    if (eval_mode)
      for (int c = 4; c < ch; ++c) o[c] = sigmoidf_(o[c]);
  }
}

// ------------------------------------------------------------------------------------------------
// SimOTA building blocks
// ------------------------------------------------------------------------------------------------
struct Gt {
  float cx, cy, w, h;
  int cls;
};

// labels [B][G][5] = (cls, cx, cy, w, h); the valid rows are the first num_gt ones (yolox_head.py:295, 323-324)
__device__ __forceinline__ Gt load_gt(const float* __restrict__ labels, int b, int gmax, int g) {
  const float* l = labels + (1LL * b * gmax + g) * 5;
  Gt t;
  t.cls = static_cast<int>(l[0]);
  t.cx = l[1]; t.cy = l[2]; t.w = l[3]; t.h = l[4];
  return t;
}

// strict "> 0" tests of get_in_boxes_info (yolox_head.py:599, 623)
__device__ __forceinline__ void in_tests(const Gt& g, float xc, float yc, float s, bool* in_box, bool* in_ctr) {
  const float hw = __fmul_rn(0.5f, g.w), hh = __fmul_rn(0.5f, g.h);
  const float bl = __fsub_rn(xc, __fsub_rn(g.cx, hw)), br = __fsub_rn(__fadd_rn(g.cx, hw), xc);
  const float bt = __fsub_rn(yc, __fsub_rn(g.cy, hh)), bb = __fsub_rn(__fadd_rn(g.cy, hh), yc);
  *in_box = fminf(fminf(bl, bt), fminf(br, bb)) > 0.0f;
  const float r = __fmul_rn(2.5f, s);
  const float cl = __fsub_rn(xc, __fsub_rn(g.cx, r)), cr = __fsub_rn(__fadd_rn(g.cx, r), xc);
  const float ct = __fsub_rn(yc, __fsub_rn(g.cy, r)), cb = __fsub_rn(__fadd_rn(g.cy, r), yc);
  *in_ctr = fminf(fminf(cl, ct), fminf(cr, cb)) > 0.0f;
}

// bboxes_iou(xyxy=False) of boxes.py:57-81 for one pair
__device__ __forceinline__ float pair_iou(const Gt& g, float bx, float by, float bw, float bh) {
  const float tlx = fmaxf(__fsub_rn(g.cx, __fmul_rn(g.w, 0.5f)), __fsub_rn(bx, __fmul_rn(bw, 0.5f)));
  const float tly = fmaxf(__fsub_rn(g.cy, __fmul_rn(g.h, 0.5f)), __fsub_rn(by, __fmul_rn(bh, 0.5f)));
  const float brx = fminf(__fadd_rn(g.cx, __fmul_rn(g.w, 0.5f)), __fadd_rn(bx, __fmul_rn(bw, 0.5f)));
  const float bry = fminf(__fadd_rn(g.cy, __fmul_rn(g.h, 0.5f)), __fadd_rn(by, __fmul_rn(bh, 0.5f)));
  const float area_a = __fmul_rn(g.w, g.h), area_b = __fmul_rn(bw, bh);
  const float en = (tlx < brx && tly < bry) ? 1.f : 0.f;
  const float inter = __fmul_rn(__fmul_rn(__fsub_rn(brx, tlx), __fsub_rn(bry, tly)), en);
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, area_b), inter));
}

__device__ __forceinline__ float neg_log_clamped(float p) { return -fmaxf(logf(p), -100.f); }  // F.binary_cross_entropy clamps log at -100

// cost of (gt, anchor): BCE(sqrt(sig(cls)*sig(obj)), onehot).sum() + 3*(-log(iou+1e-8)) + 1e5*(not in box&centre)
//   s_all = sum_c -log(1 - p_c) over all classes (per anchor), p_gt = p at the gt's class   (yolox_head.py:506-525)
__device__ __forceinline__ float pair_cost(float s_all, float p_gt, float iou, bool in_both) {
  const float cls_cost = __fadd_rn(__fsub_rn(s_all, neg_log_clamped(__fsub_rn(1.f, p_gt))), neg_log_clamped(p_gt));
  const float iou_cost = -logf(__fadd_rn(iou, 1e-8f));
  float c = __fadd_rn(cls_cost, __fmul_rn(3.0f, iou_cost));
  return __fadd_rn(c, in_both ? 0.f : 100000.0f);
}

// ------------------------------------------------------------------------------------------------
// kernel 1: number of gts per image, candidate anchors and their class-cost base
// ------------------------------------------------------------------------------------------------
__global__ void simota_count_gt_kernel(const float* __restrict__ labels, int batch, int gmax, int* __restrict__ num_gt, int* __restrict__ totals) {
  pdl_sync();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b == 0) { totals[0] = 0; totals[1] = 0; }
  if (b >= batch) return;
  int n = 0;
  for (int g = 0; g < gmax; ++g) {
    const float* l = labels + (1LL * b * gmax + g) * 5;
    const float s = ((((l[0] + l[1]) + l[2]) + l[3]) + l[4]);  // label.sum(dim=2) > 0   (yolox_head.py:295)
    n += s > 0.f ? 1 : 0;
  }
  num_gt[b] = n;
}

// contiguous rows of the [B, A, ch] fp32 head output -> shared memory.  Blocks start at multiples of 128 anchors and A * ch * 4 bytes is a
// multiple of 16 for every YOLOX configuration, so the tile is moved in 16-byte vectors when the start address allows it (4x fewer
// load / store instructions than the scalar loop; these kernels are latency-bound, not bandwidth-bound).
__device__ __forceinline__ void load_tile_f32(float* __restrict__ tile, const float* __restrict__ src, int n) {
  if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
    const int n4 = n >> 2;
    const float4* s4 = reinterpret_cast<const float4*>(src);
    float4* t4 = reinterpret_cast<float4*>(tile);
    for (int i = threadIdx.x; i < n4; i += blockDim.x) t4[i] = __ldg(s4 + i);
    for (int i = (n4 << 2) + threadIdx.x; i < n; i += blockDim.x) tile[i] = src[i];
  } else {
    for (int i = threadIdx.x; i < n; i += blockDim.x) tile[i] = src[i];
  }
}

constexpr int kPrepAnchors = 128;

__global__ void __launch_bounds__(kPrepAnchors)
simota_prep_kernel(const float* __restrict__ outputs, const float* __restrict__ labels, const int* __restrict__ num_gt, int num_anchors, int ch,
                   int gmax, Levels L, uint8_t* __restrict__ cand, float* __restrict__ s_all, int* __restrict__ match_count,
                   int* __restrict__ totals) {
  pdl_sync();
  extern __shared__ __align__(16) float tile[];  // [kPrepAnchors][ch]
  __shared__ Gt gts[kMaxGt];
  const int b = blockIdx.y;
  const int a0 = blockIdx.x * kPrepAnchors;
  const int na = min(kPrepAnchors, num_anchors - a0);
  const int ng = num_gt[b];
  if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&totals[1], ng);  // total number of gts
  const int a = a0 + threadIdx.x;
  if (ng == 0) {
    if (threadIdx.x < na) { cand[1LL * b * num_anchors + a] = 0; match_count[1LL * b * num_anchors + a] = 0; }
    return;
  }
  const float* src = outputs + (1LL * b * num_anchors + a0) * ch;
  load_tile_f32(tile, src, na * ch);
  for (int g = threadIdx.x; g < ng; g += blockDim.x) gts[g] = load_gt(labels, b, gmax, g);
  __syncthreads();
  if (threadIdx.x >= na) return;
  const Anchor an = anchor_of(L, a);
  const float xc = __fadd_rn(__fmul_rn(an.gx, an.s), __fmul_rn(0.5f, an.s));
  const float yc = __fadd_rn(__fmul_rn(an.gy, an.s), __fmul_rn(0.5f, an.s));
  bool any = false;
  for (int g = 0; g < ng; ++g) {
    bool ib, ic;
    in_tests(gts[g], xc, yc, an.s, &ib, &ic);
    any = any || ib || ic;
  }
  float s = 0.f;
  if (any) {
    const float* row = tile + threadIdx.x * ch;
    const float so = sigmoidf_(row[4]);
    for (int c = 5; c < ch; ++c) {
      const float p = sqrtf(__fmul_rn(sigmoidf_(row[c]), so));
      s = __fadd_rn(s, neg_log_clamped(__fsub_rn(1.f, p)));
    }
  }
  cand[1LL * b * num_anchors + a] = any ? 1 : 0;
  s_all[1LL * b * num_anchors + a] = s;
  match_count[1LL * b * num_anchors + a] = 0;
}

// ------------------------------------------------------------------------------------------------
// kernel 2: one block per (gt, image): dynamic k from the 10 largest IoUs, then the k cheapest candidates
// ------------------------------------------------------------------------------------------------
constexpr int kMatchThreads = 256;  // (512 threads measured slower: 0.44 vs 0.35 ms for the four SimOTA kernels -- the tournament rounds, not the scan, dominate)

struct CostIdx {
  float c;
  int i;
};
__device__ __forceinline__ bool cost_less(float c1, int i1, float c2, int i2) { return c1 < c2 || (c1 == c2 && i1 < i2); }

__global__ void __launch_bounds__(kMatchThreads)
simota_match_kernel(const float* __restrict__ outputs, const float* __restrict__ labels, const int* __restrict__ num_gt, int num_anchors, int ch,
                    int gmax, Levels L, const uint8_t* __restrict__ cand, const float* __restrict__ s_all, int* __restrict__ match_count,
                    int* __restrict__ matched_gt) {
  pdl_sync();
  const int b = blockIdx.y, g = blockIdx.x;
  if (g >= num_gt[b]) return;
  const Gt gt = load_gt(labels, b, gmax, g);
  const int tid = threadIdx.x;

  float top_iou[kTopK];
  float top_c[kTopK];
  int top_i[kTopK];
#pragma unroll
  for (int k = 0; k < kTopK; ++k) { top_iou[k] = -1.f; top_c[k] = INFINITY; top_i[k] = 0x7fffffff; }
  int my_cands = 0;

  for (int a = tid; a < num_anchors; a += kMatchThreads) {
    if (!cand[1LL * b * num_anchors + a]) continue;
    ++my_cands;
    const float* row = outputs + (1LL * b * num_anchors + a) * ch;
    const Anchor an = anchor_of(L, a);
    const float xc = __fadd_rn(__fmul_rn(an.gx, an.s), __fmul_rn(0.5f, an.s));
    const float yc = __fadd_rn(__fmul_rn(an.gy, an.s), __fmul_rn(0.5f, an.s));
    bool ib, ic;
    in_tests(gt, xc, yc, an.s, &ib, &ic);
    const float iou = pair_iou(gt, row[0], row[1], row[2], row[3]);
    const float p = sqrtf(__fmul_rn(sigmoidf_(row[5 + gt.cls]), sigmoidf_(row[4])));
    const float c = pair_cost(s_all[1LL * b * num_anchors + a], p, iou, ib && ic);
    // insert into the per-thread sorted lists (descending iou / ascending (cost, index))
    if (iou > top_iou[kTopK - 1]) {
      float v = iou;
#pragma unroll
      for (int k = 0; k < kTopK; ++k)
        if (v > top_iou[k]) { const float t = top_iou[k]; top_iou[k] = v; v = t; }
    }
    if (cost_less(c, a, top_c[kTopK - 1], top_i[kTopK - 1])) {
      float vc = c;
      int vi = a;
#pragma unroll
      for (int k = 0; k < kTopK; ++k)
        if (cost_less(vc, vi, top_c[k], top_i[k])) {
          const float tc = top_c[k]; const int ti = top_i[k];
          top_c[k] = vc; top_i[k] = vi; vc = tc; vi = ti;
        }
    }
  }

  // ---- merge: tournament over the threads' sorted heads ----
  __shared__ float s_val[kMatchThreads / 32];
  __shared__ int s_idx[kMatchThreads / 32];
  __shared__ int s_who[kMatchThreads / 32];
  __shared__ float s_bval;
  __shared__ int s_bwho, s_bidx;
  __shared__ int s_ncand;
  if (tid == 0) s_ncand = 0;
  __syncthreads();
  atomicAdd(&s_ncand, my_cands);
  __syncthreads();
  const int ncand = s_ncand;
  const int nk = min(kTopK, ncand);
  const int lane = tid & 31, wid = tid >> 5;

  // (a) sum of the nk largest IoUs, taken in descending order
  float iou_sum = 0.f;
  int head = 0;
  for (int r = 0; r < nk; ++r) {
    float v = -1.f;
#pragma unroll
    for (int k = 0; k < kTopK; ++k) if (k == head) v = top_iou[k];
    if (head >= kTopK) v = -1.f;
    int who = tid;
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, v, off);
      const int ow = __shfl_xor_sync(0xffffffffu, who, off);
      if (ov > v || (ov == v && ow < who)) { v = ov; who = ow; }
    }
    if (lane == 0) { s_val[wid] = v; s_who[wid] = who; }
    __syncthreads();
    if (tid == 0) {
      float bv = s_val[0]; int bw = s_who[0];
      for (int i = 1; i < kMatchThreads / 32; ++i)
        if (s_val[i] > bv || (s_val[i] == bv && s_who[i] < bw)) { bv = s_val[i]; bw = s_who[i]; }
      s_bval = bv; s_bwho = bw;
    }
    __syncthreads();
    if (tid == 0) iou_sum = __fadd_rn(iou_sum, s_bval);
    if (tid == s_bwho) ++head;
    __syncthreads();
  }
  __shared__ int s_k;
  if (tid == 0) {
    int k = static_cast<int>(iou_sum);  // .int() truncation (yolox_head.py:643)
    s_k = k < 1 ? 1 : k;
  }
  __syncthreads();
  const int dyn_k = min(s_k, ncand);

  // (b) the dyn_k smallest (cost, anchor) pairs
  head = 0;
  for (int r = 0; r < dyn_k; ++r) {
    float v = INFINITY;
    int vi = 0x7fffffff;
#pragma unroll
    for (int k = 0; k < kTopK; ++k) if (k == head) { v = top_c[k]; vi = top_i[k]; }
    if (head >= kTopK) { v = INFINITY; vi = 0x7fffffff; }
    int who = tid;
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, v, off);
      const int oi = __shfl_xor_sync(0xffffffffu, vi, off);
      const int ow = __shfl_xor_sync(0xffffffffu, who, off);
      if (cost_less(ov, oi, v, vi)) { v = ov; vi = oi; who = ow; }
    }
    if (lane == 0) { s_val[wid] = v; s_idx[wid] = vi; s_who[wid] = who; }
    __syncthreads();
    if (tid == 0) {
      float bv = s_val[0]; int bi = s_idx[0], bw = s_who[0];
      for (int i = 1; i < kMatchThreads / 32; ++i)
        if (cost_less(s_val[i], s_idx[i], bv, bi)) { bv = s_val[i]; bi = s_idx[i]; bw = s_who[i]; }
      s_bval = bv; s_bidx = bi; s_bwho = bw;
      if (bi != 0x7fffffff) {
        atomicAdd(&match_count[1LL * b * num_anchors + bi], 1);
        matched_gt[1LL * b * num_anchors + bi] = g;  // meaningful only when exactly one gt claims the anchor
      }
    }
    __syncthreads();
    if (tid == s_bwho) ++head;
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// kernel 3: per anchor -- resolve anchors claimed by several gts (argmin of the cost over ALL gts, first index wins:
//   torch.min(cost[:, multi], dim=0), yolox_head.py:653-657) and emit the assignment
// ------------------------------------------------------------------------------------------------
__global__ void simota_resolve_kernel(const float* __restrict__ outputs, const float* __restrict__ labels, const int* __restrict__ num_gt,
                                      int num_anchors, int ch, int gmax, Levels L, const float* __restrict__ s_all,
                                      const int* __restrict__ match_count, int* __restrict__ matched_gt, float* __restrict__ matched_iou,
                                      int* __restrict__ matched_cls, uint8_t* __restrict__ fg_mask, int* __restrict__ num_fg_img,
                                      int* __restrict__ totals) {
  pdl_sync();
  const int b = blockIdx.y;
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  int fg = 0;
  if (a < num_anchors) {
    const long long ia = 1LL * b * num_anchors + a;
    const int ng = num_gt[b];
    const int cnt = ng > 0 ? match_count[ia] : 0;
    int g = -1;
    float iou = 0.f;
    int cls = -1;
    if (cnt > 0) {
      const float* row = outputs + ia * ch;
      g = matched_gt[ia];
      if (cnt > 1) {
        const Anchor an = anchor_of(L, a);
        const float xc = __fadd_rn(__fmul_rn(an.gx, an.s), __fmul_rn(0.5f, an.s));
        const float yc = __fadd_rn(__fmul_rn(an.gy, an.s), __fmul_rn(0.5f, an.s));
        const float so = sigmoidf_(row[4]);
        float best = INFINITY;
        for (int j = 0; j < ng; ++j) {
          const Gt gt = load_gt(labels, b, gmax, j);
          bool ib, ic;
          in_tests(gt, xc, yc, an.s, &ib, &ic);
          const float pi = pair_iou(gt, row[0], row[1], row[2], row[3]);
          const float p = sqrtf(__fmul_rn(sigmoidf_(row[5 + gt.cls]), so));
          const float c = pair_cost(s_all[ia], p, pi, ib && ic);
          if (c < best) { best = c; g = j; }
        }
      }
      const Gt gt = load_gt(labels, b, gmax, g);
      iou = pair_iou(gt, row[0], row[1], row[2], row[3]);
      cls = gt.cls;
      fg = 1;
    }
    matched_gt[ia] = g;
    matched_iou[ia] = iou;
    matched_cls[ia] = cls;
    fg_mask[ia] = static_cast<uint8_t>(fg);
  }
  const unsigned m = __ballot_sync(0xffffffffu, fg);
  if ((threadIdx.x & 31) == 0 && m) {
    const int n = __popc(m);
    atomicAdd(&num_fg_img[b], n);
    atomicAdd(&totals[0], n);
  }
}

// ------------------------------------------------------------------------------------------------
// losses + gradients   (yolox_head.py:412-441; IOUloss boxes.py:125-168; BCEWithLogits)
//   loss_iou = sum_fg (1 - iou^2) / nfg, loss_obj = sum_all bce(obj, fg) / nfg, loss_cls = sum_fg sum_c bce(cls_c, onehot_c * iou) / nfg
//   total = 5*loss_iou + loss_obj + loss_cls.   nfg = max(total foreground count, 1)
// Gradients are taken w.r.t. the RAW head outputs (chain rule through the decode) and written as the bf16 NHWC tensors the
// prediction-conv backward consumes: d_cls [B, H_l, W_l, C] and d_regobj [B, H_l, W_l, 16] (reg 0-3, obj 4, rest 0).
// ------------------------------------------------------------------------------------------------
struct LossOut {
  __nv_bfloat16* d_cls[kMaxLevels];
  __nv_bfloat16* d_ro[kMaxLevels];
  float* d_dense;    // optional fp32 [B, A, 5+C] gradient w.r.t. the raw outputs (tests)
  double* loss_acc;  // [3] sums of iou / obj / cls losses (un-normalised); [4] with the L1 branch
  const float4* raw_reg;  // use_l1: the raw regression outputs [B][A] (origin_preds), else null
  double* bias_acc;  // [levels][5+C] sums of the raw-output gradients (prediction-conv bias gradients), may be null
};

__device__ __forceinline__ float bce_logits(float x, float t) { return fmaxf(x, 0.f) - x * t + log1pf(expf(-fabsf(x))); }

constexpr int kLossAnchors = 128;

__global__ void __launch_bounds__(kLossAnchors)
yolox_loss_kernel(const float* __restrict__ outputs, const float* __restrict__ labels, int num_anchors, int ch, int gmax, Levels L,
                  const uint8_t* __restrict__ fg_mask, const int* __restrict__ matched_gt, const float* __restrict__ matched_iou,
                  const int* __restrict__ matched_cls, const int* __restrict__ totals, const float* __restrict__ weights, LossOut out,
                  int want_loss, int want_grad) {
  pdl_sync();
  extern __shared__ __align__(16) float tile[];  // [kLossAnchors][ch] outputs, reused for gradients
  __shared__ double s_loss[4];
  const int b = blockIdx.y;
  int lvl = 0;  // blocks never straddle levels: each level is cut into its own 128-anchor blocks
#pragma unroll
  for (int i = 1; i < kMaxLevels; ++i)
    if (i < L.num && static_cast<int>(blockIdx.x) >= L.blk_off[i]) lvl = i;
  const int a0 = L.a_off[lvl] + (blockIdx.x - L.blk_off[lvl]) * kLossAnchors;
  const int na = min(kLossAnchors, L.a_off[lvl] + L.h[lvl] * L.w[lvl] - a0);
  const int nc = ch - 5;
  const float nfg = fmaxf(static_cast<float>(totals[0]), 1.f);
  const float w_iou = want_grad ? weights[0] / nfg : 0.f, w_obj = want_grad ? weights[1] / nfg : 0.f, w_cls = want_grad ? weights[2] / nfg : 0.f;
  const float w_l1 = (want_grad && out.raw_reg) ? weights[3] / nfg : 0.f;
  const float* src = outputs + (1LL * b * num_anchors + a0) * ch;
  load_tile_f32(tile, src, na * ch);
  if (threadIdx.x < 4) s_loss[threadIdx.x] = 0.0;
  __syncthreads();

  float l_iou = 0.f, l_obj = 0.f, l_cls = 0.f, l_l1 = 0.f;
  if (threadIdx.x < na) {
    const int a = a0 + threadIdx.x;
    const long long ia = 1LL * b * num_anchors + a;
    float* row = tile + threadIdx.x * ch;
    const bool fg = fg_mask[ia] != 0;
    const float px = row[0], py = row[1], pw = row[2], ph = row[3];
    // objectness: every anchor
    {
      const float x = row[4], t = fg ? 1.f : 0.f;
      l_obj = bce_logits(x, t);
      row[4] = (sigmoidf_(x) - t) * w_obj;
    }
    if (fg) {
      const Gt gt = load_gt(labels, b, gmax, matched_gt[ia]);
      const float miou = matched_iou[ia];
      const int mcls = matched_cls[ia];
      for (int c = 0; c < nc; ++c) {
        const float x = row[5 + c], t = (c == mcls) ? miou : 0.f;
        l_cls += bce_logits(x, t);
        row[5 + c] = (sigmoidf_(x) - t) * w_cls;
      }
      // IOUloss "iou": 1 - iou^2 with iou = I / (Ap + Ag - I + 1e-16)
      const float p_l = px - pw * 0.5f, p_r = px + pw * 0.5f, p_t = py - ph * 0.5f, p_b = py + ph * 0.5f;
      const float g_l = gt.cx - gt.w * 0.5f, g_r = gt.cx + gt.w * 0.5f, g_t = gt.cy - gt.h * 0.5f, g_b = gt.cy + gt.h * 0.5f;
      const float tlx = fmaxf(p_l, g_l), tly = fmaxf(p_t, g_t), brx = fminf(p_r, g_r), bry = fminf(p_b, g_b);
      const float en = (tlx < brx && tly < bry) ? 1.f : 0.f;
      const float iw = brx - tlx, ih = bry - tly;
      const float inter = iw * ih * en;
      const float uni = pw * ph + gt.w * gt.h - inter + 1e-16f;
      const float iou = inter / uni;
      l_iou = 1.f - iou * iou;
      // d loss / d iou = -2 iou;  d iou / d I = (U + I)/U^2;  d iou / d Ap = -I/U^2
      const float dl_diou = -2.f * iou * w_iou;
      const float di = dl_diou * (uni + inter) / (uni * uni);
      const float dap = dl_diou * (-inter) / (uni * uni);
      // sub-gradients of max / min follow torch.max/min(a, b): ties split 0.5 / 0.5
      const float s_tlx = p_l > g_l ? 1.f : (p_l == g_l ? 0.5f : 0.f), s_tly = p_t > g_t ? 1.f : (p_t == g_t ? 0.5f : 0.f);
      const float s_brx = p_r < g_r ? 1.f : (p_r == g_r ? 0.5f : 0.f), s_bry = p_b < g_b ? 1.f : (p_b == g_b ? 0.5f : 0.f);
      const float d_tlx = -ih * en * di * s_tlx, d_brx = ih * en * di * s_brx;
      const float d_tly = -iw * en * di * s_tly, d_bry = iw * en * di * s_bry;
      const float dpx = d_tlx + d_brx, dpy = d_tly + d_bry;
      const float dpw = 0.5f * (d_brx - d_tlx) + dap * ph, dph = 0.5f * (d_bry - d_tly) + dap * pw;
      const Anchor an = anchor_of(L, a);
      row[0] = dpx * an.s;  // x = (raw + grid) * s
      row[1] = dpy * an.s;
      row[2] = dpw * pw;    // w = exp(raw) * s
      row[3] = dph * ph;
      if (out.raw_reg) {
        // L1 branch (yolox_head.py:389-429, 443-448): |raw - target| with target = (gt_xy / s - grid, log(gt_wh / s + 1e-8)); d|x| = sign(x)
        const float4 r = out.raw_reg[ia];
        const float t0 = __fsub_rn(__fdiv_rn(gt.cx, an.s), an.gx), t1 = __fsub_rn(__fdiv_rn(gt.cy, an.s), an.gy);
        const float t2 = logf(__fadd_rn(__fdiv_rn(gt.w, an.s), 1e-8f)), t3 = logf(__fadd_rn(__fdiv_rn(gt.h, an.s), 1e-8f));
        const float e0 = r.x - t0, e1 = r.y - t1, e2 = r.z - t2, e3 = r.w - t3;
        l_l1 = (fabsf(e0) + fabsf(e1)) + (fabsf(e2) + fabsf(e3));
        row[0] += w_l1 * ((e0 > 0.f) - (e0 < 0.f));
        row[1] += w_l1 * ((e1 > 0.f) - (e1 < 0.f));
        row[2] += w_l1 * ((e2 > 0.f) - (e2 < 0.f));
        row[3] += w_l1 * ((e3 > 0.f) - (e3 < 0.f));
      }
    } else {
      row[0] = row[1] = row[2] = row[3] = 0.f;
      for (int c = 0; c < nc; ++c) row[5 + c] = 0.f;
    }
  }
  if (want_loss) {
    atomicAdd(&s_loss[0], static_cast<double>(l_iou));
    atomicAdd(&s_loss[1], static_cast<double>(l_obj));
    atomicAdd(&s_loss[2], static_cast<double>(l_cls));
    if (out.raw_reg) atomicAdd(&s_loss[3], static_cast<double>(l_l1));
  }
  __syncthreads();
  if (want_loss && threadIdx.x < (out.raw_reg ? 4 : 3)) atomicAdd(out.loss_acc + threadIdx.x, s_loss[threadIdx.x]);
  if (!want_grad) return;

  // ---- gradient tile -> global (coalesced) ----
  const long long pix0 = 1LL * b * L.h[lvl] * L.w[lvl] + (a0 - L.a_off[lvl]);
  if (out.d_dense) {
    float* dd = out.d_dense + (1LL * b * num_anchors + a0) * ch;
    for (int i = threadIdx.x; i < na * ch; i += blockDim.x) dd[i] = tile[i];
  }
  if (out.d_cls[lvl]) {
    __nv_bfloat16* dc = out.d_cls[lvl] + pix0 * nc;
    if ((nc & 7) == 0) {  // 16-byte stores of 8 class gradients (rows of nc bf16 start on 16-byte boundaries)
      const int v8 = nc >> 3;
      for (int i = threadIdx.x; i < na * v8; i += blockDim.x) {
        const int r = i / v8, c8 = (i - r * v8) * 8;
        const float* t = tile + r * ch + 5 + c8;
        uint4 u;
        u.x = pack_bf16x2(t[0], t[1]); u.y = pack_bf16x2(t[2], t[3]); u.z = pack_bf16x2(t[4], t[5]); u.w = pack_bf16x2(t[6], t[7]);
        *reinterpret_cast<uint4*>(dc + static_cast<size_t>(r) * nc + c8) = u;
      }
    } else {
      for (int i = threadIdx.x; i < na * nc; i += blockDim.x) dc[i] = __float2bfloat16_rn(tile[(i / nc) * ch + 5 + i % nc]);
    }
    __nv_bfloat16* dr = out.d_ro[lvl] + pix0 * 16;
    for (int i = threadIdx.x; i < na * 2; i += blockDim.x) {  // 16 padded reg+obj channels per anchor = two 16-byte stores
      const int r = i >> 1;
      const float* t = tile + r * ch;
      uint4 u = make_uint4(0u, 0u, 0u, 0u);
      if ((i & 1) == 0) { u.x = pack_bf16x2(t[0], t[1]); u.y = pack_bf16x2(t[2], t[3]); u.z = pack_bf16x2(t[4], 0.f); }
      *reinterpret_cast<uint4*>(dr + static_cast<size_t>(i) * 8) = u;
    }
  }
  if (out.bias_acc) {
    for (int c = threadIdx.x; c < ch; c += blockDim.x) {
      float s = 0.f;
      for (int r = 0; r < na; ++r) s += tile[r * ch + c];
      if (s != 0.f) atomicAdd(out.bias_acc + lvl * ch + c, static_cast<double>(s));
    }
  }
}

// (total, 5*iou, obj, cls, l1 = 0, num_fg / max(num_gts, 1))  --  the 6-tuple get_losses returns (yolox_head.py:433-441)
__global__ void yolox_loss_finish_kernel(double* __restrict__ loss_acc, const int* __restrict__ totals, float* __restrict__ out6, int with_l1) {
  pdl_sync();
  const float nfg = fmaxf(static_cast<float>(totals[0]), 1.f);
  const float li = static_cast<float>(loss_acc[0]) / nfg, lo = static_cast<float>(loss_acc[1]) / nfg, lc = static_cast<float>(loss_acc[2]) / nfg;
  const float l1 = with_l1 ? static_cast<float>(loss_acc[3]) / nfg : 0.f;
  out6[0] = 5.f * li + lo + lc + l1;  // reg_weight * loss_iou + loss_obj + loss_cls + loss_l1 (yolox_head.py:431-432)
  out6[1] = 5.f * li;
  out6[2] = lo;
  out6[3] = lc;
  out6[4] = l1;
  out6[5] = nfg / fmaxf(static_cast<float>(totals[1]), 1.f);
  loss_acc[0] = loss_acc[1] = loss_acc[2] = 0.0;
  if (with_l1) loss_acc[3] = 0.0;
}

int make_levels(const int32_t* level_hw_stride, int num_levels, int num_anchors, Levels* L) {
  YB_REQUIRE(level_hw_stride && num_levels > 0 && num_levels <= kMaxLevels, YB200_ERR_INVALID, "bad level table (num_levels=%d)", num_levels);
  L->num = num_levels;
  int off = 0, blk = 0;
  for (int i = 0; i < kMaxLevels; ++i) {
    L->blk_off[i] = blk;
    if (i < num_levels) {
      L->h[i] = level_hw_stride[3 * i]; L->w[i] = level_hw_stride[3 * i + 1]; L->stride[i] = level_hw_stride[3 * i + 2];
      YB_REQUIRE(L->h[i] > 0 && L->w[i] > 0 && L->stride[i] > 0, YB200_ERR_INVALID, "bad level %d", i);
      L->a_off[i] = off;
      off += L->h[i] * L->w[i];
      blk += (L->h[i] * L->w[i] + 127) / 128;
    } else {
      L->h[i] = L->w[i] = L->stride[i] = 1;
      L->a_off[i] = 0x7fffffff;
    }
  }
  L->a_off[kMaxLevels] = off;
  L->blk_off[kMaxLevels] = blk;
  YB_REQUIRE(off == num_anchors, YB200_ERR_INVALID, "levels cover %d anchors, tensor has %d", off, num_anchors);
  return 0;
}

}  // namespace

// ================================================================================================
// C ABI
// ================================================================================================
static int decode_impl(float* outputs, int batch, int num_anchors, int channels, const int32_t* level_hw_stride, int num_levels, int eval_mode,
                       float* raw_reg, void* stream);
extern "C" int yb200_yolox_decode(float* outputs, int batch, int num_anchors, int channels, const int32_t* level_hw_stride, int num_levels,
                                  int eval_mode, void* stream) {
  return decode_impl(outputs, batch, num_anchors, channels, level_hw_stride, num_levels, eval_mode, nullptr, stream);
}
extern "C" int yb200_yolox_decode_keep_raw(float* outputs, int batch, int num_anchors, int channels, const int32_t* level_hw_stride, int num_levels,
                                           float* raw_reg, void* stream) {
  YB_REQUIRE(raw_reg != nullptr && (reinterpret_cast<uintptr_t>(raw_reg) & 15) == 0, YB200_ERR_INVALID, "yolox_decode_keep_raw: raw_reg must be a 16-byte aligned [B][A][4] buffer");
  return decode_impl(outputs, batch, num_anchors, channels, level_hw_stride, num_levels, 0, raw_reg, stream);
}
static int decode_impl(float* outputs, int batch, int num_anchors, int channels, const int32_t* level_hw_stride, int num_levels, int eval_mode,
                       float* raw_reg, void* stream) {
  YB_REQUIRE(outputs && batch > 0 && num_anchors > 0 && channels > 5, YB200_ERR_INVALID, "yolox_decode: bad arguments");
  Levels L;
  int rc = make_levels(level_hw_stride, num_levels, num_anchors, &L);
  if (rc) return rc;
  const long long total = 1LL * batch * num_anchors;
  const int blocks = static_cast<int>(std::min<long long>((total + 127) / 128, 16LL * sm_count()));
  launch_k(decode_kernel, blocks, 128, 0, as_stream(stream), outputs, batch, num_anchors, channels, L, eval_mode, reinterpret_cast<float4*>(raw_reg));
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int64_t yb200_simota_workspace(int batch, int num_anchors) {
  if (batch <= 0 || num_anchors <= 0) return YB200_ERR_INVALID;
  const int64_t ba = 1LL * batch * num_anchors;
  // cand (u8) + s_all (f32) + match_count (i32), each padded to 256 B
  auto pad = [](int64_t v) { return (v + 255) / 256 * 256; };
  return pad(ba) + pad(4 * ba) + pad(4 * ba) + 256;
}

extern "C" int yb200_simota_assign(const float* outputs, const float* labels, int batch, int num_anchors, int channels, int max_gt,
                                   const int32_t* level_hw_stride, int num_levels, void* workspace, int32_t* num_gt, uint8_t* fg_mask,
                                   int32_t* matched_gt, float* matched_iou, int32_t* matched_cls, int32_t* num_fg_img, int32_t* totals,
                                   void* stream) {
  YB_REQUIRE(outputs && labels && workspace && num_gt && fg_mask && matched_gt && matched_iou && matched_cls && num_fg_img && totals,
             YB200_ERR_INVALID, "simota_assign: null pointer");
  YB_REQUIRE(batch > 0 && num_anchors > 0 && channels > 5 && max_gt > 0 && max_gt <= kMaxGt, YB200_ERR_INVALID,
             "simota_assign: batch=%d anchors=%d channels=%d max_gt=%d (limit %d)", batch, num_anchors, channels, max_gt, kMaxGt);
  Levels L;
  int rc = make_levels(level_hw_stride, num_levels, num_anchors, &L);
  if (rc) return rc;
  cudaStream_t st = as_stream(stream);
  const int64_t ba = 1LL * batch * num_anchors;
  auto pad = [](int64_t v) { return (v + 255) / 256 * 256; };
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  uint8_t* cand = ws;
  float* s_all = reinterpret_cast<float*>(ws + pad(ba));
  int* match_count = reinterpret_cast<int*>(ws + pad(ba) + pad(4 * ba));
  YB_CHECK_CUDA(cudaMemsetAsync(num_fg_img, 0, sizeof(int) * batch, st));
  launch_k(simota_count_gt_kernel, ceil_div(batch, 64), 64, 0, st, labels, batch, max_gt, num_gt, totals);
  YB_CHECK_CUDA(cudaGetLastError());
  const size_t tile = static_cast<size_t>(kPrepAnchors) * channels * sizeof(float);
  static PerDevice<int> smem_limit(0);
  YB_CHECK_CUDA(raise_smem_limit(smem_limit, static_cast<int>(tile), simota_prep_kernel));
  launch_k(simota_prep_kernel, dim3(ceil_div(num_anchors, kPrepAnchors), batch), kPrepAnchors, tile, st, outputs, labels, num_gt, num_anchors, channels,
                                                                                                  max_gt, L, cand, s_all, match_count, totals);
  YB_CHECK_CUDA(cudaGetLastError());
  launch_k(simota_match_kernel, dim3(max_gt, batch), kMatchThreads, 0, st, outputs, labels, num_gt, num_anchors, channels, max_gt, L, cand, s_all,
                                                                     match_count, matched_gt);
  YB_CHECK_CUDA(cudaGetLastError());
  launch_k(simota_resolve_kernel, dim3(ceil_div(num_anchors, 128), batch), 128, 0, st, outputs, labels, num_gt, num_anchors, channels, max_gt, L, s_all,
                                                                                 match_count, matched_gt, matched_iou, matched_cls, fg_mask,
                                                                                 num_fg_img, totals);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

static int yolox_loss_impl(const float* outputs, const float* labels, int batch, int num_anchors, int channels, int max_gt,
                           const int32_t* level_hw_stride, int num_levels, const uint8_t* fg_mask, const int32_t* matched_gt,
                           const float* matched_iou, const int32_t* matched_cls, const int32_t* totals, const float* weights3,
                           double* loss_acc3, float* losses6, void* const* d_cls, void* const* d_regobj, float* d_dense, double* bias_acc,
                           const float* raw_reg, void* stream);
extern "C" int yb200_yolox_loss(const float* outputs, const float* labels, int batch, int num_anchors, int channels, int max_gt,
                                const int32_t* level_hw_stride, int num_levels, const uint8_t* fg_mask, const int32_t* matched_gt,
                                const float* matched_iou, const int32_t* matched_cls, const int32_t* totals, const float* weights3,
                                double* loss_acc3, float* losses6, void* const* d_cls, void* const* d_regobj, float* d_dense, double* bias_acc,
                                void* stream) {
  return yolox_loss_impl(outputs, labels, batch, num_anchors, channels, max_gt, level_hw_stride, num_levels, fg_mask, matched_gt, matched_iou, matched_cls,
                         totals, weights3, loss_acc3, losses6, d_cls, d_regobj, d_dense, bias_acc, nullptr, stream);
}
extern "C" int yb200_yolox_loss_l1(const float* outputs, const float* raw_reg, const float* labels, int batch, int num_anchors, int channels, int max_gt,
                                   const int32_t* level_hw_stride, int num_levels, const uint8_t* fg_mask, const int32_t* matched_gt,
                                   const float* matched_iou, const int32_t* matched_cls, const int32_t* totals, const float* weights4,
                                   double* loss_acc4, float* losses6, void* const* d_cls, void* const* d_regobj, float* d_dense, double* bias_acc,
                                   void* stream) {
  YB_REQUIRE(raw_reg != nullptr && (reinterpret_cast<uintptr_t>(raw_reg) & 15) == 0, YB200_ERR_INVALID, "yolox_loss_l1: raw_reg must be a 16-byte aligned [B][A][4] buffer");
  return yolox_loss_impl(outputs, labels, batch, num_anchors, channels, max_gt, level_hw_stride, num_levels, fg_mask, matched_gt, matched_iou, matched_cls,
                         totals, weights4, loss_acc4, losses6, d_cls, d_regobj, d_dense, bias_acc, raw_reg, stream);
}
static int yolox_loss_impl(const float* outputs, const float* labels, int batch, int num_anchors, int channels, int max_gt,
                           const int32_t* level_hw_stride, int num_levels, const uint8_t* fg_mask, const int32_t* matched_gt,
                           const float* matched_iou, const int32_t* matched_cls, const int32_t* totals, const float* weights3,
                           double* loss_acc3, float* losses6, void* const* d_cls, void* const* d_regobj, float* d_dense, double* bias_acc,
                           const float* raw_reg, void* stream) {
  YB_REQUIRE(outputs && labels && fg_mask && matched_gt && matched_iou && matched_cls && totals && loss_acc3, YB200_ERR_INVALID,
             "yolox_loss: null pointer");
  const bool want_loss = losses6 != nullptr;
  const bool want_grad = weights3 != nullptr;
  YB_REQUIRE(want_loss || want_grad, YB200_ERR_INVALID, "yolox_loss: nothing to compute");
  YB_REQUIRE(!want_grad || d_dense || (d_cls && d_regobj), YB200_ERR_INVALID, "yolox_loss: gradient requested without an output buffer");
  Levels L;
  int rc = make_levels(level_hw_stride, num_levels, num_anchors, &L);
  if (rc) return rc;
  LossOut out;
  memset(&out, 0, sizeof(out));
  for (int i = 0; i < num_levels; ++i) {
    out.d_cls[i] = want_grad && d_cls ? static_cast<__nv_bfloat16*>(d_cls[i]) : nullptr;
    out.d_ro[i] = want_grad && d_regobj ? static_cast<__nv_bfloat16*>(d_regobj[i]) : nullptr;
    YB_REQUIRE((out.d_cls[i] == nullptr) == (out.d_ro[i] == nullptr), YB200_ERR_INVALID, "yolox_loss: d_cls / d_regobj must come in pairs");
  }
  out.d_dense = want_grad ? d_dense : nullptr;
  out.loss_acc = loss_acc3;
  out.raw_reg = reinterpret_cast<const float4*>(raw_reg);
  out.bias_acc = want_grad ? bias_acc : nullptr;
  cudaStream_t st = as_stream(stream);
  const size_t tile = static_cast<size_t>(kLossAnchors) * channels * sizeof(float);
  static PerDevice<int> smem_limit(0);
  YB_CHECK_CUDA(raise_smem_limit(smem_limit, static_cast<int>(tile), yolox_loss_kernel));
  static_assert(kLossAnchors == 128, "Levels::blk_off assumes 128-anchor blocks");
  launch_k(yolox_loss_kernel, dim3(L.blk_off[kMaxLevels], batch), kLossAnchors, tile, st, 
      outputs, labels, num_anchors, channels, max_gt, L, fg_mask, matched_gt, matched_iou, matched_cls, totals, weights3, out, want_loss, want_grad);
  YB_CHECK_CUDA(cudaGetLastError());
  if (want_loss) {
    launch_k(yolox_loss_finish_kernel, 1, 1, 0, st, loss_acc3, totals, losses6, raw_reg != nullptr ? 1 : 0);
    YB_CHECK_CUDA(cudaGetLastError());
  }
  return 0;
}

// sum over anchors of the raw-output gradients = bias gradients of cls_preds / reg_preds / obj_preds (yolox_head.py:103-129)
__global__ void head_bias_grad_kernel(double* __restrict__ bias_acc, int num_levels, int ch, float* __restrict__ g_reg, float* __restrict__ g_obj,
                                      float* __restrict__ g_cls, int level, int accumulate) {
  pdl_sync();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= ch) return;
  const float v = static_cast<float>(bias_acc[level * ch + c]);
  float* d = c < 4 ? g_reg + c : (c == 4 ? g_obj : g_cls + (c - 5));
  *d = accumulate ? (*d + v) : v;
  bias_acc[level * ch + c] = 0.0;
}

extern "C" int yb200_head_bias_grad(double* bias_acc, int num_levels, int channels, int level, float* grad_reg_bias4, float* grad_obj_bias1,
                                    float* grad_cls_bias, int accumulate, void* stream) {
  YB_REQUIRE(bias_acc && grad_reg_bias4 && grad_obj_bias1 && grad_cls_bias && level >= 0 && level < num_levels && channels > 5, YB200_ERR_INVALID,
             "head_bias_grad: bad arguments");
  launch_k(head_bias_grad_kernel, ceil_div(channels, 128), 128, 0, as_stream(stream), bias_acc, num_levels, channels, grad_reg_bias4, grad_obj_bias1,
                                                                               grad_cls_bias, level, accumulate);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
