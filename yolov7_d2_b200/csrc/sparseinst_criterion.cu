// SparseInst's matcher and criterion (yolov7/modeling/loss/sparseinst_loss.py):
//   yb200_sparseinst_target_masks  nested_masks_from_list(..., input_shape) + F.interpolate(bilinear, align_corners=False) (:135-154, :320-331)
//                                  of every ground-truth mask, plus its Σt²; the zero padding is never materialised
//   yb200_sparseinst_match_cost    SparseInstMatcher's C = dice^α · σ(logit[label])^β (:336-340), only the per-image blocks
//   yb200_sparseinst_set_loss      loss_labels (sigmoid focal loss, :89-122) and loss_masks_with_iou_objectness (:124-184), weighted
//   yb200_sparseinst_set_loss_bwd  their gradient w.r.t. pred_logits, pred_masks and pred_scores
// Inputs are fp32 pred_logits [B][N][K], pred_masks [B][N][HW], pred_scores [B][N].  The targets of the batch are packed: labels [G], per-image
// offsets [B+1], the resized masks [G][HW] with Σt² [G].  Every sum runs in a fixed order (per-thread strides, warp butterflies, then warp
// partials in warp order): identical calls are bit-identical.
#include <math.h>

#include "host_common.cuh"
#include "sm90.cuh"

using namespace yb;

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kQT = 8;          // query rows per cost block: each target chunk read from L2 serves 8 rows
constexpr int kChunk = 1024;    // pixels of the 8 rows staged as σ(m) in shared memory
constexpr int kBwdPix = 2048;   // pixels per backward block
constexpr int kMaxQueries = 4096;
constexpr int kSave = 8;        // per-row sums kept for the backward (see pair_sums_kernel)
constexpr float kAlpha = 0.25f;  // sigmoid_focal_loss_jit(alpha=0.25, gamma=2) (:112-118)

__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}

// the block's sum in a fixed order, returned to every thread; red holds kWarps floats
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();  // the previous call's readers are done with red
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  for (int i = 0; i < kWarps; ++i) s += red[i];
  return s;
}

__device__ __forceinline__ float sigmoid(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float softplus(float z) { return fmaxf(z, 0.f) + log1pf(expf(-fabsf(z))); }
// F.binary_cross_entropy_with_logits of one element
__device__ __forceinline__ float bce_logits(float x, float t) { return fmaxf(x, 0.f) - x * t + log1pf(expf(-fabsf(x))); }

// fvcore's sigmoid focal loss of one element, ce · (1 - p_t)^2 · α_t, written with z = (target ? -x : x): ce = softplus(z), 1 - p_t = σ(z)
__device__ __forceinline__ float focal(float x, bool pos) {
  const float z = pos ? -x : x, s = sigmoid(z);
  return (pos ? kAlpha : 1.f - kAlpha) * (softplus(z) * (s * s));
}
// its derivative w.r.t. x: d/dz = α_t σ(z)² (2 (1 - σ(z)) softplus(z) + σ(z))
__device__ __forceinline__ float focal_grad(float x, bool pos) {
  const float z = pos ? -x : x, s = sigmoid(z);
  const float d = (pos ? kAlpha : 1.f - kAlpha) * s * s * (2.f * (1.f - s) * softplus(z) + s);
  return pos ? -d : d;
}

// ATen's bilinear source index and weights (align_corners = False, no scale factor): scale = in / out, src = max(scale (dst + 0.5) - 0.5, 0),
// i0 = min(floor(src), in - 1), λ1 = clamp(src - i0, 0, 1), λ0 = 1 - λ1.  Torch's CPU build evaluates src as one fused multiply-add (without it,
// F.interpolate differs by up to 3.5e-6 on 0/1/2-valued masks); everything else is explicitly rounded, with no contraction.  At in = 4 out (the
// model) every step is exact, so the result equals F.interpolate bit for bit.
struct Tap {
  int i0, i1;
  float l0, l1;
};
__device__ __forceinline__ Tap src_tap(int dst, int in, float scale) {
  float src = __fmaf_rn(scale, __fadd_rn((float)dst, 0.5f), -0.5f);
  src = src < 0.f ? 0.f : src;
  const int i0 = min((int)floorf(src), in - 1);
  const float l1 = fminf(fmaxf(__fsub_rn(src, (float)i0), 0.f), 1.f);
  return Tap{i0, i0 < in - 1 ? i0 + 1 : i0, __fsub_rn(1.f, l1), l1};
}

// one block per target: out[g] = the mask zero-padded to in_h x in_w, resized to H x W; tsq[g] = Σ out²
__global__ void __launch_bounds__(kThreads) target_masks_kernel(const uint8_t* __restrict__ masks, const int64_t* __restrict__ table, int in_h,
                                                                 int in_w, int H, int W, float* __restrict__ out, float* __restrict__ tsq) {
  pdl_sync();
  __shared__ float red[kWarps];
  const int g = blockIdx.x;
  const int64_t off = table[3 * g];
  const int h = (int)table[3 * g + 1], w = (int)table[3 * g + 2];
  const uint8_t* m = masks + off;
  const float sh = (float)in_h / (float)H, sw = (float)in_w / (float)W;
  auto at = [&](int y, int x) { return (y < h && x < w) ? (float)m[(size_t)y * w + x] : 0.f; };
  float* o = out + (size_t)g * H * W;
  float sq = 0.f;
  for (int p = threadIdx.x; p < H * W; p += kThreads) {
    const Tap ty = src_tap(p / W, in_h, sh), tx = src_tap(p % W, in_w, sw);
    // ATen's combination order: rows first along W, then the two rows weighted along H
    const float r0 = __fadd_rn(__fmul_rn(at(ty.i0, tx.i0), tx.l0), __fmul_rn(at(ty.i0, tx.i1), tx.l1));
    const float r1 = __fadd_rn(__fmul_rn(at(ty.i1, tx.i0), tx.l0), __fmul_rn(at(ty.i1, tx.i1), tx.l1));
    const float v = __fadd_rn(__fmul_rn(r0, ty.l0), __fmul_rn(r1, ty.l1));
    o[p] = v;
    sq += v * v;
  }
  sq = block_sum(sq, red);
  if (threadIdx.x == 0) tsq[g] = sq;
}

// block (n-tile, b): C[b][n][j] = (2 Σσ(m)t / (Σσ(m)² + Σt² + 1e-4))^α · σ(logit[b, n, label_j])^β for kQT query rows n and every target j of
// image b, written at cost + N*offsets[b] + n*G_b + j.  The rows' logits are read once; σ is staged in shared memory per kChunk pixels and the
// target rows stream from L2.  Block (0, 0) also writes the status word at cost[N*G]: bit 0 a label outside [0, K), bit 1 an image with more
// targets than queries.
__global__ void __launch_bounds__(kThreads) match_cost_kernel(const float* __restrict__ logits, const float* __restrict__ masks,
                                                               const int* __restrict__ labels, const int* __restrict__ img_off,
                                                               const float* __restrict__ tmasks, const float* __restrict__ tsq, int B, int N, int K,
                                                               int HW, int G, float alpha, float beta, float* __restrict__ cost) {
  pdl_sync();
  extern __shared__ float smem[];
  float* s = smem;                    // [kQT][kChunk]
  float* dot = smem + kQT * kChunk;   // [kQT][G_b]
  __shared__ float red[kWarps];
  __shared__ float rowsq[kQT];
  if (blockIdx.x == 0 && blockIdx.y == 0) {
    int bad = 0;
    for (int j = threadIdx.x; j < G; j += kThreads) bad |= (labels[j] < 0 || labels[j] >= K) ? 1 : 0;
    for (int b = threadIdx.x; b < B; b += kThreads) bad |= (img_off[b + 1] - img_off[b] > N) ? 2 : 0;
    const int bad_label = __syncthreads_or(bad & 1), too_many = __syncthreads_or(bad & 2);
    if (threadIdx.x == 0) reinterpret_cast<int*>(cost)[(size_t)N * G] = (bad_label ? 1 : 0) | (too_many ? 2 : 0);
  }
  const int b = blockIdx.y, n0 = blockIdx.x * kQT, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g0 = img_off[b], gb = img_off[b + 1] - g0;
  if (gb <= 0 || gb > N) return;
  const int nq = min(kQT, N - n0);
  for (int i = threadIdx.x; i < kQT * gb; i += kThreads) dot[i] = 0.f;
  float ssq[kQT];
#pragma unroll
  for (int q = 0; q < kQT; ++q) ssq[q] = 0.f;
  const float* m = masks + ((size_t)b * N + n0) * HW;
  for (int p0 = 0; p0 < HW; p0 += kChunk) {
    const int np = min(kChunk, HW - p0);
    __syncthreads();  // the previous chunk's readers are done (and the zeroed dot is visible)
#pragma unroll
    for (int q = 0; q < kQT; ++q)
      for (int p = threadIdx.x; p < kChunk; p += kThreads) {
        float v = 0.f;
        if (q < nq && p < np) v = sigmoid(m[(size_t)q * HW + p0 + p]);
        s[q * kChunk + p] = v;
        ssq[q] += v * v;
      }
    __syncthreads();
    for (int j = warp; j < gb; j += kWarps) {
      const float* t = tmasks + (size_t)(g0 + j) * HW + p0;
      float acc[kQT];
#pragma unroll
      for (int q = 0; q < kQT; ++q) acc[q] = 0.f;
      for (int p = lane; p < np; p += 32) {
        const float tv = t[p];
#pragma unroll
        for (int q = 0; q < kQT; ++q) acc[q] += s[q * kChunk + p] * tv;
      }
#pragma unroll
      for (int q = 0; q < kQT; ++q) acc[q] = warp_sum(acc[q]);
      if (lane == 0)
#pragma unroll
        for (int q = 0; q < kQT; ++q) dot[q * gb + j] += acc[q];  // only this warp touches target j: chunk order is fixed
    }
  }
#pragma unroll
  for (int q = 0; q < kQT; ++q) {
    const float v = block_sum(ssq[q], red);
    if (threadIdx.x == 0) rowsq[q] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nq * gb; i += kThreads) {
    const int q = i / gb, j = i - q * gb, lab = labels[g0 + j];
    const float dice = (2.f * dot[q * gb + j]) / ((rowsq[q] + tsq[g0 + j]) + 1e-4f);
    const float prob = (lab >= 0 && lab < K) ? sigmoid(logits[((size_t)b * N + n0 + q) * K + lab]) : 0.f;
    cost[(size_t)N * g0 + (size_t)(n0 + q) * gb + j] = powf(dice, alpha) * powf(prob, beta);
  }
}

// the matched target of query row r (global index into the packed targets), or -1
__device__ __forceinline__ int row_target(const int* __restrict__ match, const int* __restrict__ img_off, int r, int N) {
  const int b = r / N, g0 = img_off[b], gb = img_off[b + 1] - g0, j = match[r];
  return (j >= 0 && j < gb) ? g0 + j : -1;
}

// block r = one query row.  save[r] = (Σ_k focal, and on a matched row: Σσt, Σσ², Σ bce, |σ ≥ 0.4 ∧ t > 0.5|, |σ ≥ 0.4|, |t > 0.5|, IoU (set by
// the finalize kernel))
__global__ void __launch_bounds__(kThreads) pair_sums_kernel(const float* __restrict__ logits, const float* __restrict__ masks,
                                                              const int* __restrict__ match, const int* __restrict__ labels,
                                                              const int* __restrict__ img_off, const float* __restrict__ tmasks, int N, int K, int HW,
                                                              float* __restrict__ save) {
  pdl_sync();
  __shared__ float red[kWarps];
  const int r = blockIdx.x, tg = row_target(match, img_off, r, N);
  const int lab = tg >= 0 ? labels[tg] : -1;
  const float* x = logits + (size_t)r * K;
  float f = 0.f;
  for (int k = threadIdx.x; k < K; k += kThreads) f += focal(x[k], k == lab);
  f = block_sum(f, red);
  float* sv = save + (size_t)kSave * r;
  if (tg < 0) {
    if (threadIdx.x == 0) sv[0] = f;
    return;
  }
  const float* m = masks + (size_t)r * HW;
  const float* t = tmasks + (size_t)tg * HW;
  float dot = 0.f, ssq = 0.f, bce = 0.f, inter = 0.f, npred = 0.f, ntgt = 0.f;
  for (int p = threadIdx.x; p < HW; p += kThreads) {
    const float xm = m[p], tv = t[p], sg = sigmoid(xm);
    dot += sg * tv;
    ssq += sg * sg;
    bce += bce_logits(xm, tv);
    const bool bp = sg >= 0.4f, bt = tv > 0.5f;
    inter += (bp && bt) ? 1.f : 0.f;
    npred += bp ? 1.f : 0.f;
    ntgt += bt ? 1.f : 0.f;
  }
  dot = block_sum(dot, red);
  ssq = block_sum(ssq, red);
  bce = block_sum(bce, red);
  inter = block_sum(inter, red);
  npred = block_sum(npred, red);
  ntgt = block_sum(ntgt, red);
  if (threadIdx.x == 0) sv[0] = f, sv[1] = dot, sv[2] = ssq, sv[3] = bce, sv[4] = inter, sv[5] = npred, sv[6] = ntgt;
}

// one block: out = (w_ce · Σfocal / num_inst, w_obj · mean bce(score, IoU), w_dice · Σ dice loss / num_inst, w_mask · Σ bce / (M · HW)) over the
// rows in order; the three mask terms are 0 when nothing is matched
__global__ void __launch_bounds__(kThreads) set_loss_finalize_kernel(const float* __restrict__ scores, const int* __restrict__ match,
                                                                      const int* __restrict__ img_off, const float* __restrict__ tsq, int B, int N,
                                                                      int HW, int num_pairs, float w_ce, float w_obj, float w_dice, float w_mask,
                                                                      float num_inst, float* __restrict__ save, float* __restrict__ out) {
  pdl_sync();
  __shared__ float red[kWarps];
  float f = 0.f, obj = 0.f, dice = 0.f, bce = 0.f;
  for (int r = threadIdx.x; r < B * N; r += kThreads) {
    float* sv = save + (size_t)kSave * r;
    f += sv[0];
    const int tg = row_target(match, img_off, r, N);
    if (tg < 0) continue;
    const float iou = sv[4] / ((sv[6] + sv[5] - sv[4]) + 1e-6f);  // compute_mask_iou (:19-27)
    sv[7] = iou;
    obj += bce_logits(scores[r], iou);
    dice += 1.f - (2.f * sv[1]) / ((sv[2] + tsq[tg]) + 1e-4f);  // dice_loss (:38-46)
    bce += sv[3];
  }
  f = block_sum(f, red);
  obj = block_sum(obj, red);
  dice = block_sum(dice, red);
  bce = block_sum(bce, red);
  if (threadIdx.x == 0) {
    const bool any = num_pairs > 0;
    out[0] = w_ce * (f / num_inst);
    out[1] = any ? w_obj * (obj / (float)num_pairs) : 0.f;
    out[2] = any ? w_dice * (dice / num_inst) : 0.f;
    out[3] = any ? w_mask * (bce / ((float)num_pairs * (float)HW)) : 0.f;
  }
}

// block (pixel chunk, row r): d pred_masks[r] on the chunk (exact zeros on an unmatched row); chunk 0 also writes d pred_logits[r] and
// d pred_scores[r].  grad = upstream gradients of the four weighted losses (device memory).
__global__ void __launch_bounds__(kThreads) set_loss_bwd_kernel(const float* __restrict__ logits, const float* __restrict__ masks,
                                                                 const float* __restrict__ scores, const int* __restrict__ match,
                                                                 const int* __restrict__ labels, const int* __restrict__ img_off,
                                                                 const float* __restrict__ tmasks, const float* __restrict__ tsq,
                                                                 const float* __restrict__ save, int N, int K, int HW, int num_pairs, float w_ce,
                                                                 float w_obj, float w_dice, float w_mask, float num_inst, const float* __restrict__ grad,
                                                                 float* __restrict__ dlogits, float* __restrict__ dmasks, float* __restrict__ dscores) {
  pdl_sync();
  const int r = blockIdx.y, tg = row_target(match, img_off, r, N);
  const float* sv = save + (size_t)kSave * r;
  if (blockIdx.x == 0) {
    const int lab = tg >= 0 ? labels[tg] : -1;
    const float g_ce = grad[0] * w_ce / num_inst;
    for (int k = threadIdx.x; k < K; k += kThreads) dlogits[(size_t)r * K + k] = g_ce * focal_grad(logits[(size_t)r * K + k], k == lab);
    if (threadIdx.x == 0) dscores[r] = tg >= 0 ? grad[1] * w_obj / (float)num_pairs * (sigmoid(scores[r]) - sv[7]) : 0.f;
  }
  const int p0 = blockIdx.x * kBwdPix, p1 = min(HW, p0 + kBwdPix);
  float* dm = dmasks + (size_t)r * HW;
  if (tg < 0) {
    for (int p = p0 + threadIdx.x; p < p1; p += kThreads) dm[p] = 0.f;
    return;
  }
  // dice: d/dσ (1 - 2A / D) = (4Aσ / D - 2t) / D with A = Σσt, D = Σσ² + Σt² + 1e-4; pixel BCE: (σ - t) / (M · HW)
  const float A = sv[1], D = (sv[2] + tsq[tg]) + 1e-4f;
  const float g_dice = grad[2] * w_dice / num_inst, g_mask = grad[3] * w_mask / ((float)num_pairs * (float)HW);
  const float* m = masks + (size_t)r * HW;
  const float* t = tmasks + (size_t)tg * HW;
  for (int p = p0 + threadIdx.x; p < p1; p += kThreads) {
    const float sg = sigmoid(m[p]), tv = t[p];
    const float dsig = g_dice * ((4.f * A * sg / D - 2.f * tv) / D);
    dm[p] = dsig * (sg * (1.f - sg)) + g_mask * (sg - tv);
  }
}

int check_preds(const char* fn, const float* logits, const float* masks, const int* labels, const int* img_off, const float* tmasks,
                const float* tsq, int B, int N, int K, int HW) {
  YB_REQUIRE(logits && masks && labels && img_off && tmasks && tsq, YB200_ERR_INVALID,
             "%s: null pred_logits, pred_masks, labels, offsets, target masks or target sums", fn);
  YB_REQUIRE(B > 0 && N > 0 && K > 0 && HW > 0, YB200_ERR_INVALID, "%s: B=%d N=%d K=%d HW=%d", fn, B, N, K, HW);
  YB_REQUIRE(N <= kMaxQueries && (long long)B * N < 65536 && (long long)B * N * HW < (1ll << 40) && ceil_div(HW, kBwdPix) < 65536,
             YB200_ERR_UNSUPPORTED, "%s: B=%d N=%d HW=%d exceed N <= %d, B*N < 65536", fn, B, N, HW, kMaxQueries);
  return 0;
}

int check_loss(const char* fn, const float* scores, const int* match, float* save, int num_pairs, float num_inst) {
  YB_REQUIRE(scores && match && save, YB200_ERR_INVALID, "%s: null pred_scores, match table or save buffer", fn);
  YB_REQUIRE(num_pairs >= 0 && num_inst > 0.f, YB200_ERR_INVALID, "%s: num_pairs=%d num_instances=%g", fn, num_pairs, num_inst);
  return 0;
}

}  // namespace

extern "C" int yb200_sparseinst_target_masks(const uint8_t* masks, const int64_t* table, int G, int in_h, int in_w, int H, int W, float* out,
                                             float* tsq, void* stream) {
  YB_REQUIRE(G >= 0 && in_h > 0 && in_w > 0 && H > 0 && W > 0, YB200_ERR_INVALID, "sparseinst_target_masks: G=%d input %dx%d output %dx%d", G, in_h,
             in_w, H, W);
  YB_REQUIRE((long long)H * W < (1ll << 31), YB200_ERR_UNSUPPORTED, "sparseinst_target_masks: output %dx%d", H, W);
  if (G == 0) return 0;
  YB_REQUIRE(masks && table && out && tsq, YB200_ERR_INVALID, "sparseinst_target_masks: null masks, table, out or tsq");
  YB_CHECK_CUDA(launch_k(target_masks_kernel, G, kThreads, 0, as_stream(stream), masks, table, in_h, in_w, H, W, out, tsq));
  return 0;
}

extern "C" int yb200_sparseinst_match_cost(const float* logits, const float* masks, const int32_t* labels, const int32_t* offsets, const float* tmasks,
                                           const float* tsq, int B, int N, int K, int HW, int G, float alpha, float beta, float* cost, void* stream) {
  if (int rc = check_preds("sparseinst_match_cost", logits, masks, labels, offsets, tmasks, tsq, B, N, K, HW)) return rc;
  YB_REQUIRE(cost, YB200_ERR_INVALID, "sparseinst_match_cost: null cost");
  YB_REQUIRE(G >= 0 && (long long)N * G < (1ll << 31), YB200_ERR_INVALID, "sparseinst_match_cost: G=%d", G);
  static PerDevice<int> smem_limit(48 * 1024);
  const int smem = (kQT * kChunk + kQT * N) * (int)sizeof(float);
  YB_CHECK_CUDA(raise_smem_limit(smem_limit, smem, match_cost_kernel));
  YB_CHECK_CUDA(launch_k(match_cost_kernel, dim3(ceil_div(N, kQT), B), kThreads, smem, as_stream(stream), logits, masks, labels, offsets, tmasks, tsq, B,
                         N, K, HW, G, alpha, beta, cost));
  return 0;
}

extern "C" int yb200_sparseinst_set_loss(const float* logits, const float* masks, const float* scores, const int32_t* match, const int32_t* labels,
                                         const int32_t* offsets, const float* tmasks, const float* tsq, int B, int N, int K, int HW, int num_pairs,
                                         float w_ce, float w_obj, float w_dice, float w_mask, float num_instances, float* save, float* out,
                                         void* stream) {
  if (int rc = check_preds("sparseinst_set_loss", logits, masks, labels, offsets, tmasks, tsq, B, N, K, HW)) return rc;
  if (int rc = check_loss("sparseinst_set_loss", scores, match, save, num_pairs, num_instances)) return rc;
  YB_REQUIRE(out, YB200_ERR_INVALID, "sparseinst_set_loss: null out");
  const cudaStream_t st = as_stream(stream);
  YB_CHECK_CUDA(launch_k(pair_sums_kernel, B * N, kThreads, 0, st, logits, masks, match, labels, offsets, tmasks, N, K, HW, save));
  YB_CHECK_CUDA(launch_k(set_loss_finalize_kernel, 1, kThreads, 0, st, scores, match, offsets, tsq, B, N, HW, num_pairs, w_ce, w_obj, w_dice, w_mask,
                         num_instances, save, out));
  return 0;
}

extern "C" int yb200_sparseinst_set_loss_bwd(const float* logits, const float* masks, const float* scores, const int32_t* match, const int32_t* labels,
                                             const int32_t* offsets, const float* tmasks, const float* tsq, const float* save, int B, int N, int K,
                                             int HW, int num_pairs, float w_ce, float w_obj, float w_dice, float w_mask, float num_instances,
                                             const float* grad, float* dlogits, float* dmasks, float* dscores, void* stream) {
  if (int rc = check_preds("sparseinst_set_loss_bwd", logits, masks, labels, offsets, tmasks, tsq, B, N, K, HW)) return rc;
  if (int rc = check_loss("sparseinst_set_loss_bwd", scores, match, const_cast<float*>(save), num_pairs, num_instances)) return rc;
  YB_REQUIRE(grad && dlogits && dmasks && dscores, YB200_ERR_INVALID, "sparseinst_set_loss_bwd: null grad, dlogits, dmasks or dscores");
  YB_CHECK_CUDA(launch_k(set_loss_bwd_kernel, dim3(ceil_div(HW, kBwdPix), B * N), kThreads, 0, as_stream(stream), logits, masks, scores, match, labels,
                         offsets, tmasks, tsq, save, N, K, HW, num_pairs, w_ce, w_obj, w_dice, w_mask, num_instances, grad, dlogits, dmasks, dscores));
  return 0;
}
