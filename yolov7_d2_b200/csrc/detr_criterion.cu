// DETR's matching cost and SetCriterion losses with their gradients, for every decoder layer in one launch each:
//   yb200_detr_match_cost    HungarianMatcher's cost matrix (yolov7/utils/detr_utils.py:65-86), only the per-image blocks
//   yb200_detr_set_loss      SetCriterion.loss_labels / loss_cardinality / loss_boxes (yolov7/modeling/meta_arch/detr.py:507-570)
//   yb200_detr_set_loss_bwd  their gradient w.r.t. the logits and the post-sigmoid boxes
// Inputs are fp32 [L][B][Q][K1] logits and [L][B][Q][4] (cx, cy, w, h) boxes; the targets of the batch are packed: labels [G], boxes [G][4] and
// per-image offsets [B+1].  One warp owns one query row: the softmax statistics of the row are computed once and serve every target and
// term.  Every sum runs in a fixed order (warp butterflies, then per-warp partials in warp order), so identical calls are bit-identical.
#include <math.h>

#include "dual4.cuh"
#include "host_common.cuh"
#include "sm90.cuh"

using namespace yb;

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kCostThreads = 256;   // 8 query rows per block
constexpr int kLossThreads = 1024;  // one block per decoder layer
constexpr int kBwdThreads = 256;
constexpr int kBwdRows = 32;        // query rows per backward block
constexpr int kMaxImages = 1024;    // per-image counters of the cardinality error live in shared memory

// a xor butterfly adds the same pairs in every lane (a + b == b + a), so all lanes end with the same bits
__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}

struct RowStat {
  float mx, sum;  // max logit and sum of exp(x - max)
  int arg;        // first index of the max (torch.argmax)
};

__device__ __forceinline__ RowStat row_stat(const float* __restrict__ x, int k1, int lane) {
  float mx = -INFINITY;
  int arg = k1;
  for (int k = lane; k < k1; k += 32) {
    const float v = x[k];
    if (v > mx || arg == k1) mx = v, arg = k;
  }
  for (int o = 16; o; o >>= 1) {
    const float m2 = __shfl_xor_sync(kFull, mx, o);
    const int a2 = __shfl_xor_sync(kFull, arg, o);
    if (m2 > mx || (m2 == mx && a2 < arg)) mx = m2, arg = a2;
  }
  float s = 0.f;
  for (int k = lane; k < k1; k += 32) s += expf(x[k] - mx);
  return RowStat{mx, warp_sum(s), arg};
}

struct Box {
  float cx, cy, w, h;
};
__device__ __forceinline__ Box load_box(const float* __restrict__ p) { return Box{p[0], p[1], p[2], p[3]}; }

// generalized_box_iou of box_cxcywh_to_xyxy(p) and box_cxcywh_to_xyxy(t) (yolov7/utils/boxes.py:28-31, 85-122) for one pair, with its
// derivatives w.r.t. p when T = D4
template <typename T>
__device__ __forceinline__ T giou(T pcx, T pcy, T pw, T ph, const Box& t) {
  const T px0 = pcx - pw * 0.5f, py0 = pcy - ph * 0.5f, px1 = pcx + pw * 0.5f, py1 = pcy + ph * 0.5f;
  const float tx0 = t.cx - 0.5f * t.w, ty0 = t.cy - 0.5f * t.h, tx1 = t.cx + 0.5f * t.w, ty1 = t.cy + 0.5f * t.h;
  const T area1 = (px1 - px0) * (py1 - py0);
  const float area2 = (tx1 - tx0) * (ty1 - ty0);
  const T inter = clamp_min(dmin(px1, cst(tx1)) - dmax(px0, cst(tx0)), 0.f) * clamp_min(dmin(py1, cst(ty1)) - dmax(py0, cst(ty0)), 0.f);
  const T uni = area1 + area2 - inter;
  const T iou = inter / uni;
  const T area = clamp_min(dmax(px1, cst(tx1)) - dmin(px0, cst(tx0)), 0.f) * clamp_min(dmax(py1, cst(ty1)) - dmin(py0, cst(ty0)), 0.f);
  return iou - (area - uni) / area;
}

__device__ __forceinline__ float giou_value(const Box& p, const Box& t) { return giou(cst(p.cx), cst(p.cy), cst(p.w), cst(p.h), t).v; }

// C[l, b][q, j] = w_bbox * |p - t|_1 + w_class * (-softmax(x)[label_j]) + w_giou * (-giou(p, t)); block (l, b) starts at l*Q*G + Q*off[b].
// Block 0 also writes the status word at cost[L*Q*G]: bit 0 a label outside [0, K1), bit 1 a target box whose xyxy corners are out of order
// (the assert of generalized_box_iou).
__global__ void match_cost_kernel(const float* __restrict__ logits, const float* __restrict__ boxes, const int* __restrict__ labels,
                                  const float* __restrict__ tboxes, const int* __restrict__ offsets, int L, int B, int Q, int K1, int G, float w_class,
                                  float w_bbox, float w_giou, float* __restrict__ cost) {
  pdl_sync();
  if (blockIdx.x == 0) {
    int bad = 0;
    for (int j = threadIdx.x; j < G; j += blockDim.x) {
      const int lab = labels[j];
      const Box t = load_box(tboxes + 4 * (size_t)j);
      if (lab < 0 || lab >= K1) bad |= 1;
      if (!(t.cx + 0.5f * t.w >= t.cx - 0.5f * t.w) || !(t.cy + 0.5f * t.h >= t.cy - 0.5f * t.h)) bad |= 2;
    }
    const int bad_label = __syncthreads_or(bad & 1), bad_box = __syncthreads_or(bad & 2);
    if (threadIdx.x == 0) reinterpret_cast<int*>(cost)[(size_t)L * Q * G] = (bad_label ? 1 : 0) | (bad_box ? 2 : 0);
  }
  const int row = blockIdx.x * (kCostThreads / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= L * B * Q) return;
  const int q = row % Q, b = (row / Q) % B, l = row / (Q * B);
  const int g0 = offsets[b], gb = offsets[b + 1] - g0;
  if (gb <= 0) return;
  const float* x = logits + (size_t)row * K1;
  const RowStat st = row_stat(x, K1, lane);
  const Box p = load_box(boxes + 4 * (size_t)row);
  float* out = cost + (size_t)l * Q * G + (size_t)Q * g0 + (size_t)q * gb;
  for (int j = lane; j < gb; j += 32) {
    const int lab = labels[g0 + j];
    const Box t = load_box(tboxes + 4 * (size_t)(g0 + j));
    const float prob = (lab >= 0 && lab < K1) ? expf(x[lab] - st.mx) / st.sum : 0.f;
    const float l1 = fabsf(p.cx - t.cx) + fabsf(p.cy - t.cy) + fabsf(p.w - t.w) + fabsf(p.h - t.h);
    out[j] = w_bbox * l1 + w_class * -prob + w_giou * -giou_value(p, t);
  }
}

// the target class of a query row (the no-object class K1 - 1 when unmatched) and its matched target, or -1
__device__ __forceinline__ int row_target(const int* __restrict__ match, const int* __restrict__ labels, const int* __restrict__ offsets, int mrow,
                                          int b, int K1, int* tg) {
  const int g0 = offsets[b], gb = offsets[b + 1] - g0, j = match[mrow];
  if (j < 0 || j >= gb) {
    *tg = -1;
    return K1 - 1;
  }
  *tg = g0 + j;
  return labels[g0 + j];
}

// out[l] = (loss_ce, loss_bbox, loss_giou, cardinality_error, class_error); one block per layer
__global__ void __launch_bounds__(kLossThreads) set_loss_kernel(const float* __restrict__ logits, const float* __restrict__ boxes,
                                                                 const int* __restrict__ match, const int* __restrict__ labels,
                                                                 const float* __restrict__ tboxes, const int* __restrict__ offsets, int B, int Q, int K1,
                                                                 float eos_coef, float num_boxes, float* __restrict__ out) {
  pdl_sync();
  __shared__ float fpart[kLossThreads / 32][3];
  __shared__ int ipart[kLossThreads / 32][3];
  __shared__ int card[kMaxImages];
  const int l = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int b = threadIdx.x; b < B; b += blockDim.x) card[b] = 0;
  __syncthreads();
  float ce = 0.f, l1 = 0.f, lg = 0.f;
  int n_eos = 0, n_matched = 0, correct = 0;
  const size_t base = (size_t)l * B * Q;
  for (int r = warp; r < B * Q; r += kLossThreads / 32) {
    const int b = r / Q;
    const float* x = logits + (base + r) * K1;
    const RowStat st = row_stat(x, K1, lane);
    int tg;
    const int t = row_target(match, labels, offsets, (int)(base + r), b, K1, &tg);
    const float w = t == K1 - 1 ? eos_coef : 1.f;
    n_eos += t == K1 - 1;
    ce += w * -((x[t] - st.mx) - logf(st.sum));
    if (lane == 0 && st.arg != K1 - 1) atomicAdd(&card[b], 1);  // integer count: exact in any order
    if (tg >= 0) {
      ++n_matched;
      correct += st.arg == t;
      const Box p = load_box(boxes + 4 * (base + r)), tb = load_box(tboxes + 4 * (size_t)tg);
      l1 += fabsf(p.cx - tb.cx) + fabsf(p.cy - tb.cy) + fabsf(p.w - tb.w) + fabsf(p.h - tb.h);
      lg += 1.f - giou_value(p, tb);
    }
  }
  if (lane == 0) {
    fpart[warp][0] = ce, fpart[warp][1] = l1, fpart[warp][2] = lg;
    ipart[warp][0] = n_eos, ipart[warp][1] = n_matched, ipart[warp][2] = correct;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float s_ce = 0.f, s_l1 = 0.f, s_g = 0.f;
    int s_eos = 0, s_m = 0, s_c = 0;
    for (int i = 0; i < kLossThreads / 32; ++i) {
      s_ce += fpart[i][0], s_l1 += fpart[i][1], s_g += fpart[i][2];
      s_eos += ipart[i][0], s_m += ipart[i][1], s_c += ipart[i][2];
    }
    float card_err = 0.f;
    for (int b = 0; b < B; ++b) card_err += fabsf((float)card[b] - (float)(offsets[b + 1] - offsets[b]));
    float* o = out + 5 * l;
    o[0] = s_ce / ((float)(B * Q - s_eos) + eos_coef * (float)s_eos);
    o[1] = s_l1 / num_boxes;
    o[2] = s_g / num_boxes;
    o[3] = card_err / (float)B;
    o[4] = s_m == 0 ? 100.f : 100.f - (float)s_c * (float)(100.0 / s_m);  // misc.accuracy: correct * (100 / n); 100 when nothing is matched
  }
}

// d logits = g_ce * w / Σw * (softmax - onehot(t)); d boxes = g_bbox / num_boxes * sign(p - t) - g_giou / num_boxes * d giou / d p on matched rows
__global__ void __launch_bounds__(kBwdThreads) set_loss_bwd_kernel(const float* __restrict__ logits, const float* __restrict__ boxes,
                                                                    const int* __restrict__ match, const int* __restrict__ labels,
                                                                    const float* __restrict__ tboxes, const int* __restrict__ offsets, int B, int Q,
                                                                    int K1, float eos_coef, float num_boxes, const float* __restrict__ grad,
                                                                    float* __restrict__ dlogits, float* __restrict__ dboxes) {
  pdl_sync();
  __shared__ int eos_part[kBwdThreads / 32];
  const int l = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t base = (size_t)l * B * Q;
  // the layer's weight sum Σw, counted exactly as the forward counts it
  int n_eos = 0;
  for (int r = threadIdx.x; r < B * Q; r += blockDim.x) {
    int tg;
    n_eos += row_target(match, labels, offsets, (int)(base + r), r / Q, K1, &tg) == K1 - 1;
  }
  n_eos = __reduce_add_sync(kFull, n_eos);
  if (lane == 0) eos_part[warp] = n_eos;
  __syncthreads();
  n_eos = 0;
  for (int i = 0; i < kBwdThreads / 32; ++i) n_eos += eos_part[i];
  const float wsum = (float)(B * Q - n_eos) + eos_coef * (float)n_eos;
  const float g_ce = grad[3 * l], g_l1 = grad[3 * l + 1] / num_boxes, g_giou = grad[3 * l + 2] / num_boxes;
  const int r_end = min(B * Q, (int)(blockIdx.x + 1) * kBwdRows);
  for (int r = blockIdx.x * kBwdRows + warp; r < r_end; r += kBwdThreads / 32) {
    const float* x = logits + (base + r) * K1;
    float* dx = dlogits + (base + r) * K1;
    const RowStat st = row_stat(x, K1, lane);
    int tg;
    const int t = row_target(match, labels, offsets, (int)(base + r), r / Q, K1, &tg);
    const float coef = g_ce * (t == K1 - 1 ? eos_coef : 1.f) / wsum;
    for (int k = lane; k < K1; k += 32) dx[k] = coef * (expf(x[k] - st.mx) / st.sum - (k == t ? 1.f : 0.f));
    if (lane < 4) {
      float d = 0.f;
      if (tg >= 0) {
        const float* pp = boxes + 4 * (base + r);
        const Box tb = load_box(tboxes + 4 * (size_t)tg);
        // lane c differentiates w.r.t. coordinate c only (a constant index keeps the dual number in registers)
        const D4 g = giou(lane == 0 ? var(pp[0], 0) : cst(pp[0]), lane == 1 ? var(pp[1], 0) : cst(pp[1]), lane == 2 ? var(pp[2], 0) : cst(pp[2]),
                          lane == 3 ? var(pp[3], 0) : cst(pp[3]), tb);
        const float diff = pp[lane] - (lane == 0 ? tb.cx : lane == 1 ? tb.cy : lane == 2 ? tb.w : tb.h);
        d = g_l1 * (float)((diff > 0.f) - (diff < 0.f)) - g_giou * g.g[0];
      }
      dboxes[4 * (base + r) + lane] = d;
    }
  }
}

int check_common(const char* fn, const float* logits, const float* boxes, const int* labels, const float* tboxes, const int* offsets, int L, int B,
                 int Q, int K1) {
  YB_REQUIRE(logits && boxes && offsets && labels && tboxes, YB200_ERR_INVALID, "%s: null logits, boxes, labels, target boxes or offsets", fn);
  YB_REQUIRE(L > 0 && B > 0 && Q > 0 && K1 >= 2, YB200_ERR_INVALID, "%s: L=%d B=%d Q=%d K1=%d", fn, L, B, Q, K1);
  YB_REQUIRE((long long)L * B * Q <= (1 << 24) && B <= kMaxImages, YB200_ERR_UNSUPPORTED, "%s: L*B*Q=%lld rows and B=%d images exceed %d and %d", fn,
             (long long)L * B * Q, B, 1 << 24, kMaxImages);
  return 0;
}

int check_loss(const char* fn, const int* match, float eos_coef, float num_boxes) {
  YB_REQUIRE(match, YB200_ERR_INVALID, "%s: null match table", fn);
  YB_REQUIRE(eos_coef >= 0.f && num_boxes > 0.f, YB200_ERR_INVALID, "%s: eos_coef=%g num_boxes=%g", fn, eos_coef, num_boxes);
  return 0;
}

}  // namespace

extern "C" int yb200_detr_match_cost(const float* logits, const float* boxes, const int32_t* labels, const float* target_boxes, const int32_t* offsets,
                                     int L, int B, int Q, int K1, int G, float w_class, float w_bbox, float w_giou, float* cost, void* stream) {
  if (int rc = check_common("detr_match_cost", logits, boxes, labels, target_boxes, offsets, L, B, Q, K1)) return rc;
  YB_REQUIRE(cost, YB200_ERR_INVALID, "detr_match_cost: null cost");
  YB_REQUIRE(G >= 0 && (long long)L * Q * G < (1ll << 31), YB200_ERR_INVALID, "detr_match_cost: G=%d", G);
  const int blocks = ceil_div(L * B * Q, kCostThreads / 32);
  YB_CHECK_CUDA(launch_k(match_cost_kernel, blocks, kCostThreads, 0, as_stream(stream), logits, boxes, labels, target_boxes, offsets, L, B, Q, K1, G,
                         w_class, w_bbox, w_giou, cost));
  return 0;
}

extern "C" int yb200_detr_set_loss(const float* logits, const float* boxes, const int32_t* match, const int32_t* labels, const float* target_boxes,
                                   const int32_t* offsets, int L, int B, int Q, int K1, float eos_coef, float num_boxes, float* out, void* stream) {
  if (int rc = check_common("detr_set_loss", logits, boxes, labels, target_boxes, offsets, L, B, Q, K1)) return rc;
  if (int rc = check_loss("detr_set_loss", match, eos_coef, num_boxes)) return rc;
  YB_REQUIRE(out, YB200_ERR_INVALID, "detr_set_loss: null out");
  YB_CHECK_CUDA(launch_k(set_loss_kernel, L, kLossThreads, 0, as_stream(stream), logits, boxes, match, labels, target_boxes, offsets, B, Q, K1, eos_coef,
                         num_boxes, out));
  return 0;
}

extern "C" int yb200_detr_set_loss_bwd(const float* logits, const float* boxes, const int32_t* match, const int32_t* labels, const float* target_boxes,
                                       const int32_t* offsets, int L, int B, int Q, int K1, float eos_coef, float num_boxes, const float* grad,
                                       float* dlogits, float* dboxes, void* stream) {
  if (int rc = check_common("detr_set_loss_bwd", logits, boxes, labels, target_boxes, offsets, L, B, Q, K1)) return rc;
  if (int rc = check_loss("detr_set_loss_bwd", match, eos_coef, num_boxes)) return rc;
  YB_REQUIRE(grad && dlogits && dboxes, YB200_ERR_INVALID, "detr_set_loss_bwd: null grad, dlogits or dboxes");
  const dim3 grid(ceil_div(B * Q, kBwdRows), L);
  YB_CHECK_CUDA(launch_k(set_loss_bwd_kernel, grid, kBwdThreads, 0, as_stream(stream), logits, boxes, match, labels, target_boxes, offsets, B, Q, K1,
                         eos_coef, num_boxes, grad, dlogits, dboxes));
  return 0;
}
