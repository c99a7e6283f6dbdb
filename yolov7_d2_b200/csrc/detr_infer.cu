// DETR's meta-architecture work around the network (yolov7/modeling/meta_arch/detr.py, yolov7/modeling/backbone/detr_backbone.py): the padding
// masks and sine position embeddings of every backbone level (MaskedBackboneTraceFriendly.mask_out_padding :389-403, PositionEmbeddingSine
// :334-375), the target boxes of `prepare_targets` (:204-217), and `inference` (:219-265) followed by detectron2's detector_postprocess.  No
// float atomics and fixed-order sums: the results are bit-reproducible.  Every fp32 operation below is one IEEE operation written with an
// explicit rounding intrinsic, so that no multiply-add is contracted and each value has the bits of the reference's torch arithmetic.
#include "host_common.cuh"
#include "infer_compact.cuh"
#include "sm90.cuh"

#include <math.h>

#include <algorithm>

using namespace yb;

namespace {

struct MaskPosArgs {
  yb200_detr_level lv[YB200_DETR_MAX_LEVELS];
  long long first[YB200_DETR_MAX_LEVELS + 1];  // prefix of the levels' pos element counts
  int nlevels, B, npf;
};

// One thread per position element [b][c][y][x] of every level; the c == 0 threads also write the mask.  The valid region of image b is the
// top-left (hv, wv) rectangle, so not_mask.cumsum has a closed form: y_embed = x < wv ? min(y + 1, hv) : 0 and its last row is x < wv ? hv : 0
// (the same with the axes swapped for x_embed), exact integers in fp32.  Then e / (last + 1e-6) * fp32(2 pi), e / dim_t[c], sin on even
// channels and cos on odd ones; the y half comes first.
__global__ void __launch_bounds__(256) mask_pos_kernel(MaskPosArgs a, const int32_t* __restrict__ valid, const float* __restrict__ dim_t) {
  pdl_sync();
  const float two_pi = static_cast<float>(6.283185307179586);
  const int C = 2 * a.npf;
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < a.first[a.nlevels];
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    int l = 0;
    while (t >= a.first[l + 1]) ++l;
    const yb200_detr_level& lv = a.lv[l];
    const long long e = t - a.first[l];
    const int x = static_cast<int>(e % lv.w);
    long long r = e / lv.w;
    const int y = static_cast<int>(r % lv.h);
    r /= lv.h;
    const int c = static_cast<int>(r % C);
    const int b = static_cast<int>(r / C);
    const int* v = valid + 2 * (static_cast<long long>(l) * a.B + b);
    const int hv = min(max(v[0], 0), lv.h), wv = min(max(v[1], 0), lv.w);
    if (c == 0) lv.mask[(static_cast<long long>(b) * lv.h + y) * lv.w + x] = static_cast<uint8_t>(!(y < hv && x < wv));
    const bool ax = c >= a.npf;  // false: the y half
    const int cc = ax ? c - a.npf : c;
    int num, last;
    if (!ax) num = x < wv ? min(y + 1, hv) : 0, last = x < wv ? hv : 0;
    else num = y < hv ? min(x + 1, wv) : 0, last = y < hv ? wv : 0;
    const float emb = __fmul_rn(__fdiv_rn(static_cast<float>(num), __fadd_rn(static_cast<float>(last), 1e-6f)), two_pi);
    const float arg = __fdiv_rn(emb, dim_t[cc]);
    lv.pos[e] = (cc & 1) ? cosf(arg) : sinf(arg);
  }
}

constexpr int kInferWarps = 8;

// One warp per (image, query) row.  probabilities p_k = exp(l_k - max) / Σ exp(l_j - max) (max and sum over all K1 logits, butterfly order);
// score = max over the first K1 - 1 of p with the lowest k on ties; keep = score > threshold.  Lane 0 then runs the box chain of `inference`
// and detector_postprocess: cxcywh -> xyxy, Boxes.scale by the image size, Boxes.scale by the output / image ratios, clip to the output size,
// nonempty.  keep[row] bit 0 = kept after the threshold and nonempty(); bit 1 = a thresholded box is not finite (Boxes.clip asserts).
__global__ void __launch_bounds__(32 * kInferWarps) detr_infer_rows_kernel(const float* __restrict__ logits, const float* __restrict__ boxes, int B, int Q,
                                                                           int K1, const float* __restrict__ sizes, float threshold,
                                                                           float* __restrict__ score, int32_t* __restrict__ label,
                                                                           uint8_t* __restrict__ keep, float* __restrict__ box) {
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const long long row = static_cast<long long>(blockIdx.x) * kInferWarps + (threadIdx.x >> 5);
  if (row >= static_cast<long long>(B) * Q) return;
  const float* l = logits + row * K1;
  float m = -INFINITY;
  for (int k = lane; k < K1; k += 32) m = fmaxf(m, l[k]);
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float s = 0.f;
  for (int k = lane; k < K1; k += 32) s = __fadd_rn(s, expf(__fsub_rn(l[k], m)));
  for (int o = 16; o > 0; o >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
  float best = -1.f;
  int arg = K1;
  for (int k = lane; k < K1 - 1; k += 32) {
    const float p = __fdiv_rn(expf(__fsub_rn(l[k], m)), s);
    if (p > best) best = p, arg = k;
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
    if (ob > best || (ob == best && oa < arg)) best = ob, arg = oa;
  }
  if (lane) return;
  if (isnan(s)) best = NAN, arg = 0;  // torch's max propagates NaN
  const int b = static_cast<int>(row / Q);
  const float* sz = sizes + 6 * b;  // (image w, image h, out w / image w, out h / image h, out w, out h)
  const float* bx = boxes + 4 * row;
  const float hw = __fmul_rn(0.5f, bx[2]), hh = __fmul_rn(0.5f, bx[3]);
  float x0 = __fsub_rn(bx[0], hw), y0 = __fsub_rn(bx[1], hh), x1 = __fadd_rn(bx[0], hw), y1 = __fadd_rn(bx[1], hh);
  x0 = __fmul_rn(__fmul_rn(x0, sz[0]), sz[2]), x1 = __fmul_rn(__fmul_rn(x1, sz[0]), sz[2]);
  y0 = __fmul_rn(__fmul_rn(y0, sz[1]), sz[3]), y1 = __fmul_rn(__fmul_rn(y1, sz[1]), sz[3]);
  const bool kept = best > threshold;
  const bool finite = isfinite(x0) && isfinite(y0) && isfinite(x1) && isfinite(y1);
  x0 = fminf(fmaxf(x0, 0.f), sz[4]), x1 = fminf(fmaxf(x1, 0.f), sz[4]);
  y0 = fminf(fmaxf(y0, 0.f), sz[5]), y1 = fminf(fmaxf(y1, 0.f), sz[5]);
  const bool nonempty = __fsub_rn(x1, x0) > 0.f && __fsub_rn(y1, y0) > 0.f;
  score[row] = best;
  label[row] = arg;
  keep[row] = static_cast<uint8_t>((kept && nonempty && finite ? 1 : 0) | (kept && !finite ? 2 : 0));
  box[4 * row] = x0, box[4 * row + 1] = y0, box[4 * row + 2] = x1, box[4 * row + 3] = y1;
}

// One CTA per image: gt_boxes / [w, h, w, h], then box_xyxy_to_cxcywh ((x0 + x1) / 2, (y0 + y1) / 2, x1 - x0, y1 - y0)
__global__ void __launch_bounds__(128) pack_targets_kernel(const float* __restrict__ in, const int32_t* __restrict__ table, float* __restrict__ out) {
  pdl_sync();
  const int32_t* t = table + 4 * blockIdx.x;  // (first box, count, h, w)
  const float h = static_cast<float>(t[2]), w = static_cast<float>(t[3]);
  for (int i = threadIdx.x; i < t[1]; i += blockDim.x) {
    const long long r = 4LL * (t[0] + i);
    const float x0 = __fdiv_rn(in[r], w), y0 = __fdiv_rn(in[r + 1], h), x1 = __fdiv_rn(in[r + 2], w), y1 = __fdiv_rn(in[r + 3], h);
    out[r] = __fdiv_rn(__fadd_rn(x0, x1), 2.f);
    out[r + 1] = __fdiv_rn(__fadd_rn(y0, y1), 2.f);
    out[r + 2] = __fsub_rn(x1, x0);
    out[r + 3] = __fsub_rn(y1, y0);
  }
}

}  // namespace

extern "C" int yb200_detr_mask_pos(const yb200_detr_level* levels, int nlevels, int B, const int32_t* valid, const float* dim_t, int npf, void* stream) {
  YB_REQUIRE(levels && valid && dim_t, YB200_ERR_INVALID, "detr_mask_pos: null pointer");
  YB_REQUIRE(nlevels > 0 && nlevels <= YB200_DETR_MAX_LEVELS, YB200_ERR_UNSUPPORTED, "detr_mask_pos: %d levels (1 to %d)", nlevels,
             YB200_DETR_MAX_LEVELS);
  YB_REQUIRE(B > 0 && npf > 0 && npf % 2 == 0, YB200_ERR_INVALID, "detr_mask_pos: B %d, num_pos_feats %d (positive and even)", B, npf);
  MaskPosArgs a{};
  a.nlevels = nlevels, a.B = B, a.npf = npf;
  for (int l = 0; l < nlevels; ++l) {
    const yb200_detr_level& lv = levels[l];
    YB_REQUIRE(lv.mask && lv.pos, YB200_ERR_INVALID, "detr_mask_pos: level %d has a null pointer", l);
    YB_REQUIRE(lv.h > 0 && lv.w > 0, YB200_ERR_INVALID, "detr_mask_pos: level %d is %dx%d", l, lv.h, lv.w);
    a.lv[l] = lv;
    a.first[l + 1] = a.first[l] + 2LL * npf * B * lv.h * lv.w;
  }
  const long long total = a.first[nlevels];
  const int blocks = static_cast<int>(std::max<long long>(1, std::min<long long>((total + 255) / 256, 32LL * sm_count())));
  YB_CHECK_CUDA(launch_k(mask_pos_kernel, blocks, 256, 0, as_stream(stream), a, valid, dim_t));
  return 0;
}

extern "C" int yb200_detr_infer(const float* logits, const float* boxes, int B, int Q, int K1, const float* sizes, float threshold, float* score,
                                int32_t* label, uint8_t* keep, float* box, int32_t* counts, int32_t* offsets, int32_t* kept_query, float* kept_score,
                                int64_t* kept_label, float* kept_box, int32_t* status, void* stream) {
  YB_REQUIRE(logits && boxes && sizes, YB200_ERR_INVALID, "detr_infer: null input pointer");
  YB_REQUIRE(score && label && keep && box && counts && offsets && kept_query && kept_score && kept_label && kept_box && status, YB200_ERR_INVALID,
             "detr_infer: null output pointer");
  YB_REQUIRE(B > 0 && Q > 0 && K1 >= 2, YB200_ERR_INVALID, "detr_infer: B %d, Q %d, K1 %d (at least one class and no-object)", B, Q, K1);
  YB_REQUIRE(1LL * B * Q < (1LL << 31) / kInferWarps, YB200_ERR_UNSUPPORTED, "detr_infer: %d x %d queries", B, Q);
  cudaStream_t st = as_stream(stream);
  YB_CHECK_CUDA(launch_k(detr_infer_rows_kernel, ceil_div(B * Q, kInferWarps), 32 * kInferWarps, 0, st, logits, boxes, B, Q, K1, sizes, threshold,
                         score, label, keep, box));
  YB_CHECK_CUDA(launch_k(infer_compact_kernel, 1, 256, 0, st, static_cast<const uint8_t*>(keep), static_cast<const float*>(score),
                         static_cast<const int32_t*>(label), static_cast<const float*>(box), B, Q, counts, offsets, kept_query, kept_score, kept_label,
                         kept_box, status));
  return 0;
}

extern "C" int yb200_detr_pack_targets(const float* boxes, const int32_t* table, int B, int G, float* out, void* stream) {
  YB_REQUIRE(boxes && table && out, YB200_ERR_INVALID, "detr_pack_targets: null pointer");
  YB_REQUIRE(B > 0 && G >= 0, YB200_ERR_INVALID, "detr_pack_targets: %d images, %d boxes", B, G);
  if (G == 0) return 0;
  YB_CHECK_CUDA(launch_k(pack_targets_kernel, B, 128, 0, as_stream(stream), boxes, table, out));
  return 0;
}
