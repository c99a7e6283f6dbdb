// SparseInst's meta-architecture work around the network (yolov7/modeling/meta_arch/sparseinst.py): the input normalisation and padding of
// `preprocess_inputs` (:96-100) for a whole batch, and `inference` (:179-241) -- class scores, the cls threshold, mask-ness rescoring, and the
// two bilinear resizes of every kept mask (to the padded input, crop, to the original size) fused with the mask threshold.  Every sum runs in
// a fixed order and there are no float atomics: the results are bit-reproducible.
#include "host_common.cuh"
#include "infer_compact.cuh"
#include "sm90.cuh"

#include <math.h>

#include <algorithm>

using namespace yb;

namespace {

// (float(x) - mean[c]) / std[c] into the zero-padded [n][3][hp][wp] batch: one IEEE subtract and one IEEE divide, torch's arithmetic for
// `(image - pixel_mean) / pixel_std`; pixels beyond an image's (h, w) are 0, ImageList.from_tensors' pad value
template <typename T>
__global__ void __launch_bounds__(256) normalize_pad_kernel(const T* __restrict__ img, const int64_t* __restrict__ table, const float* __restrict__ mean,
                                                            const float* __restrict__ stdv, int hp, int wp, float* __restrict__ out, long long total) {
  pdl_sync();
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total; t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(t % wp);
    const long long r = t / wp;
    const int y = static_cast<int>(r % hp);
    const long long nc = r / hp;
    const int c = static_cast<int>(nc % 3);
    const long long n = nc / 3;
    const long long off = table[3 * n];
    const int h = static_cast<int>(table[3 * n + 1]), w = static_cast<int>(table[3 * n + 2]);
    float v = 0.f;
    if (y < h && x < w) v = (static_cast<float>(img[off + (static_cast<long long>(c) * h + y) * w + x]) - mean[c]) / stdv[c];
    out[t] = v;
  }
}

__device__ __forceinline__ float sigmoidf(float x) { return 1.f / (1.f + expf(-x)); }  // ATen's sigmoid for fp32

constexpr int kScoreThreads = 256;

// One CTA per (image, query): v_k = sqrt(sigmoid(l_k) * sigmoid(s)), score = max_k v_k with the lowest k on ties (ATen's max(dim)), keep =
// score > cls_threshold; for a kept query, with m = sigmoid(mask pixel), rescored = score * (Σ m [m > thr] / (Σ [m > thr] + 1e-6)) (:25-27).
// The pixel sums run strided per thread, then a fixed tree over the CTA.
__global__ void __launch_bounds__(kScoreThreads) infer_scores_kernel(const float* __restrict__ logits, const float* __restrict__ obj,
                                                                       const float* __restrict__ masks, int K, int HW, float cls_thr, float mask_thr,
                                                                       float* __restrict__ score, int32_t* __restrict__ label, uint8_t* __restrict__ keep,
                                                                       float* __restrict__ rescored) {
  pdl_sync();
  __shared__ float s_sum[kScoreThreads], s_cnt[kScoreThreads];
  __shared__ float s_score;
  __shared__ int s_keep;
  const long long row = blockIdx.x;
  if (threadIdx.x == 0) {
    const float so = sigmoidf(obj[row]);
    const float* l = logits + row * K;
    float best = 0.f;
    int arg = 0;
    for (int k = 0; k < K; ++k) {
      const float v = sqrtf(sigmoidf(l[k]) * so);
      if (k == 0 || v > best) best = v, arg = k;
    }
    const int kp = best > cls_thr;
    score[row] = best;
    label[row] = arg;
    keep[row] = static_cast<uint8_t>(kp);
    s_score = best;
    s_keep = kp;
  }
  __syncthreads();
  if (!s_keep) {
    if (threadIdx.x == 0) rescored[row] = 0.f;
    return;
  }
  const float* m = masks + row * HW;
  float a = 0.f, c = 0.f;
  for (int i = threadIdx.x; i < HW; i += kScoreThreads) {
    const float p = sigmoidf(m[i]);
    if (p > mask_thr) a += p, c += 1.f;
  }
  s_sum[threadIdx.x] = a;
  s_cnt[threadIdx.x] = c;
  __syncthreads();
  for (int s = kScoreThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      s_sum[threadIdx.x] += s_sum[threadIdx.x + s];
      s_cnt[threadIdx.x] += s_cnt[threadIdx.x + s];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) rescored[row] = s_score * (s_sum[0] / (s_cnt[0] + 1e-6f));
}

// ATen's upsample_bilinear2d source index (align_corners=False, size given): scale = in / out, src = max(scale (dst + 0.5) - 0.5, 0),
// i0 = (int)src, i1 = i0 + (i0 < in - 1), l1 = src - i0, l0 = 1 - l1, all fp32
struct Tap {
  int i0, i1;
  float l0, l1;
};
__device__ __forceinline__ Tap tap(float scale, int dst, int in) {
  float s = scale * (static_cast<float>(dst) + 0.5f) - 0.5f;
  s = s < 0.f ? 0.f : s;
  Tap t;
  t.i0 = static_cast<int>(s);
  t.i1 = t.i0 + (t.i0 < in - 1 ? 1 : 0);
  t.l1 = s - static_cast<float>(t.i0);
  t.l0 = 1.f - t.l1;
  return t;
}
// h0 (w0 x00 + w1 x01) + h1 (w0 x10 + w1 x11): the order of ATen's CUDA kernel
__device__ __forceinline__ float blend(const Tap& ty, const Tap& tx, const float* p, int pitch, int y0, int x0) {
  const float* r0 = p + (ty.i0 - y0) * pitch - x0;
  const float* r1 = p + (ty.i1 - y0) * pitch - x0;
  return ty.l0 * (tx.l0 * r0[tx.i0] + tx.l1 * r0[tx.i1]) + ty.l1 * (tx.l0 * r1[tx.i0] + tx.l1 * r1[tx.i1]);
}

struct PasteArgs {
  yb200_paste_image img[YB200_PASTE_MAX_IMAGES];
  int B, N, hm, wm, hp, wp;
  int ty, tx, tiles_x;            // output tile and the tile grid's width
  int sa_rows, sa_cols;           // shared-memory extents of the source window and of the resize-A window
  int a_rows, a_cols;
};

// One CTA per (output tile, kept mask).  Three stages in shared memory, none in global memory:
//   S = sigmoid(mask) on the source window the tile needs;
//   A = resize A (Hm, Wm) -> (Hp, Wp) of S on the window of padded-input pixels the tile's resize-B taps read (crop coordinates = padded
//       coordinates, the crop starts at (0, 0));
//   out = resize B (h, w) -> (H0, W0) of A, > mask_threshold, as uint8.
__global__ void __launch_bounds__(256) paste_masks_kernel(const float* __restrict__ masks, const int32_t* __restrict__ kept_query, PasteArgs a,
                                                          float mask_thr, uint8_t* __restrict__ out) {
  pdl_sync();
  extern __shared__ float smem[];
  const int j = blockIdx.y;
  int b = 0;
  while (b < a.B - 1 && j >= a.img[b].first + a.img[b].count) ++b;
  const yb200_paste_image& im = a.img[b];
  const int q = kept_query[j];
  if (q < 0 || q >= a.N) return;
  const int Y0 = (blockIdx.x / a.tiles_x) * a.ty, X0 = (blockIdx.x % a.tiles_x) * a.tx;
  if (Y0 >= im.out_h || X0 >= im.out_w) return;
  const int Y1 = min(Y0 + a.ty, im.out_h) - 1, X1 = min(X0 + a.tx, im.out_w) - 1;
  const float sby = static_cast<float>(im.h) / static_cast<float>(im.out_h), sbx = static_cast<float>(im.w) / static_cast<float>(im.out_w);
  const float say = static_cast<float>(a.hm) / static_cast<float>(a.hp), sax = static_cast<float>(a.wm) / static_cast<float>(a.wp);
  // the padded-input window read by resize B, and the source window read by resize A (taps are monotone in dst)
  const int yb0 = tap(sby, Y0, im.h).i0, yb1 = tap(sby, Y1, im.h).i1, xb0 = tap(sbx, X0, im.w).i0, xb1 = tap(sbx, X1, im.w).i1;
  const int ys0 = tap(say, yb0, a.hm).i0, ys1 = tap(say, yb1, a.hm).i1, xs0 = tap(sax, xb0, a.wm).i0, xs1 = tap(sax, xb1, a.wm).i1;
  const int nyb = yb1 - yb0 + 1, nxb = xb1 - xb0 + 1, nys = ys1 - ys0 + 1, nxs = xs1 - xs0 + 1;
  float* S = smem;
  float* A = smem + a.sa_rows * a.sa_cols;
  const float* src = masks + (static_cast<long long>(b) * a.N + q) * a.hm * a.wm;
  // 128 threads across the columns, 2 down the rows: each thread computes its column's taps once per column
  const int c0 = threadIdx.x % 128, r0 = threadIdx.x / 128;
  for (int c = c0; c < nxs; c += 128)
    for (int r = r0; r < nys; r += 2) S[r * a.sa_cols + c] = sigmoidf(src[static_cast<long long>(ys0 + r) * a.wm + xs0 + c]);
  __syncthreads();
  for (int c = c0; c < nxb; c += 128) {
    const Tap tx = tap(sax, xb0 + c, a.wm);
    for (int r = r0; r < nyb; r += 2) A[r * a.a_cols + c] = blend(tap(say, yb0 + r, a.hm), tx, S, a.sa_cols, ys0, xs0);
  }
  __syncthreads();
  uint8_t* o = out + im.out_off + static_cast<long long>(j - im.first) * im.out_h * im.out_w;
  for (int c = c0; c <= X1 - X0; c += 128) {
    const Tap tx = tap(sbx, X0 + c, im.w);
    for (int r = r0; r <= Y1 - Y0; r += 2) {
      const float v = blend(tap(sby, Y0 + r, im.h), tx, A, a.a_cols, yb0, xb0);
      o[static_cast<long long>(Y0 + r) * im.out_w + X0 + c] = static_cast<uint8_t>(v > mask_thr);
    }
  }
}

// Upper bound on the rows a window of `t` consecutive destination pixels taps when resizing `in` -> `out`: the source span (t - 1) * scale,
// one more for i0 to i1, one for the partial first pixel and one against rounding of the fp32 index arithmetic
int window(int t, int in, int out) {
  const double span = static_cast<double>(in) / static_cast<double>(out) * (t - 1);
  return std::min(in, static_cast<int>(span) + 4);
}

constexpr int kPasteSmem = 48 * 1024;

}  // namespace

extern "C" int yb200_normalize_pad(const void* images, int is_f32, const int64_t* table, int n, const float* mean, const float* std, int hp, int wp,
                                   float* out, void* stream) {
  YB_REQUIRE(images && table && mean && std && out, YB200_ERR_INVALID, "normalize_pad: null pointer");
  YB_REQUIRE(n > 0 && hp > 0 && wp > 0, YB200_ERR_INVALID, "normalize_pad: %d images padded to %dx%d", n, hp, wp);
  const long long total = 3LL * n * hp * wp;
  const int blocks = static_cast<int>(std::max<long long>(1, std::min<long long>((total + 255) / 256, 16LL * sm_count())));
  if (is_f32)
    launch_k(normalize_pad_kernel<float>, blocks, 256, 0, as_stream(stream), static_cast<const float*>(images), table, mean, std, hp, wp, out, total);
  else
    launch_k(normalize_pad_kernel<uint8_t>, blocks, 256, 0, as_stream(stream), static_cast<const uint8_t*>(images), table, mean, std, hp, wp, out,
             total);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_sparseinst_infer_scores(const float* logits, const float* scores, const float* masks, int B, int N, int K, int HW,
                                             float cls_threshold, float mask_threshold, float* score, int32_t* label, uint8_t* keep, float* rescored,
                                             int32_t* counts, int32_t* offsets, int32_t* kept_query, float* kept_score, int64_t* kept_label,
                                             void* stream) {
  YB_REQUIRE(logits && scores && masks, YB200_ERR_INVALID, "sparseinst_infer_scores: null input pointer");
  YB_REQUIRE(score && label && keep && rescored && counts && offsets && kept_query && kept_score && kept_label, YB200_ERR_INVALID,
             "sparseinst_infer_scores: null output pointer");
  YB_REQUIRE(B > 0 && N > 0 && K > 0 && HW > 0, YB200_ERR_INVALID, "sparseinst_infer_scores: B %d, N %d, K %d, HW %d", B, N, K, HW);
  YB_REQUIRE(1LL * B * N < (1LL << 31), YB200_ERR_UNSUPPORTED, "sparseinst_infer_scores: %d x %d queries", B, N);
  cudaStream_t st = as_stream(stream);
  launch_k(infer_scores_kernel, B * N, kScoreThreads, 0, st, logits, scores, masks, K, HW, cls_threshold, mask_threshold, score, label, keep, rescored);
  YB_CHECK_CUDA(cudaGetLastError());
  launch_k(infer_compact_kernel, 1, 256, 0, st, static_cast<const uint8_t*>(keep), static_cast<const float*>(rescored),
           static_cast<const int32_t*>(label), static_cast<const float*>(nullptr), B, N, counts, offsets, kept_query, kept_score, kept_label,
           static_cast<float*>(nullptr), static_cast<int32_t*>(nullptr));
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_sparseinst_paste_masks(const float* masks, int N, int Hm, int Wm, const int32_t* kept_query, const yb200_paste_image* images, int B,
                                            int hp, int wp, float mask_threshold, uint8_t* out, void* stream) {
  YB_REQUIRE(masks && kept_query && images && out, YB200_ERR_INVALID, "sparseinst_paste_masks: null pointer");
  YB_REQUIRE(N > 0 && Hm > 0 && Wm > 0 && hp > 0 && wp > 0, YB200_ERR_INVALID, "sparseinst_paste_masks: N %d, masks %dx%d, padded %dx%d", N, Hm, Wm,
             hp, wp);
  YB_REQUIRE(B > 0 && B <= YB200_PASTE_MAX_IMAGES, YB200_ERR_UNSUPPORTED, "sparseinst_paste_masks: %d images (1 to %d per call)", B,
             YB200_PASTE_MAX_IMAGES);
  PasteArgs a{};
  a.B = B, a.N = N, a.hm = Hm, a.wm = Wm, a.hp = hp, a.wp = wp;
  int total = 0, max_h = 1, max_w = 1;
  for (int b = 0; b < B; ++b) {
    const yb200_paste_image& im = images[b];
    YB_REQUIRE(im.h > 0 && im.w > 0 && im.h <= hp && im.w <= wp && im.out_h > 0 && im.out_w > 0, YB200_ERR_INVALID,
               "sparseinst_paste_masks: image %d of %dx%d (padded %dx%d) to %dx%d", b, im.h, im.w, hp, wp, im.out_h, im.out_w);
    YB_REQUIRE(im.count >= 0 && im.count <= N && im.first == total && im.out_off >= 0, YB200_ERR_INVALID,
               "sparseinst_paste_masks: image %d has masks [%d, %d + %d) after %d, output offset %lld", b, im.first, im.first, im.count, total,
               static_cast<long long>(im.out_off));
    total += im.count;
    a.img[b] = im;
    if (im.count) max_h = std::max(max_h, im.out_h), max_w = std::max(max_w, im.out_w);
  }
  YB_REQUIRE(total < 65536, YB200_ERR_UNSUPPORTED, "sparseinst_paste_masks: %d masks (at most 65535 per call)", total);
  if (total == 0) return 0;
  // the largest tile (up to 16 x 128) whose two windows fit in 48 KB for every image of the batch
  int ty = 16, tx = 128;
  for (;;) {
    int ar = 0, ac = 0, sr = 0, sc = 0;
    for (int b = 0; b < B; ++b) {
      const yb200_paste_image& im = images[b];
      if (!im.count) continue;
      const int r = window(ty, im.h, im.out_h), c = window(tx, im.w, im.out_w);
      ar = std::max(ar, r), ac = std::max(ac, c);
      sr = std::max(sr, window(r, Hm, hp)), sc = std::max(sc, window(c, Wm, wp));
    }
    if (4LL * (ar * ac + sr * sc) <= kPasteSmem || (ty == 1 && tx == 1)) {
      a.a_rows = ar, a.a_cols = ac, a.sa_rows = sr, a.sa_cols = sc;
      break;
    }
    if (tx > 32 || ty == 1) tx = std::max(1, tx / 2);
    else ty /= 2;
  }
  const int smem = 4 * (a.a_rows * a.a_cols + a.sa_rows * a.sa_cols);
  YB_REQUIRE(smem <= kPasteSmem, YB200_ERR_UNSUPPORTED, "sparseinst_paste_masks: a 1x1 output tile needs %d bytes of windows", smem);
  a.ty = ty, a.tx = tx, a.tiles_x = ceil_div(max_w, tx);
  const long long tiles = 1LL * a.tiles_x * ceil_div(max_h, ty);
  YB_REQUIRE(tiles < (1LL << 31), YB200_ERR_UNSUPPORTED, "sparseinst_paste_masks: %dx%d output", max_h, max_w);
  launch_k(paste_masks_kernel, dim3(static_cast<unsigned>(tiles), total), 256, smem, as_stream(stream), masks, kept_query, a, mask_threshold, out);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
