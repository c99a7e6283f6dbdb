// Mosaic, random_perspective and mixup of the YOLOX training mapper (MyDatasetMapper2, yolov7/data/dataset_mapper.py:477-767 and
// data_augment.py:31-102) for a whole batch: one launch per stage, one thread per output pixel (all three channels), no atomics.
//
// The arithmetic is OpenCV's (4.x), restated so that the mosaic and the warp match cv2 byte for byte:
//   * cv2.resize(uint8, INTER_LINEAR): source coordinate fx = float((d + 0.5) * (1 / (dst / src)) - 0.5) in double, 11-bit weights, columns
//     clamped to the image, rows clamped only as row indices (the weight stays); the vertical pass is the SIMD one of resize.cpp:
//     ((H0 >> 4) * b0 >> 16) + ((H1 >> 4) * b1 >> 16), then (v + 2) >> 2.  An exact 2x downscale (INTER_AREA inside cv2) gives the same bytes.
//   * cv2.warpAffine(INTER_LINEAR, borderValue 114): the inverted matrix (from the host) in double, AB_BITS = 10, INTER_BITS = 5,
//     15-bit bilinear weights (32 (32 - fy)(32 - fx) ...), taps outside the canvas read 114.
//   * the mixup's float64 cv2.resize: double coordinates (scale = src / dst) and a + (b - a) f interpolation, no fused multiply-add (the
//     __d*_rn intrinsics keep nvcc from contracting), truncated to uint8 like numpy's assignment into a uint8 array.  cv2's float64 path is
//     not restated bit for bit: its values agree to about 1e-12, and a value within that of an integer can truncate to the neighbouring
//     byte.  On random 114-padded canvases this arithmetic truncates differently from cv2 on 9e-6 of the bytes
//     (8.5e-5 with scale = 1 / (dst / src) and weighted sums).
// The tiles are resized to uint8 before the warp samples them (the reference materialises the 2h x 2w canvas); here every warp tap recomputes
// the canvas pixel it reads from the source, with the same rounding.
#include "host_common.cuh"
#include "sm90.cuh"

using namespace yb;

namespace {

constexpr int kAugThreads = 256;
constexpr int kPad = 114;

// source coordinate of destination index d for an ssz -> dsz resize (resize.cpp, computeResizeCoefs of the generic path)
__device__ __forceinline__ void resize_coord(int d, int dsz, int ssz, bool clamp_weight, int& s0, int& s1, float& f) {
  const double scale = 1.0 / (static_cast<double>(dsz) / static_cast<double>(ssz));
  const float fx = __double2float_rn(__dadd_rn(__dmul_rn(static_cast<double>(d) + 0.5, scale), -0.5));
  int s = static_cast<int>(floorf(fx));
  f = __fsub_rn(fx, static_cast<float>(s));
  if (clamp_weight) {
    if (s < 0) { f = 0.f; s = 0; }
    if (s >= ssz - 1) { f = 0.f; s = ssz - 1; }
  }
  s0 = min(max(s, 0), ssz - 1);
  s1 = min(max(s + 1, 0), ssz - 1);
}

// the coordinate of the float64 resize of the mixup, with scale = src / dst (closer to cv2's float64 path than 1 / (dst / src))
__device__ __forceinline__ void resize_coord_f64(int d, int dsz, int ssz, bool clamp_weight, int& s0, int& s1, double& f) {
  const double scale = static_cast<double>(ssz) / static_cast<double>(dsz);
  const double fx = __dadd_rn(__dmul_rn(static_cast<double>(d) + 0.5, scale), -0.5);
  int s = static_cast<int>(floor(fx));
  f = __dadd_rn(fx, -static_cast<double>(s));
  if (clamp_weight) {
    if (s < 0) { f = 0.0; s = 0; }
    if (s >= ssz - 1) { f = 0.0; s = ssz - 1; }
  }
  s0 = min(max(s, 0), ssz - 1);
  s1 = min(max(s + 1, 0), ssz - 1);
}

// pixel (ty, tx) of cv2.resize(src [sh][sw][3], (tw, th), INTER_LINEAR), all three channels
__device__ __forceinline__ void resize_u8_px(const uint8_t* __restrict__ src, int sh, int sw, int th, int tw, int ty, int tx, int v[3]) {
  int x0, x1, y0, y1;
  float fx, fy;
  resize_coord(tx, tw, sw, true, x0, x1, fx);
  resize_coord(ty, th, sh, false, y0, y1, fy);
  const int a0 = __float2int_rn((1.f - fx) * 2048.f), a1 = __float2int_rn(fx * 2048.f);
  const int b0 = __float2int_rn((1.f - fy) * 2048.f), b1 = __float2int_rn(fy * 2048.f);
  const uint8_t* r0 = src + static_cast<size_t>(y0) * sw * 3;
  const uint8_t* r1 = src + static_cast<size_t>(y1) * sw * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int h0 = r0[x0 * 3 + c] * a0 + r0[x1 * 3 + c] * a1;
    const int h1 = r1[x0 * 3 + c] * a0 + r1[x1 * 3 + c] * a1;
    const int s = (((h0 >> 4) * b0) >> 16) + (((h1 >> 4) * b1) >> 16);
    v[c] = min(max((s + 2) >> 2, 0), 255);
  }
}

// pixel (cy, cx) of the 2h x 2w mosaic canvas (114 outside the tiles)
__device__ __forceinline__ void canvas_px(const yb200_mosaic_desc& d, const uint8_t* __restrict__ src, int cy, int cx, int v[3]) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (cx >= d.rect[4 * k] && cy >= d.rect[4 * k + 1] && cx < d.rect[4 * k + 2] && cy < d.rect[4 * k + 3]) {
      resize_u8_px(src + d.src_off[k], d.src_h[k], d.src_w[k], d.tile_h[k], d.tile_w[k], cy - d.pad[2 * k + 1], cx - d.pad[2 * k], v);
      return;
    }
  }
  v[0] = v[1] = v[2] = kPad;
}

// cv2.warpAffine's fixed-point source position of output pixel (x, y), in 1/32 pixel
__device__ __forceinline__ void warp_pos(const double* m, int x, int y, int& X, int& Y) {
  const int ax = __double2int_rn(__dmul_rn(__dmul_rn(m[0], static_cast<double>(x)), 1024.0));
  const int bx = __double2int_rn(__dmul_rn(__dmul_rn(m[3], static_cast<double>(x)), 1024.0));
  const int x0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[1], static_cast<double>(y)), m[2]), 1024.0)) + 16;
  const int y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[4], static_cast<double>(y)), m[5]), 1024.0)) + 16;
  X = (x0 + ax) >> 5;
  Y = (y0 + bx) >> 5;
}

__global__ void __launch_bounds__(kAugThreads)
mosaic_warp_kernel(const yb200_mosaic_desc* __restrict__ table, const uint8_t* __restrict__ src, uint8_t* __restrict__ out) {
  pdl_sync();
  const yb200_mosaic_desc& d = table[blockIdx.y];
  const int npix = d.out_h * d.out_w;
  const int p = blockIdx.x * kAugThreads + threadIdx.x;
  if (p >= npix) return;
  const int y = p / d.out_w, x = p - y * d.out_w;
  uint8_t* o = out + d.out_off + p;
  if (d.mode == 0) {  // pass-through: HWC -> CHW
    const uint8_t* s = src + d.src_off[0] + static_cast<size_t>(p) * 3;
    o[0] = s[0];
    o[npix] = s[1];
    o[2 * npix] = s[2];
    return;
  }
  int X, Y;
  warp_pos(d.minv, x, y, X, Y);
  const int sx = min(max(X >> 5, -32768), 32767), sy = min(max(Y >> 5, -32768), 32767);  // cv2 keeps the integer part as short
  const int fx = X & 31, fy = Y & 31;
  const int ch = 2 * d.in_h, cw = 2 * d.in_w;
  int acc[3] = {1 << 14, 1 << 14, 1 << 14};
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int ty = sy + (t >> 1), tx = sx + (t & 1);
    const int wgt = ((t >> 1) ? fy : 32 - fy) * ((t & 1) ? fx : 32 - fx) * 32;
    int v[3] = {kPad, kPad, kPad};
    if (ty >= 0 && ty < ch && tx >= 0 && tx < cw) canvas_px(d, src, ty, tx, v);
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] += v[c] * wgt;
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c * npix] = static_cast<uint8_t>(min(max(acc[c] >> 15, 0), 255));
}

// pixel (jy, jx) of the jittered mixup canvas: the float64 resize of the in_h x in_w canvas (the uint8-resized source at the top left, 114
// elsewhere) to jit_h x jit_w, truncated to uint8
__device__ __forceinline__ void jitter_px(const yb200_mosaic_desc& d, const uint8_t* __restrict__ msrc, int jy, int jx, int v[3]) {
  int x0, x1, y0, y1;
  double fx, fy;
  resize_coord_f64(jx, d.jit_w, d.in_w, true, x0, x1, fx);
  resize_coord_f64(jy, d.jit_h, d.in_h, false, y0, y1, fy);
  double tap[4][3];
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int cy = (t >> 1) ? y1 : y0, cx = (t & 1) ? x1 : x0;
    int u[3] = {kPad, kPad, kPad};
    if (cy < d.mix_h && cx < d.mix_w) resize_u8_px(msrc, d.src_h[4], d.src_w[4], d.mix_h, d.mix_w, cy, cx, u);
#pragma unroll
    for (int c = 0; c < 3; ++c) tap[t][c] = static_cast<double>(u[c]);
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {  // a + (b - a) f: exact where the taps are equal, as cv2's float64 result is there
    const double h0 = __dadd_rn(tap[0][c], __dmul_rn(__dsub_rn(tap[1][c], tap[0][c]), fx));
    const double h1 = __dadd_rn(tap[2][c], __dmul_rn(__dsub_rn(tap[3][c], tap[2][c]), fx));
    const double r = __dadd_rn(h0, __dmul_rn(__dsub_rn(h1, h0), fy));
    v[c] = min(max(static_cast<int>(r), 0), 255);
  }
}

__global__ void __launch_bounds__(kAugThreads)
mosaic_mixup_kernel(const yb200_mosaic_desc* __restrict__ table, const uint8_t* __restrict__ src, uint8_t* __restrict__ out) {
  pdl_sync();
  const yb200_mosaic_desc& d = table[blockIdx.y];
  if (d.mode != 1 || !d.mix) return;
  const int npix = d.out_h * d.out_w;
  const int p = blockIdx.x * kAugThreads + threadIdx.x;
  if (p >= npix) return;
  const int y = p / d.out_w, x = p - y * d.out_w;
  const int py = y + d.y_off, px = x + d.x_off;  // position in the zero-padded, flipped jittered canvas
  int v[3] = {0, 0, 0};
  if (py < d.jit_h && px < d.jit_w) jitter_px(d, src + d.src_off[4], py, d.flip ? d.jit_w - 1 - px : px, v);
  uint8_t* o = out + d.out_off + p;
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c * npix] = static_cast<uint8_t>((o[c * npix] + v[c]) >> 1);  // float32 0.5 a + 0.5 b, truncated
}

int check_args(const yb200_mosaic_desc* table, int n, const uint8_t* src, const uint8_t* out, int max_h, int max_w, const char* what) {
  YB_REQUIRE(table && src && out, YB200_ERR_INVALID, "%s: null pointer", what);
  YB_REQUIRE(n > 0 && n <= 65535, YB200_ERR_INVALID, "%s: batch of %d samples (1..65535)", what, n);
  YB_REQUIRE(max_h > 0 && max_w > 0 && max_h <= 16384 && max_w <= 16384, YB200_ERR_INVALID, "%s: output size %dx%d", what, max_h, max_w);
  return 0;
}

}  // namespace

extern "C" int yb200_mosaic_warp(const yb200_mosaic_desc* table_dev, int n, const uint8_t* src, uint8_t* out, int max_h, int max_w,
                                 void* stream) {
  if (int rc = check_args(table_dev, n, src, out, max_h, max_w, "mosaic_warp")) return rc;
  const dim3 grid(ceil_div(max_h * max_w, kAugThreads), n);
  YB_CHECK_CUDA(launch_k(mosaic_warp_kernel, grid, kAugThreads, 0, as_stream(stream), table_dev, src, out));
  return 0;
}

extern "C" int yb200_mosaic_mixup(const yb200_mosaic_desc* table_dev, int n, const uint8_t* src, uint8_t* out, int max_h, int max_w,
                                  void* stream) {
  if (int rc = check_args(table_dev, n, src, out, max_h, max_w, "mosaic_mixup")) return rc;
  const dim3 grid(ceil_div(max_h * max_w, kAugThreads), n);
  YB_CHECK_CUDA(launch_k(mosaic_mixup_kernel, grid, kAugThreads, 0, as_stream(stream), table_dev, src, out));
  return 0;
}
