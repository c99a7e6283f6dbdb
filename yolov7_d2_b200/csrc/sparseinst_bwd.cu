// Backward kernels of the SparseInst IAM decoders (yolov7/modeling/transcoders/decoder_sparseinst.py:27-250) that are not GEMMs: the adjoint
// of the bilinear x2 up-sampling of the mask logits, the backward of the instance normalisation inst = raw / max(sum prob, 1e-6), and the
// sigmoid backward of the instance activation maps.  Everything else of the decoder backward is convolution data / weight gradients and column
// sums (conv_api.cu, convnext.cu).  Every sum runs in a fixed order and there are no atomics: the results are bit-reproducible.
#include "host_common.cuh"
#include "sm90.cuh"

#include <algorithm>

using namespace yb;

namespace {

// weight of input row `y` in output row `o` of yb200_upsample_bilinear2x_f32 (ATen's align_corners=False x2: source (o + 0.5) / 2 - 0.5,
// negative coordinates clamped to 0, the upper neighbour clamped to the last row)
__device__ __forceinline__ float up2x_weight(int o, int y, int h) {
  const int yy = o >> 1;
  const int y0 = (o & 1) ? yy : max(yy - 1, 0);
  const int y1 = min(y0 + 1, h - 1);
  const float l = (o & 1) ? 0.25f : (yy == 0 ? 0.f : 0.75f);
  return (y0 == y ? 1.f - l : 0.f) + (y1 == y ? l : 0.f);
}

constexpr int kUpPix = 32;  // pixels of one row per CTA (one per lane)
constexpr int kUpCh = 64;   // channels per pass: 8 warps x 8 channels

// dx[n][y][x][c] = sum over the (up to) 4 x 4 outputs that read input (y, x) of weight * dout[n][c][oy][ox], rows then columns in ascending
// order; channels c >= maps are written as 0.  Each warp computes 8 channels of 32 pixels (lane = pixel); the CTA's [32 pixels][64 channels]
// tile is transposed in shared memory so that every pixel's channels are stored as 16-byte chunks.
__global__ void __launch_bounds__(256) upsample_bilinear2x_bwd_kernel(const float* __restrict__ dout, int maps, int h, int w, __nv_bfloat16* __restrict__ dx,
                                                                      int c, int pitch) {
  pdl_sync();
  __shared__ __align__(16) __nv_bfloat16 tile[kUpPix][kUpCh + 8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int x = blockIdx.x * kUpPix + lane, y = blockIdx.y, n = blockIdx.z;
  const int W2 = 2 * w;
  const int oy0 = max(2 * y - 1, 0), oy1 = min(2 * y + 2, 2 * h - 1);
  const int ox0 = max(2 * x - 1, 0), ox1 = min(2 * x + 2, W2 - 1);
  for (int c0 = 0; c0 < c; c0 += kUpCh) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int ch = c0 + warp * 8 + j;
      float acc = 0.f;
      if (ch < maps && x < w) {
        const float* g = dout + (static_cast<size_t>(n) * maps + ch) * (2LL * h) * W2;
        for (int oy = oy0; oy <= oy1; ++oy) {
          const float wy = up2x_weight(oy, y, h);
          float row = 0.f;
          for (int ox = ox0; ox <= ox1; ++ox) row += up2x_weight(ox, x, w) * g[static_cast<size_t>(oy) * W2 + ox];
          acc += wy * row;
        }
      }
      tile[lane][warp * 8 + j] = __float2bfloat16_rn(acc);
    }
    __syncthreads();
    const int p = threadIdx.x >> 3, q = threadIdx.x & 7;  // pixel, 8-channel chunk
    const int px = blockIdx.x * kUpPix + p;
    if (px < w && c0 + q * 8 < c)
      *reinterpret_cast<uint4*>(dx + ((static_cast<size_t>(n) * h + y) * w + px) * pitch + c0 + q * 8) = *reinterpret_cast<const uint4*>(&tile[p][q * 8]);
    __syncthreads();
  }
}

constexpr int kNbRows = 32;  // raw rows per CTA (4 per warp)

// Backward of inst[r][c] = raw[r][c] / max(norm[r], 1e-6) for every image: G (the gradient of inst, bf16) is read through the row map
// r -> (r % rows_per_group, (r / rows_per_group) * cols) of the [rows / rows_per_group * cols]-wide gradient view, so the grouped decoder's
// reshape(B, G, N, C).transpose(1, 2) needs no relayout.  Writes d raw = G / max(norm, 1e-6) as bf16 [rows][cols] and [cols][rows] (the
// transpose through shared memory) and d norm = -sum_c d raw * raw / max(norm, 1e-6) (= -sum_c G raw / max(norm, 1e-6)^2; 0 where the clamp is
// active, norm < 1e-6), fp32.  d norm is summed from the STORED bf16 d raw: the aggregation backward then sees operands for which the exact
// identity sum_p prob_p (F_p . d raw + d norm) = 0 of the normalisation (a common scale of the probabilities does not change inst) still holds,
// so the IAM convolution's gradients do not inherit the bf16 rounding of d raw through that large cancellation.
__global__ void __launch_bounds__(256) iam_normalize_bwd_kernel(const __nv_bfloat16* __restrict__ g, long long g_sn, int g_pitch, int g_rows,
                                                                const float* __restrict__ raw, const float* __restrict__ norm, int rows, int cols,
                                                                int rows_per_group, __nv_bfloat16* __restrict__ draw, __nv_bfloat16* __restrict__ draw_t,
                                                                float* __restrict__ dnorm) {
  pdl_sync();
  extern __shared__ __align__(16) __nv_bfloat16 s_d[];  // [kNbRows][cols + 2]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.y, r0 = blockIdx.x * kNbRows;
  const int sp = cols + 2;
  for (int j = 0; j < kNbRows / 8; ++j) {
    const int rl = warp * (kNbRows / 8) + j, r = r0 + rl;
    if (r >= rows) break;
    const int i = r % rows_per_group, k = r / rows_per_group;
    const __nv_bfloat16* gr = i < g_rows ? g + b * g_sn + static_cast<long long>(i) * g_pitch + static_cast<long long>(k) * cols : nullptr;
    const float* rr = raw + (static_cast<long long>(b) * rows + r) * cols;
    const float nv = norm[static_cast<long long>(b) * rows + r];
    const float m = fmaxf(nv, 1e-6f);
    float s = 0.f;
    for (int cc = lane; cc < cols; cc += 32) {
      const float gv = gr ? __bfloat162float(gr[cc]) : 0.f;
      const __nv_bfloat16 d = __float2bfloat16_rn(gv / m);
      s += __bfloat162float(d) * rr[cc];
      draw[(static_cast<long long>(b) * rows + r) * cols + cc] = d;
      s_d[rl * sp + cc] = d;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) dnorm[static_cast<long long>(b) * rows + r] = nv >= 1e-6f ? -s / m : 0.f;
  }
  __syncthreads();
  const int nr = min(kNbRows, rows - r0);
  for (int cc = warp; cc < cols; cc += 8)
    if (lane < nr) draw_t[(static_cast<long long>(b) * cols + cc) * rows + r0 + lane] = s_d[lane * sp + cc];
}

struct View {
  const __nv_bfloat16* p;
  int c, pitch;
};

// dx[.., k * group_out + i] = i < group_in ? dy[.., k * group_in + i] * sigmoid'(x[.., k * group_in + i]) : 0, sigmoid' = e / (1 + e)^2 with
// e = exp(-|x|) in fp32 (1 - p of a rounded p near 1 would be too coarse)
__global__ void __launch_bounds__(256) sigmoid_bwd_kernel(View dy, View x, __nv_bfloat16* __restrict__ dx, int dx_c, int dx_pitch, int group_in,
                                                          int group_out, long long npix) {
  pdl_sync();
  const int chunks = dx_c >> 3;
  const long long total = npix * chunks;
  for (long long t = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; t < total; t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long pix = t / chunks;
    const int o = static_cast<int>(t - pix * chunks) * 8;
    const int k = o / group_out, i = o - k * group_out;
    uint4 out = make_uint4(0u, 0u, 0u, 0u);
    if (i < group_in) {
      const int ci = k * group_in + i;
      const uint4 a = *reinterpret_cast<const uint4*>(dy.p + pix * dy.pitch + ci);
      const uint4 v = *reinterpret_cast<const uint4*>(x.p + pix * x.pitch + ci);
      auto f = [](float d, float z) {
        const float e = expf(-fabsf(z));
        const float q = 1.f + e;
        return d * (e / (q * q));
      };
      out.x = pack_bf16x2(f(bf16_lo(a.x), bf16_lo(v.x)), f(bf16_hi(a.x), bf16_hi(v.x)));
      out.y = pack_bf16x2(f(bf16_lo(a.y), bf16_lo(v.y)), f(bf16_hi(a.y), bf16_hi(v.y)));
      out.z = pack_bf16x2(f(bf16_lo(a.z), bf16_lo(v.z)), f(bf16_hi(a.z), bf16_hi(v.z)));
      out.w = pack_bf16x2(f(bf16_lo(a.w), bf16_lo(v.w)), f(bf16_hi(a.w), bf16_hi(v.w)));
    }
    *reinterpret_cast<uint4*>(dx + pix * dx_pitch + o) = out;
  }
}

}  // namespace

extern "C" int yb200_upsample_bilinear2x_bwd_f32(const float* dout, int maps, const yb200_act* dx, void* stream) {
  int rc;
  if ((rc = check_act(dx, "upsample_bilinear2x_bwd_f32 dx"))) return rc;
  YB_REQUIRE(dout != nullptr, YB200_ERR_INVALID, "upsample_bilinear2x_bwd_f32: null dout");
  YB_REQUIRE(maps > 0 && maps <= dx->c, YB200_ERR_INVALID, "upsample_bilinear2x_bwd_f32: %d maps for a %d-channel dx", maps, dx->c);
  YB_REQUIRE(dx->h <= 65535 && dx->n <= 65535, YB200_ERR_UNSUPPORTED, "upsample_bilinear2x_bwd_f32: %d images of %d rows", dx->n, dx->h);
  __nv_bfloat16* out = static_cast<__nv_bfloat16*>(dx->ptr) + dx->c_off;
  launch_k(upsample_bilinear2x_bwd_kernel, dim3(ceil_div(dx->w, kUpPix), dx->h, dx->n), 256, 0, as_stream(stream), dout, maps, dx->h, dx->w, out, dx->c,
           dx->c_pitch);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_iam_normalize_bwd(const yb200_act* g, const float* raw, const float* normalizer, int rows, int cols, int rows_per_group, void* draw,
                                       void* draw_t, float* dnorm, void* stream) {
  int rc;
  if ((rc = check_act(g, "iam_normalize_bwd g"))) return rc;
  YB_REQUIRE(raw && normalizer && draw && draw_t && dnorm, YB200_ERR_INVALID, "iam_normalize_bwd: null pointer");
  YB_REQUIRE(rows > 0 && cols > 0 && rows_per_group > 0 && rows % rows_per_group == 0, YB200_ERR_INVALID,
             "iam_normalize_bwd: %d rows in groups of %d", rows, rows_per_group);
  YB_REQUIRE(g->h == 1 && g->c == rows / rows_per_group * cols, YB200_ERR_INVALID, "iam_normalize_bwd: g must be a [n][1][rows][%d] view (got %dx%dx%dx%d)",
             rows / rows_per_group * cols, g->n, g->h, g->w, g->c);
  YB_REQUIRE(cols <= 2048 && g->n <= 65535, YB200_ERR_UNSUPPORTED, "iam_normalize_bwd: %d columns, %d images", cols, g->n);
  const int smem = kNbRows * (cols + 2) * 2;
  static PerDevice<int> smem_limit(48 * 1024);
  YB_CHECK_CUDA(raise_smem_limit(smem_limit, smem, iam_normalize_bwd_kernel));
  launch_k(iam_normalize_bwd_kernel, dim3(ceil_div(rows, kNbRows), g->n), 256, smem, as_stream(stream), static_cast<const __nv_bfloat16*>(g->ptr) + g->c_off,
           1LL * g->w * g->c_pitch, g->c_pitch, g->w, raw, normalizer, rows, cols, rows_per_group, static_cast<__nv_bfloat16*>(draw),
           static_cast<__nv_bfloat16*>(draw_t), dnorm);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_sigmoid_bwd(const yb200_act* dy, const yb200_act* x, const yb200_act* dx, int group_in, int group_out, void* stream) {
  int rc;
  if ((rc = check_act(dy, "sigmoid_bwd dy"))) return rc;
  if ((rc = check_act(x, "sigmoid_bwd x"))) return rc;
  if ((rc = check_act(dx, "sigmoid_bwd dx"))) return rc;
  YB_REQUIRE(same_shape(dy, x), YB200_ERR_INVALID, "sigmoid_bwd: dy and x shapes differ");
  YB_REQUIRE(group_in > 0 && group_in % 8 == 0 && group_out % 8 == 0 && group_in <= group_out && dx->c % group_out == 0 &&
                 dy->c == dx->c / group_out * group_in,
             YB200_ERR_INVALID, "sigmoid_bwd: groups of %d -> %d channels do not map %d onto %d channels", group_in, group_out, dy->c, dx->c);
  YB_REQUIRE(dx->n == dy->n && dx->h == dy->h && dx->w == dy->w, YB200_ERR_INVALID, "sigmoid_bwd: dx pixel grid differs from dy");
  const long long npix = 1LL * dx->n * dx->h * dx->w;
  const long long total = npix * (dx->c / 8);
  const int blocks = static_cast<int>(std::min<long long>((total + 255) / 256, 16LL * sm_count()));
  launch_k(sigmoid_bwd_kernel, blocks, 256, 0, as_stream(stream), View{static_cast<const __nv_bfloat16*>(dy->ptr) + dy->c_off, dy->c, dy->c_pitch},
           View{static_cast<const __nv_bfloat16*>(x->ptr) + x->c_off, x->c, x->c_pitch}, static_cast<__nv_bfloat16*>(dx->ptr) + dx->c_off, dx->c, dx->c_pitch,
           group_in, group_out, npix);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
