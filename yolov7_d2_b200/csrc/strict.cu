// STRICT mode (YB200_STRICT / YoloxEngine(strict=True)): the forward pass of the YOLOX path with fp32-grade arithmetic, for the
// north_star check "fp32 losses and logits within 1e-3 relative" against the fp32 reference.
//
// Activations are stored as SPLIT bf16 planes: a = a0 + a1 [+ a2] with a0 = bf16(a), a1 = bf16(a - a0), a2 = bf16(a - a0 - a1) -- 16 significant
// bits with two planes, all 24 bits of the fp32 value with three (the default) --, the planes `lo_delta` channels apart in one NHWC buffer, so every channel-slice view (torch.cat / Focus / upsample
// fusions of the fast path) keeps working and the SAME wgmma implicit-GEMM kernel computes the partial products a_i * w_j (i + j < planes) into one fp32
// accumulator (conv_api.cu: yb200_conv2d_fwd_split).  The pre-BatchNorm convolution output z stays in fp32.  The kernels here
// are the element-wise stages around that GEMM; they are a verification mode, written for clarity, not for speed.
#include <algorithm>

#include "host_common.cuh"
#include "sm90.cuh"

using namespace yb;

namespace {

struct SplitView {  // device-side view of a split activation: plane j at p + j * lo, value = sum of the planes
  __nv_bfloat16* p;
  int n, h, w, c, pitch, lo, planes;
};

int mk_split(const yb200_act* a, int lo_delta, int planes, const char* name, SplitView* v) {
  if (const int rc = check_act(a, name, 1)) return rc;
  YB_REQUIRE((planes == 2 || planes == 3) && lo_delta > 0 && a->c_off + (planes - 1) * lo_delta + a->c <= a->c_pitch, YB200_ERR_INVALID,
             "%s: plane %d [%d, %d) outside the pitch %d", name, planes - 1, a->c_off + (planes - 1) * lo_delta,
             a->c_off + (planes - 1) * lo_delta + a->c, a->c_pitch);
  v->p = static_cast<__nv_bfloat16*>(a->ptr) + a->c_off;
  v->n = a->n; v->h = a->h; v->w = a->w; v->c = a->c; v->pitch = a->c_pitch; v->lo = lo_delta; v->planes = planes;
  return 0;
}

__device__ __forceinline__ float split_load(const SplitView& v, long long pix, int ch) {
  const __nv_bfloat16* q = v.p + pix * v.pitch + ch;
  float a = __bfloat162float(q[0]) + __bfloat162float(q[v.lo]);  // exact in fp32 (16 significant bits)
  if (v.planes == 3) a += __bfloat162float(q[2 * v.lo]);          // exact: the three planes are the 24 bits of one fp32 value
  return a;
}
__device__ __forceinline__ void split_store(const SplitView& v, long long pix, int ch, float a) {
  __nv_bfloat16* q = v.p + pix * v.pitch + ch;
  for (int pl = 0; pl < v.planes; ++pl) {
    const __nv_bfloat16 h = __float2bfloat16_rn(a);
    q[pl * v.lo] = h;
    a -= __bfloat162float(h);
  }
}

// per-channel sum / sum of squares of an fp32 NHWC slice, fp64 accumulation (block partials, then one atomic per channel and block)
__global__ void strict_bn_stats_kernel(const float* __restrict__ z, long long npix, int pitch, int c, double* __restrict__ sum,
                                       double* __restrict__ sq) {
  pdl_sync();
  // blockDim = (32 channels, 8 pixel rows); grid = (channel groups, pixel blocks)
  const int ch = blockIdx.x * 32 + threadIdx.x;
  __shared__ double s1[8][32], s2[8][32];
  double a = 0.0, b = 0.0;
  if (ch < c) {
    for (long long pix = blockIdx.y * 8LL + threadIdx.y; pix < npix; pix += 8LL * gridDim.y) {
      const double v = static_cast<double>(z[pix * pitch + ch]);
      a += v;
      b += v * v;
    }
  }
  s1[threadIdx.y][threadIdx.x] = a;
  s2[threadIdx.y][threadIdx.x] = b;
  __syncthreads();
  if (threadIdx.y == 0 && ch < c) {
    for (int r = 1; r < 8; ++r) { a += s1[r][threadIdx.x]; b += s2[r][threadIdx.x]; }
    atomicAdd(sum + ch, a);
    atomicAdd(sq + ch, b);
  }
}

// a = SiLU(z*scale + shift) [+ residual], written as a split pair; optionally also 2x nearest-upsampled into `up`
__global__ void strict_bn_apply_silu_kernel(const float* __restrict__ z, int z_pitch, const float* __restrict__ scale,
                                            const float* __restrict__ shift, SplitView res, int has_res, SplitView out, SplitView up, int has_up) {
  pdl_sync();
  const long long total = 1LL * out.n * out.h * out.w * out.c;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ch = static_cast<int>(i % out.c);
    const long long pix = i / out.c;
    const float u = fmaf(z[pix * z_pitch + ch], scale[ch], shift[ch]);
    float a = u / (1.f + expf(-u));  // x * sigmoid(x), as nn.SiLU
    if (has_res) a += split_load(res, pix, ch);
    split_store(out, pix, ch, a);
    if (has_up) {
      const int x = static_cast<int>(pix % out.w);
      const int y = static_cast<int>((pix / out.w) % out.h);
      const long long b = pix / (1LL * out.w * out.h);
      const long long p00 = (b * up.h + 2 * y) * up.w + 2 * x;
      split_store(up, p00, ch, a);
      split_store(up, p00 + 1, ch, a);
      split_store(up, p00 + up.w, ch, a);
      split_store(up, p00 + up.w + 1, ch, a);
    }
  }
}

// SPP max-pools k = 5, 9, 13 (stride 1, -inf padding) on the reconstructed fp32 values
__global__ void strict_spp_pool_kernel(SplitView x, SplitView o5, SplitView o9, SplitView o13) {
  pdl_sync();
  const long long total = 1LL * x.n * x.h * x.w * x.c;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ch = static_cast<int>(i % x.c);
    const long long pix = i / x.c;
    const int px = static_cast<int>(pix % x.w);
    const int py = static_cast<int>((pix / x.w) % x.h);
    const long long b = pix / (1LL * x.w * x.h);
    float m5 = -INFINITY, m9 = -INFINITY, m13 = -INFINITY;
    for (int dy = -6; dy <= 6; ++dy) {
      const int yy = py + dy;
      if (yy < 0 || yy >= x.h) continue;
      for (int dx = -6; dx <= 6; ++dx) {
        const int xx = px + dx;
        if (xx < 0 || xx >= x.w) continue;
        const float v = split_load(x, (b * x.h + yy) * x.w + xx, ch);
        const int r = max(abs(dy), abs(dx));
        m13 = fmaxf(m13, v);
        if (r <= 4) m9 = fmaxf(m9, v);
        if (r <= 2) m5 = fmaxf(m5, v);
      }
    }
    split_store(o5, pix, ch, m5);
    split_store(o9, pix, ch, m9);
    split_store(o13, pix, ch, m13);
  }
}

int grid_for(long long work, int threads) {
  const long long b = (work + threads - 1) / threads;
  return static_cast<int>(std::max<long long>(1, std::min<long long>(b, 64LL * sm_count())));
}

}  // namespace

extern "C" int yb200_strict_bn_stats(const float* z, int64_t npix, int z_pitch, int z_off, int c, double* stat_sum, double* stat_sqsum,
                                     void* stream) {
  YB_REQUIRE(z && stat_sum && stat_sqsum && npix > 0 && c > 0 && z_off >= 0 && z_off + c <= z_pitch, YB200_ERR_INVALID,
             "strict_bn_stats: bad arguments (npix=%lld c=%d off=%d pitch=%d)", (long long)npix, c, z_off, z_pitch);
  const int gy = static_cast<int>(std::min<long long>((npix + 7) / 8, 8LL * sm_count()));
  launch_k(strict_bn_stats_kernel, dim3(ceil_div(c, 32), gy), dim3(32, 8), 0, as_stream(stream), z + z_off, npix, z_pitch, c, stat_sum, stat_sqsum);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_strict_bn_apply_silu(const float* z, int z_pitch, int z_off, const float* scale, const float* shift,
                                          const yb200_act* residual, int residual_lo, const yb200_act* out, int out_lo,
                                          const yb200_act* out_up2x, int up_lo, int planes, void* stream) {
  int rc;
  SplitView vo, vr, vu;
  YB_REQUIRE(z && scale && shift && out, YB200_ERR_INVALID, "strict_bn_apply_silu: null pointer");
  if ((rc = mk_split(out, out_lo, planes, "strict_bn_apply_silu out", &vo))) return rc;
  YB_REQUIRE(z_off >= 0 && z_off + out->c <= z_pitch, YB200_ERR_INVALID, "strict_bn_apply_silu: z slice outside its pitch");
  vr = vo; vu = vo;
  if (residual) {
    if ((rc = mk_split(residual, residual_lo, planes, "strict_bn_apply_silu residual", &vr))) return rc;
    YB_REQUIRE(residual->n == out->n && residual->h == out->h && residual->w == out->w && residual->c == out->c, YB200_ERR_INVALID,
               "strict_bn_apply_silu: residual shape mismatch");
  }
  if (out_up2x) {
    if ((rc = mk_split(out_up2x, up_lo, planes, "strict_bn_apply_silu out_up2x", &vu))) return rc;
    YB_REQUIRE(out_up2x->n == out->n && out_up2x->h == 2 * out->h && out_up2x->w == 2 * out->w && out_up2x->c == out->c, YB200_ERR_INVALID,
               "strict_bn_apply_silu: upsampled view must be [n,2h,2w,c]");
  }
  const long long total = 1LL * out->n * out->h * out->w * out->c;
  launch_k(strict_bn_apply_silu_kernel, grid_for(total, 256), 256, 0, as_stream(stream), z + z_off, z_pitch, scale, shift, vr, residual != nullptr, vo, vu,
                                                                                  out_up2x != nullptr);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_strict_spp_pool(const yb200_act* x, const yb200_act* o5, const yb200_act* o9, const yb200_act* o13, int lo_delta, int planes,
                                     void* stream) {
  int rc;
  SplitView vx, v5, v9, v13;
  if ((rc = mk_split(x, lo_delta, planes, "strict_spp_pool x", &vx)) || (rc = mk_split(o5, lo_delta, planes, "strict_spp_pool o5", &v5)) ||
      (rc = mk_split(o9, lo_delta, planes, "strict_spp_pool o9", &v9)) || (rc = mk_split(o13, lo_delta, planes, "strict_spp_pool o13", &v13)))
    return rc;
  YB_REQUIRE(o5->c == x->c && o9->c == x->c && o13->c == x->c && o5->h == x->h && o5->w == x->w, YB200_ERR_INVALID, "strict_spp_pool: shape mismatch");
  const long long total = 1LL * x->n * x->h * x->w * x->c;
  launch_k(strict_spp_pool_kernel, grid_for(total, 128), 128, 0, as_stream(stream), vx, v5, v9, v13);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
