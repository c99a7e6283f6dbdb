#include "host_common.cuh"

#include <mutex>

namespace yb {

static thread_local char g_err[1024] = "";

char* err_buf() { return g_err; }

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int current_device() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  return dev;
}

int sm_count() {
  static int n[64] = {0};
  const int dev = current_device() & 63;
  if (n[dev] == 0) {
    if (cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n[dev] <= 0) n[dev] = 132;
  }
  return n[dev];
}

int check_act(const yb200_act* a, const char* name, int mult) {
  YB_REQUIRE(a != nullptr && a->ptr != nullptr, YB200_ERR_INVALID, "%s: null view", name);
  YB_REQUIRE(a->n > 0 && a->h > 0 && a->w > 0 && a->c > 0, YB200_ERR_INVALID, "%s: empty extent (%dx%dx%dx%d)", name, a->n, a->h, a->w, a->c);
  YB_REQUIRE(a->c % mult == 0 && a->c_pitch % mult == 0 && a->c_off % mult == 0 && a->c_off + a->c <= a->c_pitch, YB200_ERR_INVALID,
             "%s: channels (c=%d pitch=%d off=%d) must be multiples of %d with off+c<=pitch", name, a->c, a->c_pitch, a->c_off, mult);
  return 0;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

static CUtensorMapSwizzle swizzle_for(int inner_bytes) {
  return inner_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
         : inner_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
         : inner_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                             : CU_TENSOR_MAP_SWIZZLE_NONE;
}

int make_act_map(CUtensorMap* m, const yb200_act& a, bool s2d, int box_c, int tw, int th, int tn) {
  EncodeTiledFn fn = encode_fn();
  YB_REQUIRE(fn != nullptr, YB200_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  YB_REQUIRE(box_c == 16 || box_c == 32 || box_c == 64, YB200_ERR_INVALID, "activation box width %d", box_c);
  YB_REQUIRE((reinterpret_cast<uintptr_t>(a.ptr) & 15) == 0 && a.c_pitch % 8 == 0, YB200_ERR_INVALID,
             "activation buffer must be 16B aligned with a channel pitch multiple of 8");
  const cuuint64_t pitch = static_cast<cuuint64_t>(a.c_pitch) * 2;  // bytes per pixel
  cuuint64_t gdim[5], gstr[4];
  if (!s2d) {
    gdim[0] = a.c_pitch; gdim[1] = a.w; gdim[2] = 1; gdim[3] = a.h; gdim[4] = a.n;
    gstr[0] = pitch; gstr[1] = pitch * a.w; gstr[2] = pitch * a.w; gstr[3] = pitch * a.w * a.h;
  } else {
    YB_REQUIRE(a.h % 2 == 0 && a.w % 2 == 0, YB200_ERR_UNSUPPORTED, "stride-2 view needs even h,w (got %dx%d)", a.h, a.w);
    gdim[0] = 2 * a.c_pitch; gdim[1] = a.w / 2; gdim[2] = 2; gdim[3] = a.h / 2; gdim[4] = a.n;
    gstr[0] = 2 * pitch; gstr[1] = pitch * a.w; gstr[2] = 2 * pitch * a.w; gstr[3] = pitch * a.w * a.h;
  }
  cuuint32_t box[5] = {static_cast<cuuint32_t>(box_c), static_cast<cuuint32_t>(tw), 1u, static_cast<cuuint32_t>(th),
                       static_cast<cuuint32_t>(tn)};
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, a.ptr, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle_for(box_c * 2), CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  YB_REQUIRE(r == CUDA_SUCCESS, YB200_ERR_CUDA,
             "cuTensorMapEncodeTiled(act n=%d h=%d w=%d pitch=%d box=%d,%d,%d,%d) failed: %d", a.n, a.h, a.w, a.c_pitch,
             box_c, tw, th, tn, static_cast<int>(r));
  return 0;
}

int make_mat_map(CUtensorMap* m, const void* ptr, long long rows, long long cols, int box_rows, int box_cols) {
  EncodeTiledFn fn = encode_fn();
  YB_REQUIRE(fn != nullptr, YB200_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  YB_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && cols % 8 == 0, YB200_ERR_INVALID,
             "matrix must be 16B aligned with a row length multiple of 8");
  cuuint64_t gdim[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t gstr[1] = {static_cast<cuuint64_t>(cols) * 2};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim, gstr, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(box_cols * 2), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  YB_REQUIRE(r == CUDA_SUCCESS, YB200_ERR_CUDA, "cuTensorMapEncodeTiled(mat %lldx%lld box %dx%d) failed: %d", rows, cols,
             box_rows, box_cols, static_cast<int>(r));
  return 0;
}

int make_pix_map(CUtensorMap* m, const void* base, int c, int w, int h, int n, long long sx, long long sy, long long sn, int box_c, int bw, int bh,
                 int bn) {
  EncodeTiledFn fn = encode_fn();
  YB_REQUIRE(fn != nullptr, YB200_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  YB_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0 && sx % 8 == 0 && sy % 8 == 0 && sn % 8 == 0, YB200_ERR_INVALID,
             "16-bit pixel view must start 16B aligned with strides that are multiples of 8 elements (strides %lld, %lld, %lld)", sx, sy, sn);
  cuuint64_t gdim[4] = {static_cast<cuuint64_t>(c), static_cast<cuuint64_t>(w), static_cast<cuuint64_t>(h), static_cast<cuuint64_t>(n)};
  cuuint64_t gstr[3] = {static_cast<cuuint64_t>(sx) * 2, static_cast<cuuint64_t>(sy) * 2, static_cast<cuuint64_t>(sn) * 2};
  cuuint32_t box[4] = {static_cast<cuuint32_t>(box_c), static_cast<cuuint32_t>(bw), static_cast<cuuint32_t>(bh), static_cast<cuuint32_t>(bn)};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT16, 4, const_cast<void*>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle_for(box_c * 2), CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  YB_REQUIRE(r == CUDA_SUCCESS, YB200_ERR_CUDA, "cuTensorMapEncodeTiled(pixels c=%d w=%d h=%d n=%d box=%d,%d,%d,%d) failed: %d", c, w, h, n,
             box_c, bw, bh, bn, static_cast<int>(r));
  return 0;
}

void choose_tile(int n, int h, int w, int npix, int* log_tw, int* log_th) {
  const int lp = ilog2(npix);
  long long best = -1;
  int bw = 0, bh = 0;
  for (int lw = lp; lw >= 0; --lw) {
    for (int lh = lp - lw; lh >= 0; --lh) {
      const int tw = 1 << lw, th = 1 << lh, tn = npix >> (lw + lh);
      const long long cost = 1LL * ceil_div(w, tw) * tw * ceil_div(h, th) * th * ceil_div(n, tn) * tn;
      if (best < 0 || cost < best) {  // ties keep the widest / tallest tile (longest contiguous runs)
        best = cost; bw = lw; bh = lh;
      }
    }
  }
  *log_tw = bw;
  *log_th = bh;
}

}  // namespace yb

extern "C" int yb200_version(void) { return YB200_VERSION; }
extern "C" const char* yb200_last_error(void) { return yb::err_buf(); }
