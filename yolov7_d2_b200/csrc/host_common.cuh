// Host-side helpers shared by the C-ABI translation units: error reporting, TMA descriptor encoding,
// tile selection.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <utility>

#include "../../include/yb200.h"

namespace yb {

char* err_buf();
int fail(int code, const char* fmt, ...);
int sm_count();  // of the CURRENT device
int current_device();
// function attributes (dynamic shared memory limits) are per device: caches of "already raised to N bytes" must be too
template <typename T>
struct PerDevice {
  T v[64];
  T init;
  bool used[64];
  explicit PerDevice(T init_value) : init(init_value) { memset(used, 0, sizeof(used)); }
  T& cur() {
    const int d = current_device() & 63;
    if (!used[d]) { v[d] = init; used[d] = true; }
    return v[d];
  }
};

// Kernels that take more dynamic shared memory than the default must opt in with a function attribute.  Raises the limit of every kernel
// in `kernels` to `bytes` when that exceeds what `limit` records for the current device; `limit` is the call site's static cache.
template <typename... K>
inline cudaError_t raise_smem_limit(PerDevice<int>& limit, int bytes, K*... kernels) {
  int& cur = limit.cur();
  if (bytes <= cur) return cudaSuccess;
  cudaError_t e = cudaSuccess;
  ((e = e == cudaSuccess ? cudaFuncSetAttribute(kernels, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) : e), ...);
  if (e == cudaSuccess) cur = bytes;
  return e;
}

#define YB_CHECK_CUDA(expr)                                                                      \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) return yb::fail(YB200_ERR_CUDA, "%s: %s", #expr, cudaGetErrorString(_e)); \
  } while (0)
#define YB_REQUIRE(cond, code, ...) \
  do {                              \
    if (!(cond)) return yb::fail(code, __VA_ARGS__); \
  } while (0)

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// Argument checks of an activation view: non-null, positive extents, and c, c_pitch, c_off multiples of `mult` with c_off + c <= c_pitch.
// Returns 0 or YB200_ERR_INVALID with a message that starts with `name` (entry point and argument).
int check_act(const yb200_act* a, const char* name, int mult = 8);
inline bool same_shape(const yb200_act* a, const yb200_act* b) { return a->n == b->n && a->h == b->h && a->w == b->w && a->c == b->c; }
inline bool same_geometry(const yb200_act* a, const yb200_act* b) { return same_shape(a, b) && a->c_pitch == b->c_pitch; }

// 5-D TMA view (c, w, p, h, n) of an NHWC bf16 activation.  space_to_depth=false: p is a dummy dimension of
// extent 1.  space_to_depth=true (stride-2 taps): rows split into (h/2, p=row parity) and the column parity is
// folded into the channel coordinate (c' = col_parity*c_pitch + c).
int make_act_map(CUtensorMap* m, const yb200_act& a, bool space_to_depth, int box_c, int tw, int th, int tn);
// 2-D K-major bf16 matrix [rows][cols], box [box_rows][box_cols]
int make_mat_map(CUtensorMap* m, const void* ptr, long long rows, long long cols, int box_rows, int box_cols);
// 4-D (c, x, y, n) view of 16-bit values: element (c, x, y, n) at base + c + x * sx + y * sy + n * sn (strides in elements), extents
// (c, w, h, n); box (box_c, bw, bh, bn) in the swizzle of its 2 * box_c-byte rows.  Rejects a base that is not 16-byte aligned and strides
// that are not multiples of 8 elements (TMA requirements).
int make_pix_map(CUtensorMap* m, const void* base, int c, int w, int h, int n, long long sx, long long sy, long long sn, int box_c, int bw, int bh,
                 int bn);

// pick (tw, th, tn) with tw*th*tn == npix (power of two) minimising padded pixels for an (n,h,w) grid
void choose_tile(int n, int h, int w, int npix, int* log_tw, int* log_th);

// Programmatic dependent launch: every kernel of the YOLOX path starts with pdl_sync() (griddepcontrol.wait, then launch_dependents) and is
// launched through launch_k with the programmatic-stream-serialization attribute.  The next kernel of the stream (or of the captured graph) is
// then scheduled while this one drains: its CTAs take the SM slots that free up and park at their own griddepcontrol.wait until this grid has
// completed and flushed -- launch latency and block scheduling of ~540 launches per step leave the critical path.  The weight-gradient kernels
// (side stream) launch plainly through launch_k_opt(false, ...): a parked CTA of theirs holds up to 160 KB of shared memory that the main
// stream's kernels then cannot use.
template <typename... K, typename... A>
inline cudaError_t launch_k_opt(bool pdl, void (*kernel)(K...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<A>(args)...);
}
template <typename... K, typename... A>
inline cudaError_t launch_k(void (*kernel)(K...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
  return launch_k_opt(true, kernel, grid, block, smem, st, std::forward<A>(args)...);
}

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
inline int ilog2(int v) { int l = 0; while ((1 << l) < v) ++l; return l; }

}  // namespace yb
