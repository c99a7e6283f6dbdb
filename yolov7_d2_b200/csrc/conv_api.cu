// C-ABI entry points for the convolution family (forward, data gradient, weight gradient, weight packing).
#include "conv_gemm.cuh"
#include "host_common.cuh"
#include "wgrad_gemm.cuh"

#include <algorithm>
#include <cstring>

namespace yb {

// ------------------------------------------------------------------------------------------------
// kernel dispatch
// ------------------------------------------------------------------------------------------------
// Tensor maps of the TMA-store epilogue (ConvOutMaps) from the output geometry of `p`: the (n, y, x) -> offset mapping of the output and of
// the addend, over the work items' pixel grid with its valid extents, and the output's own channels; the box is the 64-row half tile of one
// consumer warpgroup.  A four-phase data gradient gets one map per output-parity phase, the phase's offset in its base.
static int make_out_maps(ConvOutMaps* om, const ConvGemmParams& p, int bn) {
  YB_REQUIRE(p.out_sc == 1, YB200_ERR_INVALID, "conv: a 16-bit output needs channel stride 1");
  int hx, hy, hn;
  conv_half_offset(p.log_tw, p.log_th, hx, hy, hn);
  const int tw = 1 << p.log_tw, th = 1 << p.log_th, tn = 128 >> (p.log_tw + p.log_th);
  const int bw = hx ? tw / 2 : tw, bh = hy ? th / 2 : th, bnn = hn ? tn / 2 : tn;
  const int box_c = bn < 64 ? bn : 64;
  for (int ph = 0; ph < (p.num_phases == 4 ? 4 : 1); ++ph) {
    const int oph = ph >> 1, opw = ph & 1;
    const char* out = static_cast<const char*>(p.out) + 2 * (oph * p.out_sh + opw * p.out_sw);
    int rc = make_pix_map(&om->out[ph], out, p.cout, p.w_valid, p.h_valid, p.n_valid, p.out_mw * p.out_sw, p.out_mh * p.out_sh, p.out_sn, box_c,
                          bw, bh, bnn);
    if (rc) return rc;
    if (p.addend == nullptr) continue;
    const char* add = reinterpret_cast<const char*>(p.addend) + 2 * (oph * p.add_sh + opw * p.add_sw);
    rc = make_pix_map(&om->add[ph], add, p.cout, p.w_valid, p.h_valid, p.n_valid, p.out_mw * p.add_sw, p.out_mh * p.add_sh, p.add_sn, box_c, bw,
                      bh, bnn);
    if (rc) return rc;
  }
  return 0;
}

template <int BN, int BK>
static int launch_conv_inst(const CUtensorMap& tmA, const CUtensorMap& tmB, const ConvGemmParams& p, dim3 grid, cudaStream_t st) {
  using Cfg = ConvGemmCfg<BN, BK>;
  const bool ext = p.epi_mode >= EPI_BF16_AFFINE;  // ConvNeXt / transformer epilogues live in their own instantiations
  // the 16-bit YOLOX modes store through tensor maps (the TMA-store epilogue of conv_gemm_persistent_kernel)
  ConvOutMaps om;
  memset(&om, 0, sizeof(om));
  if (!ext && p.epi_mode != EPI_F32_BIAS) {
    const int rc = make_out_maps(&om, p, BN);
    if (rc) return rc;
  }
  // persistent kernel: one or two CTAs per SM as its launch bounds (conv_min_ctas); the ring is as deep as the CTA's share of shared
  // memory allows after the epilogue staging tiles
  const int phases = p.num_phases == 4 ? 4 : 1;
  const int m_tiles = grid.x * phases, n_tiles = grid.y;  // work items of one column tile (pixel tiles x output-parity phases)
  const int occ = conv_min_ctas(BN, BK);
  // fp32 rows with channel stride 1 and an odd pitch ([B, A, 85]): chunks go through a per-warp transpose scratch behind the ring
  const bool xpose = p.epi_mode == EPI_F32_BIAS && p.out_sc == 1;
  const int fixed = ConvEpiCfg<BN>::kStageBytes + (xpose ? kXposeBytes : 0);
  const int budget = (occ == 1 ? 212 : 104) * 1024 - 1024 - fixed;
  int slots_kb = budget / Cfg::kStageBytes;  // k-blocks that fit in the ring
  // narrow layers (BLOCK_K 16 / 32) would spend their time on mbarrier round trips: put several k-blocks (up to 144
  // channels-taps) behind one barrier, keeping at least two ring slots
  const int num_kb = phases == 4 ? p.cin_blocks : p.num_taps * p.cin_blocks;  // phases: 1 / 2 / 2 / 4 (or 1 each) taps -- slots must divide all
  int kbs = 1;
  if (BK <= 32)
    for (int t = 1; t <= num_kb; ++t)
      if (num_kb % t == 0 && t * BK <= 144 && 2 * t <= slots_kb) kbs = t;
  int pst = slots_kb / kbs;
  if (pst > kMaxStagesP) pst = kMaxStagesP;
  if (pst < 2) pst = 2;
  const int smem = pst * kbs * Cfg::kStageBytes + 1024 + fixed;
  static PerDevice<int> smem_limit(0);
  YB_CHECK_CUDA(raise_smem_limit(smem_limit, smem, conv_gemm_persistent_kernel<BN, BK, false>, conv_gemm_persistent_kernel<BN, BK, true>));
  int groups = (occ * sm_count()) / n_tiles;
  if (groups < 1) groups = 1;
  if (groups > m_tiles) groups = m_tiles;
  if (phases == 4 && groups > 1 && groups % 2 == 0) --groups;  // odd stride through the work items: every CTA cycles through all four phases (1 / 2 / 2 / 4 taps)
  ConvGemmParams pp = p;
  pp.xpose = xpose ? 1 : 0;
  if (ext)
    launch_k(conv_gemm_persistent_kernel<BN, BK, true>, groups * n_tiles, kConvThreadsP, smem, st, tmA, tmB, pp, om, pst, kbs, n_tiles, m_tiles);
  else
    launch_k(conv_gemm_persistent_kernel<BN, BK, false>, groups * n_tiles, kConvThreadsP, smem, st, tmA, tmB, pp, om, pst, kbs, n_tiles, m_tiles);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

static int launch_conv(int bn, int bk, const CUtensorMap& tmA, const CUtensorMap& tmB, const ConvGemmParams& p, dim3 grid, cudaStream_t st) {
#define YB_CASE(BN, BK) \
  if (bn == BN && bk == BK) return launch_conv_inst<BN, BK>(tmA, tmB, p, grid, st);
  YB_CASE(16, 16) YB_CASE(16, 32) YB_CASE(16, 64)
  YB_CASE(32, 16) YB_CASE(32, 32) YB_CASE(32, 64)
  YB_CASE(64, 16) YB_CASE(64, 32) YB_CASE(64, 64)
  YB_CASE(128, 16) YB_CASE(128, 32) YB_CASE(128, 64)
#undef YB_CASE
  return fail(YB200_ERR_UNSUPPORTED, "no conv_gemm instantiation for BLOCK_N=%d BLOCK_K=%d", bn, bk);
}

static int pick_block_k(int c) { return c % 64 == 0 ? 64 : (c % 32 == 0 ? 32 : (c % 16 == 0 ? 16 : 0)); }
// column tiles up to 128: a 64 x 256 fp32 accumulator per consumer warpgroup (128 registers per thread) leaves too few registers for
// the epilogue and spills
static int pick_block_n(int c) { return c > 64 ? 128 : (c > 32 ? 64 : (c > 16 ? 32 : 16)); }

// check_act with the message prefix "<entry point> <argument>"
static int check_arg(const yb200_act* a, const char* who, const char* arg) {
  char name[96];
  snprintf(name, sizeof(name), "%s %s", who, arg);
  return check_act(a, name);
}

// fill the forward-style tap table (reads input pixel  stride*o + k - pad)
static int fill_fwd_taps(ConvTap* taps, const yb200_act& x, int ksize, int stride, int k_per_tap) {
  int nt = 0;
  if (ksize == 1) {
    taps[nt++] = ConvTap{x.c_off, 0, 0, 0, 0};
  } else if (ksize == 2) {  // 2x2 stride 2, no padding: input pixel (2*o + kh, 2*o + kw) = (row parity kh, column parity kw) of cell o
    for (int kh = 0; kh < 2; ++kh)
      for (int kw = 0; kw < 2; ++kw) taps[nt++] = ConvTap{kw * x.c_pitch + x.c_off, 0, kh, 0, (kh * 2 + kw) * k_per_tap};
  } else {
    for (int kh = 0; kh < 3; ++kh)
      for (int kw = 0; kw < 3; ++kw) {
        ConvTap t{};
        if (stride == 1) {
          t.c0 = x.c_off; t.dw = kw - 1; t.p = 0; t.dh = kh - 1;
        } else {  // input row 2*o + kh - 1: kh=0 -> (parity 1, o-1), kh=1 -> (0, o), kh=2 -> (1, o)
          t.p = (kh == 1) ? 0 : 1; t.dh = (kh == 0) ? -1 : 0;
          const int pw = (kw == 1) ? 0 : 1;
          t.dw = (kw == 0) ? -1 : 0;
          t.c0 = pw * x.c_pitch + x.c_off;
        }
        t.kb = (kh * 3 + kw) * k_per_tap;
        taps[nt++] = t;
      }
  }
  return nt;
}

// Output geometries: each returns a zeroed parameter block with the output set.
// 16-bit NHWC view
static ConvGemmParams out_view(const yb200_act& o) {
  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  p.out = static_cast<__nv_bfloat16*>(o.ptr) + o.c_off;
  p.out_sw = o.c_pitch;
  p.out_sh = 1LL * o.c_pitch * o.w;
  p.out_sn = 1LL * o.c_pitch * o.w * o.h;
  p.out_sc = 1;
  p.out_mh = 1; p.out_mw = 1;
  return p;
}
// fp32 [B, A, C] rows: pixel (y, x) of a w-wide grid is row a_off + y * w + x, its channels start at column c_off
static ConvGemmParams out_rows_f32(float* out, int w, int a_total, int a_off, int c_total, int c_off) {
  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  p.out = out + 1LL * a_off * c_total + c_off;
  p.out_sn = 1LL * a_total * c_total;
  p.out_sh = 1LL * w * c_total;
  p.out_sw = c_total;
  p.out_sc = 1;
  p.out_mh = 1; p.out_mw = 1;
  return p;
}
// fp32 NCHW [n][cout][h][w], h * w < 2^31
static ConvGemmParams out_nchw_f32(float* out, int cout, int h, int w) {
  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  const long long hw = 1LL * h * w;
  p.out = out;                 // element (n, y, x, c) at n*cout*hw + c*hw + y*w + x: lanes (pixels) write consecutive floats per channel
  p.out_sn = 1LL * cout * hw;
  p.out_sh = w;
  p.out_sw = 1;
  p.out_sc = static_cast<int>(hw);
  p.out_mh = 1; p.out_mw = 1;
  return p;
}
// fp32 NHWC [n][h][w][pitch]
static ConvGemmParams out_nhwc_f32(float* out, int pitch, int h, int w) {
  ConvGemmParams p;
  memset(&p, 0, sizeof(p));
  p.out = out;
  p.out_sw = pitch;
  p.out_sh = 1LL * pitch * w;
  p.out_sn = 1LL * pitch * w * h;
  p.out_sc = 1;
  p.out_mh = 1; p.out_mw = 1;
  return p;
}

// residual added in the epilogue, a 16-bit NHWC view of the output's shape
static void set_addend(ConvGemmParams& p, const yb200_act* a) {
  p.addend = static_cast<const __nv_bfloat16*>(a->ptr) + a->c_off;
  p.add_sw = a->c_pitch;
  p.add_sh = 1LL * a->c_pitch * a->w;
  p.add_sn = 1LL * a->c_pitch * a->w * a->h;
}

static void set_tiles(ConvGemmParams& p, int n, int h, int w) {
  choose_tile(n, h, w, 128, &p.log_tw, &p.log_th);
  const int tw = 1 << p.log_tw, th = 1 << p.log_th, tn = 128 >> (p.log_tw + p.log_th);
  p.tiles_w = ceil_div(w, tw); p.tiles_h = ceil_div(h, th); p.tiles_n = ceil_div(n, tn);
  p.n_valid = n; p.h_valid = h; p.w_valid = w;
}

}  // namespace yb

using namespace yb;

// ------------------------------------------------------------------------------------------------
// weights
// ------------------------------------------------------------------------------------------------
__global__ void pack_conv_weight_kernel(const float* __restrict__ w, const float* __restrict__ cout_scale, int cout, int cin, int taps, int cout_pad,
                                        int cin_pad, __nv_bfloat16* __restrict__ wf, __nv_bfloat16* __restrict__ wd) {
  pdl_sync();
  const long long total = 1LL * cout_pad * taps * cin_pad;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ci = static_cast<int>(i % cin_pad);
    const int t = static_cast<int>((i / cin_pad) % taps);
    const int co = static_cast<int>(i / (1LL * cin_pad * taps));
    float v = (co < cout && ci < cin) ? w[(1LL * co * cin + ci) * taps + t] : 0.f;
    if (cout_scale != nullptr && co < cout) v *= cout_scale[co];
    const __nv_bfloat16 b = __float2bfloat16_rn(v);
    if (wf) wf[i] = b;
    if (wd) wd[(1LL * ci * taps + t) * cout_pad + co] = b;
  }
}

static int pack_weight_impl(const float* w_oihw, const float* cout_scale, int cout, int cin, int ksize, int cout_pad, int cin_pad, void* w_fwd,
                            void* w_dgrad, void* stream) {
  YB_REQUIRE(w_oihw && (w_fwd || w_dgrad), YB200_ERR_INVALID, "pack_conv_weight: null pointer");
  YB_REQUIRE(cout > 0 && cin > 0 && (ksize >= 1 && ksize <= 3) && cout_pad >= cout && cin_pad >= cin, YB200_ERR_INVALID,
             "pack_conv_weight: bad sizes cout=%d cin=%d k=%d pads=%d,%d", cout, cin, ksize, cout_pad, cin_pad);
  const long long total = 1LL * cout_pad * ksize * ksize * cin_pad;
  const int blocks = static_cast<int>(std::min<long long>((total + 255) / 256, 4096));
  launch_k(pack_conv_weight_kernel, blocks, 256, 0, as_stream(stream), w_oihw, cout_scale, cout, cin, ksize * ksize, cout_pad, cin_pad,
                                                                 static_cast<__nv_bfloat16*>(w_fwd),
                                                                 static_cast<__nv_bfloat16*>(w_dgrad));
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// every convolution of a plan in ONE launch: the per-layer kernels are a few microseconds of work each, so ~70 launches per step are pure
// launch latency at the head of the step.  `table` (device memory, built once per plan) lists the layers; `prefix[i]` = padded elements of
// layers 0..i-1 (prefix[n] = total), so a thread finds its layer by binary search.
constexpr int kPackMaxLayers = 256;
__global__ void __launch_bounds__(256)
pack_conv_weights_batched_kernel(const yb200_pack_desc* __restrict__ table, const long long* __restrict__ prefix, int n) {
  pdl_sync();
  // Work unit = one ROW of a packed operand, one warp per row: forward rows (co, tap) run over ci, data-gradient rows (ci, tap) over co, so both
  // outputs are written with consecutive 2-byte stores; the fp32 source is gathered (9 M parameters: L2 resident).  Row r of the launch belongs
  // to layer l with rows_before[l] <= r: the row prefix is rebuilt per block in shared memory (n <= 256 layers), one binary search per row.
  __shared__ int s_rows[kPackMaxLayers + 1];
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int l = 0; l < n; ++l) {
      s_rows[l] = acc;
      const yb200_pack_desc d = table[l];
      const int taps = d.ksize * d.ksize;
      acc += (d.w_fwd ? d.cout_pad * taps : 0) + (d.w_dgrad ? d.cin_pad * taps : 0);
    }
    s_rows[n] = acc;
  }
  __syncthreads();
  const int total_rows = s_rows[n];
  const int lane = threadIdx.x & 31;
  const int warps = (gridDim.x * blockDim.x) >> 5;
  for (int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < total_rows; r += warps) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (s_rows[mid] <= r) lo = mid; else hi = mid - 1;
    }
    const yb200_pack_desc d = table[lo];
    const int taps = d.ksize * d.ksize;
    int q = r - s_rows[lo];
    const int fwd_rows = d.w_fwd ? d.cout_pad * taps : 0;
    if (q < fwd_rows) {  // forward operand [cout_pad][taps][cin_pad]
      const int co = q / taps, t = q - co * taps;
      __nv_bfloat16* dst = static_cast<__nv_bfloat16*>(d.w_fwd) + static_cast<size_t>(q) * d.cin_pad;
      const float* src = d.w_oihw + static_cast<size_t>(co) * d.cin * taps + t;
      for (int ci = lane; ci < d.cin_pad; ci += 32)
        dst[ci] = __float2bfloat16_rn((co < d.cout && ci < d.cin) ? src[static_cast<size_t>(ci) * taps] : 0.f);
    } else {             // data-gradient operand [cin_pad][taps][cout_pad]
      q -= fwd_rows;
      const int ci = q / taps, t = q - ci * taps;
      __nv_bfloat16* dst = static_cast<__nv_bfloat16*>(d.w_dgrad) + static_cast<size_t>(q) * d.cout_pad;
      const float* src = d.w_oihw + static_cast<size_t>(ci) * taps + t;
      for (int co = lane; co < d.cout_pad; co += 32)
        dst[co] = __float2bfloat16_rn((co < d.cout && ci < d.cin) ? src[static_cast<size_t>(co) * d.cin * taps] : 0.f);
    }
  }
}

extern "C" int yb200_pack_conv_weights_batched(const yb200_pack_desc* table_dev, const int64_t* prefix_dev, int n, int64_t total, void* stream) {
  YB_REQUIRE(table_dev && prefix_dev && n > 0 && n <= kPackMaxLayers && total > 0, YB200_ERR_INVALID, "pack_conv_weights_batched: bad arguments (n=%d)", n);
  const int blocks = static_cast<int>(std::min<long long>((2 * total + 255) / 256, 16LL * sm_count()));
  launch_k(pack_conv_weights_batched_kernel, blocks, 256, 0, as_stream(stream), table_dev, reinterpret_cast<const long long*>(prefix_dev), n);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_pack_conv_weight(const float* w_oihw, int cout, int cin, int ksize, int cout_pad, int cin_pad, void* w_fwd,
                                      void* w_dgrad, void* stream) {
  return pack_weight_impl(w_oihw, nullptr, cout, cin, ksize, cout_pad, cin_pad, w_fwd, w_dgrad, stream);
}

__global__ void scale_bias_kernel(const float* __restrict__ scale, const float* __restrict__ bias, int n, float* __restrict__ out) {
  pdl_sync();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = scale[i] * bias[i];
}

extern "C" int yb200_pack_conv_weight_scaled(const float* w_oihw, const float* cout_scale, const float* bias, int cout, int cin, int ksize,
                                             int cout_pad, int cin_pad, void* w_fwd, void* w_dgrad, float* scaled_bias, void* stream) {
  YB_REQUIRE(cout_scale != nullptr, YB200_ERR_INVALID, "pack_conv_weight_scaled: null scale");
  YB_REQUIRE((bias == nullptr) == (scaled_bias == nullptr), YB200_ERR_INVALID, "pack_conv_weight_scaled: pass both bias and scaled_bias or neither");
  if (bias) launch_k(scale_bias_kernel, ceil_div(cout, 256), 256, 0, as_stream(stream), cout_scale, bias, cout, scaled_bias);
  return pack_weight_impl(w_oihw, cout_scale, cout, cin, ksize, cout_pad, cin_pad, w_fwd, w_dgrad, stream);
}

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
// lo_delta > 0 selects the STRICT (operand-split) form: activations and weights are sums of `planes` bf16 values (x = x0 + x1 [+ x2], 8 more
// significant bits per plane: 16 bits with two planes, the full 24 of fp32 with three); plane j of an activation lives j * lo_delta channels
// after plane 0 in the same NHWC buffer and the weight matrix is [rows][plane 0 taps | plane 1 taps | plane 2 taps].  The product keeps every
// term x_i * w_j with i + j < planes (the dropped ones are below 2^-8planes relative) as extra taps of the SAME implicit GEMM -- one fp32
// accumulator, no extra kernel: 3 taps per spatial tap for two planes, 6 for three.
static void expand_split_taps(ConvGemmParams& p, int c, int lo_delta, int planes) {
  const int nt = p.num_taps;
  const int plane_kb = nt * c;
  int terms[6][2], nterm = 0;  // (activation plane, weight plane), largest products first
  for (int sum = 0; sum < planes; ++sum)
    for (int i = 0; i <= sum; ++i) { terms[nterm][0] = i; terms[nterm][1] = sum - i; ++nterm; }
  for (int t = nt - 1; t >= 0; --t) {
    const ConvTap b = p.taps[t];
    for (int q = 0; q < nterm; ++q) {
      ConvTap e = b;
      e.c0 = b.c0 + terms[q][0] * lo_delta;
      e.kb = b.kb + terms[q][1] * plane_kb;
      p.taps[nterm * t + q] = e;
    }
  }
  p.num_taps = nterm * nt;
}

// The launch shared by the forward entry points (`who` names the entry point in messages).  The weight matrix has `w_rows` rows: cout, or
// n * cout with one matrix per image (p.b_img_rows).
static int conv_fwd_common(const char* who, const yb200_act* x, const void* w_fwd, long long w_rows, int cout, int ksize, int stride,
                           ConvGemmParams& p, cudaStream_t st, int lo_delta = 0, int planes = 1, int group = 0) {
  YB_REQUIRE(w_fwd != nullptr, YB200_ERR_INVALID, "%s: null weights", who);
  YB_REQUIRE((ksize == 1 && stride == 1) || (ksize == 2 && stride == 2) || (ksize == 3 && (stride == 1 || stride == 2)), YB200_ERR_UNSUPPORTED,
             "%s: ksize=%d stride=%d not implemented", who, ksize, stride);
  const int bk = pick_block_k(x->c);
  YB_REQUIRE(bk != 0, YB200_ERR_UNSUPPORTED, "%s: input channels %d must be a multiple of 16", who, x->c);
  const int bn = pick_block_n(cout);
  const int oh = x->h / stride, ow = x->w / stride;
  set_tiles(p, x->n, oh, ow);
  p.num_taps = fill_fwd_taps(p.taps, *x, ksize, stride, x->c);
  long long kcols = 1LL * p.num_taps * x->c;
  if (lo_delta > 0) {
    YB_REQUIRE(planes == 2 || planes == 3, YB200_ERR_INVALID, "%s: %d planes", who, planes);
    YB_REQUIRE(lo_delta % 8 == 0 && x->c_off + (planes - 1) * lo_delta + x->c <= x->c_pitch, YB200_ERR_INVALID,
               "%s: plane %d [%d, %d) outside the channel pitch %d", who, planes - 1, x->c_off + (planes - 1) * lo_delta,
               x->c_off + (planes - 1) * lo_delta + x->c, x->c_pitch);
    expand_split_taps(p, x->c, lo_delta, planes);
    kcols *= planes;
  }
  p.cin_blocks = x->c / bk;
  p.cout = cout;
  if (group > 1 && ksize == 3 && stride == 1 && lo_delta == 0 && p.cin_blocks == 1 && x->c_off == 0 && x->c == x->c_pitch && (x->c / group) % 16 == 0) {
    // pixel-grouped 3x3 convolution (yb200_conv2d_fwd_fold): of the left neighbour GROUP only its last pixel reaches this group's outputs, of the
    // right neighbour only its first.  The side taps therefore load / multiply `cpp` channels instead of group * cpp: their activation box starts
    // at the needed pixel (the rest of the box lies beyond the channel extent: TMA zero fill, no L2 traffic) and the weight box at the matching
    // columns.  The products beyond the first cpp channels are zero either way (zero-filled activations on the left, zero weights of the
    // expanded matrix on the right).
    const int cpp = x->c / group;
    for (int t = 0; t < p.num_taps; ++t) {
      ConvTap& tp = p.taps[t];
      if (tp.dw == -1) { tp.c0 += (group - 1) * cpp; tp.kb += (group - 1) * cpp; }
    }
  }
  const int tw = 1 << p.log_tw, th = 1 << p.log_th, tn = 128 >> (p.log_tw + p.log_th);
  CUtensorMap tmA, tmB;
  int rc = make_act_map(&tmA, *x, stride == 2, bk, tw, th, tn);
  if (rc) return rc;
  rc = make_mat_map(&tmB, w_fwd, w_rows, kcols, bn, bk);
  if (rc) return rc;
  dim3 grid(p.tiles_w * p.tiles_h * p.tiles_n, ceil_div(cout, bn));
  return launch_conv(bn, bk, tmA, tmB, p, grid, st);
}

// checks shared by the forward entry points with a 16-bit NHWC output: the views, the stride, output grid = input grid / stride, and an
// optional residual of the output's shape
static int check_fwd(const char* who, const yb200_act* x, const yb200_act* out, const char* out_name, const yb200_act* residual, int stride) {
  int rc;
  if ((rc = check_arg(x, who, "x"))) return rc;
  if ((rc = check_arg(out, who, out_name))) return rc;
  if (residual && (rc = check_arg(residual, who, "residual"))) return rc;
  YB_REQUIRE(stride == 1 || stride == 2, YB200_ERR_UNSUPPORTED, "%s: stride %d", who, stride);
  YB_REQUIRE(out->n == x->n && out->h * stride == x->h && out->w * stride == x->w, YB200_ERR_INVALID,
             "%s: output %dx%dx%d does not match input %dx%dx%d / stride %d", who, out->n, out->h, out->w, x->n, x->h, x->w, stride);
  YB_REQUIRE(!residual || same_shape(residual, out), YB200_ERR_INVALID, "%s: residual shape mismatch", who);
  return 0;
}

static int conv2d_fwd_impl(const char* who, const yb200_act* x, const void* w_fwd, const yb200_act* z, int ksize, int stride, double* stat_sum,
                           double* stat_sqsum, int stat_fold, void* stream) {
  int rc;
  if ((rc = check_fwd(who, x, z, "z", nullptr, stride))) return rc;
  YB_REQUIRE((stat_sum == nullptr) == (stat_sqsum == nullptr), YB200_ERR_INVALID, "%s: pass both or neither stat buffer", who);
  ConvGemmParams p = out_view(*z);
  p.epi_mode = stat_sum ? EPI_F16_STATS : EPI_F16;
  p.stat_sum = stat_sum;
  p.stat_sq = stat_sqsum;
  p.stat_fold = stat_fold;
  return conv_fwd_common(who, x, w_fwd, z->c, z->c, ksize, stride, p, as_stream(stream), 0, 1, stat_fold > 0 ? z->c / stat_fold : 0);
}

extern "C" int yb200_conv2d_fwd(const yb200_act* x, const void* w_fwd, const yb200_act* z, int ksize, int stride,
                                double* stat_sum, double* stat_sqsum, void* stream) {
  return conv2d_fwd_impl("conv2d_fwd", x, w_fwd, z, ksize, stride, stat_sum, stat_sqsum, 0, stream);
}

extern "C" int yb200_conv2d_fwd_fold(const yb200_act* x, const void* w_fwd, const yb200_act* z, int ksize, int stride, double* stat_sum,
                                     double* stat_sqsum, int stat_fold, void* stream) {
  YB_REQUIRE(stat_fold > 0 && z && z->c % stat_fold == 0, YB200_ERR_INVALID, "conv2d_fwd_fold: output channels must be a multiple of stat_fold");
  return conv2d_fwd_impl("conv2d_fwd_fold", x, w_fwd, z, ksize, stride, stat_sum, stat_sqsum, stat_fold, stream);
}

extern "C" int yb200_conv2d_bn_silu_fwd(const yb200_act* x, const void* w_fwd, const float* scale, const float* shift,
                                        const yb200_act* residual, const yb200_act* out, int ksize, int stride, void* stream) {
  YB_REQUIRE(scale && shift, YB200_ERR_INVALID, "conv2d_bn_silu_fwd: null scale / shift");
  int rc;
  if ((rc = check_fwd("conv2d_bn_silu_fwd", x, out, "out", residual, stride))) return rc;
  ConvGemmParams p = out_view(*out);
  p.epi_mode = EPI_BF16_BN_SILU;
  p.scale = scale;
  p.shift = shift;
  if (residual) set_addend(p, residual);
  return conv_fwd_common("conv2d_bn_silu_fwd", x, w_fwd, out->c, out->c, ksize, stride, p, as_stream(stream));
}

extern "C" int yb200_conv2d_affine_fwd(const yb200_act* x, const void* w_fwd, const float* scale, const float* shift,
                                       const yb200_act* residual, const yb200_act* out, int ksize, int stride, void* stream) {
  int rc;
  if ((rc = check_fwd("conv2d_affine_fwd", x, out, "out", residual, stride))) return rc;
  ConvGemmParams p = out_view(*out);
  p.epi_mode = EPI_BF16_AFFINE;
  p.scale = scale;
  p.shift = shift;
  if (residual) set_addend(p, residual);
  return conv_fwd_common("conv2d_affine_fwd", x, w_fwd, out->c, out->c, ksize, stride, p, as_stream(stream));
}

extern "C" int yb200_conv2d_relu_fwd(const yb200_act* x, const void* w_fwd, const float* bias, const yb200_act* out, int ksize, int stride,
                                     void* stream) {
  int rc;
  if ((rc = check_fwd("conv2d_relu_fwd", x, out, "out", nullptr, stride))) return rc;
  ConvGemmParams p = out_view(*out);
  p.epi_mode = EPI_BF16_BIAS_RELU;
  p.shift = bias;
  return conv_fwd_common("conv2d_relu_fwd", x, w_fwd, out->c, out->c, ksize, stride, p, as_stream(stream));
}

extern "C" int yb200_linear_relu_fwd(const yb200_act* x, const void* w_fwd, const float* bias, const yb200_act* h_out, void* stream) {
  return yb200_conv2d_relu_fwd(x, w_fwd, bias, h_out, 1, 1, stream);
}

extern "C" int yb200_linear_gelu_fwd(const yb200_act* x, const void* w_fwd, const float* bias, const yb200_act* u_out, const yb200_act* h_out,
                                     void* stream) {
  int rc;
  if ((rc = check_fwd("linear_gelu_fwd", x, h_out, "h", nullptr, 1))) return rc;
  if (u_out && (rc = check_act(u_out, "linear_gelu_fwd u"))) return rc;
  YB_REQUIRE(!u_out || same_geometry(u_out, h_out), YB200_ERR_INVALID, "linear_gelu_fwd: u and h must have the same shape and channel pitch");
  ConvGemmParams p = out_view(*h_out);
  p.epi_mode = EPI_BF16_BIAS_GELU;
  p.shift = bias;
  if (u_out) p.aux_out = static_cast<__nv_bfloat16*>(u_out->ptr) + u_out->c_off;
  return conv_fwd_common("linear_gelu_fwd", x, w_fwd, h_out->c, h_out->c, 1, 1, p, as_stream(stream));
}

// batched: one weight matrix PER IMAGE (w_fwd: [n][cout][cin] bf16, i.e. n * cout rows), torch.bmm(pred_kernel, mask_features) of a whole batch in
// one launch.  Pixel tiles must not span images: accepted when the tile choose_tile picks is 128 pixels of one image (width x height = 128).
static int conv1x1_nchw_impl(const char* who, const yb200_act* x, const void* w_fwd, const float* bias, int cout, float* out_nchw, bool batched,
                             void* stream) {
  int rc;
  if ((rc = check_arg(x, who, "x"))) return rc;
  YB_REQUIRE(out_nchw && cout > 0 && cout <= 128, YB200_ERR_INVALID, "%s: bad arguments (cout=%d)", who, cout);
  YB_REQUIRE(1LL * x->h * x->w < (1LL << 31), YB200_ERR_UNSUPPORTED, "%s: plane too large", who);
  ConvGemmParams p = out_nchw_f32(out_nchw, cout, x->h, x->w);
  p.bias = bias;  // may be null (staged as zeros)
  p.epi_mode = EPI_F32_BIAS;
  if (!batched) return conv_fwd_common(who, x, w_fwd, cout, cout, 1, 1, p, as_stream(stream));
  int log_tw, log_th;
  choose_tile(x->n, x->h, x->w, 128, &log_tw, &log_th);
  YB_REQUIRE(log_tw + log_th == 7, YB200_ERR_UNSUPPORTED, "%s: a 128-pixel tile would span images at %dx%d (use yb200_conv1x1_nchw_f32 per image)", who,
             x->h, x->w);
  p.b_img_rows = cout;
  return conv_fwd_common(who, x, w_fwd, 1LL * x->n * cout, cout, 1, 1, p, as_stream(stream));
}

extern "C" int yb200_conv1x1_nchw_f32(const yb200_act* x, const void* w_fwd, const float* bias, int cout, float* out_nchw, void* stream) {
  return conv1x1_nchw_impl("conv1x1_nchw_f32", x, w_fwd, bias, cout, out_nchw, false, stream);
}

extern "C" int yb200_conv1x1_nchw_f32_batched(const yb200_act* x, const void* w_fwd, int cout, float* out_nchw, void* stream) {
  return conv1x1_nchw_impl("conv1x1_nchw_f32_batched", x, w_fwd, nullptr, cout, out_nchw, true, stream);
}

// lo_delta = 0, planes = 1: the plain bf16 form; lo_delta > 0: the strict form (conv_fwd_common)
static int conv1x1_bias_f32_impl(const char* who, const yb200_act* x, int lo_delta, int planes, const void* w_fwd, const float* bias, int cout,
                                 float* out, int a_total, int a_off, int c_total, int c_off, void* stream) {
  int rc;
  if ((rc = check_arg(x, who, "x"))) return rc;
  YB_REQUIRE(bias && out && cout > 0 && cout <= 128, YB200_ERR_INVALID, "%s: bad arguments (cout=%d)", who, cout);
  YB_REQUIRE(a_off >= 0 && a_off + x->h * x->w <= a_total && c_off >= 0 && c_off + cout <= c_total, YB200_ERR_INVALID,
             "%s: slice [%d+%d, %d+%d] outside [%d, %d]", who, a_off, x->h * x->w, c_off, cout, a_total, c_total);
  ConvGemmParams p = out_rows_f32(out, x->w, a_total, a_off, c_total, c_off);
  p.bias = bias;
  p.epi_mode = EPI_F32_BIAS;
  return conv_fwd_common(who, x, w_fwd, cout, cout, 1, 1, p, as_stream(stream), lo_delta, planes);
}

extern "C" int yb200_conv1x1_bias_f32(const yb200_act* x, const void* w_fwd, const float* bias, int cout, float* out,
                                      int a_total, int a_off, int c_total, int c_off, void* stream) {
  return conv1x1_bias_f32_impl("conv1x1_bias_f32", x, 0, 1, w_fwd, bias, cout, out, a_total, a_off, c_total, c_off, stream);
}

// ------------------------------------------------------------------------------------------------
// strict (operand-split) forward: fp32 results from bf16 tensor-core products
// ------------------------------------------------------------------------------------------------
__global__ void pack_conv_weight_split_kernel(const float* __restrict__ w, int cout, int cin, int taps, int cout_pad, int cin_pad, int planes,
                                              __nv_bfloat16* __restrict__ out) {
  pdl_sync();
  const long long per_plane = 1LL * taps * cin_pad;
  const long long total = 1LL * cout_pad * per_plane;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ci = static_cast<int>(i % cin_pad);
    const int t = static_cast<int>((i / cin_pad) % taps);
    const int co = static_cast<int>(i / per_plane);
    float r = (co < cout && ci < cin) ? w[(1LL * co * cin + ci) * taps + t] : 0.f;
    __nv_bfloat16* row = out + planes * co * per_plane + 1LL * t * cin_pad + ci;
    for (int pl = 0; pl < planes; ++pl) {
      const __nv_bfloat16 h = __float2bfloat16_rn(r);
      row[pl * per_plane] = h;
      r -= __bfloat162float(h);  // exact: the residual of a bf16 rounding is representable in fp32
    }
  }
}

extern "C" int yb200_pack_conv_weight_split(const float* w_oihw, int cout, int cin, int ksize, int cout_pad, int cin_pad, int planes, void* w_split,
                                            void* stream) {
  YB_REQUIRE(w_oihw && w_split, YB200_ERR_INVALID, "pack_conv_weight_split: null pointer");
  YB_REQUIRE(cout > 0 && cin > 0 && (ksize >= 1 && ksize <= 3) && cout_pad >= cout && cin_pad >= cin && (planes == 2 || planes == 3), YB200_ERR_INVALID,
             "pack_conv_weight_split: bad sizes cout=%d cin=%d k=%d pads=%d,%d planes=%d", cout, cin, ksize, cout_pad, cin_pad, planes);
  const long long total = 1LL * cout_pad * ksize * ksize * cin_pad;
  const int blocks = static_cast<int>(std::min<long long>((total + 255) / 256, 4096));
  launch_k(pack_conv_weight_split_kernel, blocks, 256, 0, as_stream(stream), w_oihw, cout, cin, ksize * ksize, cout_pad, cin_pad, planes,
                                                                       static_cast<__nv_bfloat16*>(w_split));
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_conv2d_fwd_split(const yb200_act* x, int lo_delta, int planes, const void* w_split, int cout, int ksize, int stride, float* z,
                                      int z_pitch, int z_off, void* stream) {
  int rc;
  if ((rc = check_act(x, "conv2d_fwd_split x"))) return rc;
  YB_REQUIRE(z && cout > 0 && z_off >= 0 && z_off + cout <= z_pitch && lo_delta > 0, YB200_ERR_INVALID,
             "conv2d_fwd_split: bad output slice [%d, %d) of %d (lo_delta %d)", z_off, z_off + cout, z_pitch, lo_delta);
  YB_REQUIRE(stride == 1 || stride == 2, YB200_ERR_UNSUPPORTED, "conv2d_fwd_split: stride %d", stride);
  ConvGemmParams p = out_nhwc_f32(z + z_off, z_pitch, x->h / stride, x->w / stride);
  p.epi_mode = EPI_F32_BIAS;  // bias == null: staged as zeros
  return conv_fwd_common("conv2d_fwd_split", x, w_split, cout, cout, ksize, stride, p, as_stream(stream), lo_delta, planes);
}

extern "C" int yb200_conv1x1_bias_f32_split(const yb200_act* x, int lo_delta, int planes, const void* w_split, const float* bias, int cout, float* out,
                                            int a_total, int a_off, int c_total, int c_off, void* stream) {
  YB_REQUIRE(lo_delta > 0, YB200_ERR_INVALID, "conv1x1_bias_f32_split: lo_delta %d", lo_delta);
  return conv1x1_bias_f32_impl("conv1x1_bias_f32_split", x, lo_delta, planes, w_split, bias, cout, out, a_total, a_off, c_total, c_off, stream);
}

// ------------------------------------------------------------------------------------------------
// data gradient
// ------------------------------------------------------------------------------------------------
static int dgrad_impl(const yb200_act* dz, const void* w_dgrad, const yb200_act* dx, const yb200_act* addend, int ksize, int stride,
                      const yb200_act* gelu_u, double* colsum, void* stream, int act_mode = EPI_BF16_GELU_BWD) {
  int rc;
  if ((rc = check_act(dz, "conv2d_dgrad dz"))) return rc;
  if ((rc = check_act(dx, "conv2d_dgrad dx"))) return rc;
  if (addend && (rc = check_act(addend, "conv2d_dgrad addend"))) return rc;
  YB_REQUIRE(w_dgrad != nullptr, YB200_ERR_INVALID, "conv2d_dgrad: null weights");
  YB_REQUIRE((ksize == 1 && stride == 1) || (ksize == 2 && stride == 2) || (ksize == 3 && (stride == 1 || stride == 2)), YB200_ERR_UNSUPPORTED,
             "conv2d_dgrad: ksize=%d stride=%d not implemented", ksize, stride);
  YB_REQUIRE(dz->n == dx->n && dz->h * stride == dx->h && dz->w * stride == dx->w, YB200_ERR_INVALID,
             "conv2d_dgrad: dz %dx%dx%d vs dx %dx%dx%d stride %d", dz->n, dz->h, dz->w, dx->n, dx->h, dx->w, stride);
  YB_REQUIRE(!addend || (addend->n == dx->n && addend->h == dx->h && addend->w == dx->w && addend->c == dx->c), YB200_ERR_INVALID,
             "conv2d_dgrad: addend shape mismatch");
  const int bk = pick_block_k(dz->c);
  YB_REQUIRE(bk != 0, YB200_ERR_UNSUPPORTED, "conv2d_dgrad: dz channels %d must be a multiple of 16", dz->c);
  const int cin = dx->c;
  const int bn = pick_block_n(cin);
  const int taps_total = ksize * ksize;
  cudaStream_t st = as_stream(stream);

  ConvGemmParams p = out_view(*dx);
  p.epi_mode = EPI_BF16;
  if (gelu_u) {
    p.epi_mode = act_mode;
    p.aux_in = static_cast<const __nv_bfloat16*>(gelu_u->ptr) + gelu_u->c_off;
    p.stat_sum = colsum;
  }
  p.cout = cin;
  p.cin_blocks = dz->c / bk;
  if (addend) set_addend(p, addend);
  set_tiles(p, dz->n, dz->h, dz->w);  // pixel grid = dz grid (for stride 2: each work item is one output-parity class of a tile)
  const int tw = 1 << p.log_tw, th = 1 << p.log_th, tn = 128 >> (p.log_tw + p.log_th);
  CUtensorMap tmA, tmB;
  if ((rc = make_act_map(&tmA, *dz, false, bk, tw, th, tn))) return rc;
  if ((rc = make_mat_map(&tmB, w_dgrad, cin, 1LL * taps_total * dz->c, bn, bk))) return rc;
  dim3 grid(p.tiles_w * p.tiles_h * p.tiles_n, ceil_div(cin, bn));

  if (stride == 1) {
    int nt = 0;
    if (ksize == 1) {
      p.taps[nt++] = ConvTap{dz->c_off, 0, 0, 0, 0};
    } else {
      // dx[y,x] = sum_k dz[y + 1 - kh, x + 1 - kw] * W[kh,kw]
      for (int kh = 0; kh < 3; ++kh)
        for (int kw = 0; kw < 3; ++kw) p.taps[nt++] = ConvTap{dz->c_off, 1 - kw, 0, 1 - kh, (kh * 3 + kw) * dz->c};
    }
    p.num_taps = nt;
    return launch_conv(bn, bk, tmA, tmB, p, grid, st);
  }
  // stride 2: input pixel (2i+ph, 2j+pw) receives  kh with (ph + 1 - kh) even:  ph=0 -> kh=1 (row i);  ph=1 -> kh=0 (row i+1), kh=2 (row i)
  auto phase_taps = [&](int ph, int pw, ConvTap* out) {
    int nt = 0;
    if (ksize == 2) out[nt++] = ConvTap{dz->c_off, 0, 0, 0, (ph * 2 + pw) * dz->c};  // 2x2 s2: input pixel (2i+ph, 2j+pw) sees only tap (ph, pw)
    for (int kh = 0; kh < 3 && ksize == 3; ++kh) {
      if (((ph + 1 - kh) & 1) != 0) continue;
      const int dh = (ph + 1 - kh) / 2;
      for (int kw = 0; kw < 3; ++kw) {
        if (((pw + 1 - kw) & 1) != 0) continue;
        const int dw = (pw + 1 - kw) / 2;
        out[nt++] = ConvTap{dz->c_off, dw, 0, dh, (kh * 3 + kw) * dz->c};
      }
    }
    return nt;
  };
  p.out_mh = 2; p.out_mw = 2;
  // all four phases in ONE persistent launch: the phases of a pixel tile run back to back on neighbouring CTAs and share its dz tile in L2
  int nt = 0;
  for (int ph = 0; ph < 2; ++ph)
    for (int pw = 0; pw < 2; ++pw) {
      p.phase_tap[ph * 2 + pw] = nt;
      nt += phase_taps(ph, pw, p.taps + nt);
    }
  p.phase_tap[4] = nt;
  p.num_taps = nt;
  p.num_phases = 4;
  return launch_conv(bn, bk, tmA, tmB, p, grid, st);
}

extern "C" int yb200_conv2d_dgrad(const yb200_act* dz, const void* w_dgrad, const yb200_act* dx, const yb200_act* addend,
                                  int ksize, int stride, void* stream) {
  return dgrad_impl(dz, w_dgrad, dx, addend, ksize, stride, nullptr, nullptr, stream);
}

extern "C" int yb200_linear_dgrad_gelu(const yb200_act* dh_src, const void* w_dgrad, const yb200_act* u, const yb200_act* du, double* bias_grad_sum,
                                       void* stream) {
  int rc;
  if ((rc = check_act(u, "linear_dgrad_gelu u"))) return rc;
  if ((rc = check_act(du, "linear_dgrad_gelu du"))) return rc;
  YB_REQUIRE(same_geometry(u, du), YB200_ERR_INVALID, "linear_dgrad_gelu: u and du must have the same shape and channel pitch");
  return dgrad_impl(dh_src, w_dgrad, du, nullptr, 1, 1, u, bias_grad_sum, stream);
}

extern "C" int yb200_linear_dgrad_relu(const yb200_act* dz, const void* w_dgrad, const yb200_act* h, const yb200_act* du, double* bias_grad_sum,
                                       void* stream) {
  int rc;
  if ((rc = check_act(h, "linear_dgrad_relu h"))) return rc;
  if ((rc = check_act(du, "linear_dgrad_relu du"))) return rc;
  YB_REQUIRE(same_geometry(h, du), YB200_ERR_INVALID, "linear_dgrad_relu: h and du must have the same shape and channel pitch");
  return dgrad_impl(dz, w_dgrad, du, nullptr, 1, 1, h, bias_grad_sum, stream, EPI_BF16_RELU_BWD);
}

extern "C" int yb200_conv2d_dgrad_relu(const yb200_act* dz, const void* w_dgrad, const yb200_act* h, const yb200_act* dx, const yb200_act* addend,
                                       int ksize, int stride, void* stream) {
  int rc;
  if ((rc = check_arg(h, "conv2d_dgrad_relu", "h"))) return rc;
  if ((rc = check_arg(dx, "conv2d_dgrad_relu", "dx"))) return rc;
  YB_REQUIRE((ksize == 1 || ksize == 3) && stride == 1, YB200_ERR_UNSUPPORTED, "conv2d_dgrad_relu: ksize=%d stride=%d not implemented", ksize, stride);
  YB_REQUIRE(same_geometry(h, dx), YB200_ERR_INVALID, "conv2d_dgrad_relu: h and dx must have the same shape and channel pitch");
  return dgrad_impl(dz, w_dgrad, dx, addend, ksize, stride, h, nullptr, stream, EPI_BF16_RELU_BWD);
}

// ------------------------------------------------------------------------------------------------
// weight gradient
// ------------------------------------------------------------------------------------------------
namespace {
struct WgradPlan {
  WgradParams p;
  int splits;
  int smem;
  int tw, th, tn;
  long long workspace_bytes() const { return 4LL * splits * p.cout * p.num_taps * p.cin; }  // fp32 partial sums of every split
};

int plan_wgrad(const yb200_act* x, const yb200_act* dz, int ksize, int stride, WgradPlan* pl, int group = 0) {
  int rc;
  if ((rc = check_act(x, "conv2d_wgrad x"))) return rc;
  if ((rc = check_act(dz, "conv2d_wgrad dz"))) return rc;
  YB_REQUIRE((ksize == 1 && stride == 1) || (ksize == 2 && stride == 2) || (ksize == 3 && (stride == 1 || stride == 2)), YB200_ERR_UNSUPPORTED,
             "conv2d_wgrad: ksize=%d stride=%d not implemented", ksize, stride);
  YB_REQUIRE(dz->n == x->n && dz->h * stride == x->h && dz->w * stride == x->w, YB200_ERR_INVALID,
             "conv2d_wgrad: dz %dx%dx%d vs x %dx%dx%d stride %d", dz->n, dz->h, dz->w, x->n, x->h, x->w, stride);
  YB_REQUIRE(x->c % 16 == 0, YB200_ERR_UNSUPPORTED, "conv2d_wgrad: input channels %d must be a multiple of 16", x->c);
  YB_REQUIRE(dz->c % 16 == 0, YB200_ERR_UNSUPPORTED, "conv2d_wgrad: output channels %d must be a multiple of 16", dz->c);
  WgradParams& p = pl->p;
  memset(&p, 0, sizeof(p));
  p.cout = dz->c;
  p.cin = x->c;
  p.kc_a = dz->c >= 64 ? 64 : (dz->c >= 32 ? 32 : 16);
  YB_REQUIRE(dz->c % p.kc_a == 0 || dz->c == dz->c_pitch, YB200_ERR_UNSUPPORTED,
             "conv2d_wgrad: dz channel slice %d not a multiple of %d", dz->c, p.kc_a);
  // boxes of kc_a channels per 128-row tile; a box that overshoots the slice (48 -> 2 x 32, 80 -> 2 x 64, 96 -> 2 x 64) is legal only when
  // the slice ends at the channel pitch (required above): the overshoot is then out of bounds for TMA and zero filled
  p.ma = ceil_div(dz->c < 128 ? dz->c : 128, p.kc_a);
  p.cout_tiles = ceil_div(dz->c, 128);
  p.kc_b = x->c % 64 == 0 ? 64 : (x->c % 32 == 0 ? 32 : 16);
  p.bn = x->c % 128 == 0 ? 128 : (x->c % 64 == 0 ? 64 : p.kc_b);
  p.nb = p.bn / p.kc_b;
  p.cin_tiles = x->c / p.bn;
  p.num_taps = fill_fwd_taps(p.taps, *x, ksize, stride, 0);
  if (group > 1) {
    // pixel-grouped 3x3 convolution (the stem): the expanded weight matrix is non-zero for the left / right neighbour group only at its last /
    // first pixel, and only those entries are folded back onto the parameter.  The side taps therefore load and multiply cpp = C / group channels.
    const int cpp = x->c / group;
    YB_REQUIRE(ksize == 3 && stride == 1 && x->c % group == 0 && cpp % 16 == 0 && x->c_off == 0 && x->c == x->c_pitch && p.cin_tiles == 1 && p.nb == 1,
               YB200_ERR_UNSUPPORTED, "conv2d_wgrad_grouped: needs a 3x3 stride-1 convolution on a whole [.., %d x 16k]-channel grouped tensor of <= 64 channels (got c=%d pitch=%d group=%d)",
               group, x->c, x->c_pitch, group);
    for (int t = 0; t < p.num_taps; ++t) {
      ConvTap& tp = p.taps[t];
      tp.kb = 0;
      if (tp.dw == -1) { tp.c0 += (group - 1) * cpp; tp.kb = (group - 1) * cpp; tp.ks = cpp / 16; }
      if (tp.dw == 1) tp.ks = cpp / 16;
    }
  }
  // taps per CTA: the accumulators of all of them live in registers (TPC * BN / 2 per thread), so 128-wide cin tiles take one tap each
  p.tpc = (p.num_taps == 1 || p.bn == 128) ? 1 : 3;
  p.tap_groups = ceil_div(p.num_taps, p.tpc);
  p.dz_c0 = dz->c_off;
  choose_tile(dz->n, dz->h, dz->w, kWgPix, &p.log_tw, &p.log_th);
  pl->tw = 1 << p.log_tw; pl->th = 1 << p.log_th; pl->tn = kWgPix >> (p.log_tw + p.log_th);
  p.tiles_w = ceil_div(dz->w, pl->tw); p.tiles_h = ceil_div(dz->h, pl->th); p.tiles_n = ceil_div(dz->n, pl->tn);
  p.num_blocks = p.tiles_w * p.tiles_h * p.tiles_n;
  const int base = p.cout_tiles * p.cin_tiles * p.tap_groups;
  const int occ_regs = p.tpc * p.bn <= 96 ? 2 : 1;  // CTAs per SM the accumulator registers allow (wgrad_gemm_kernel launch bounds)
  const int stage = kWgPix * 2 * (p.kc_a * p.ma + p.kc_b * p.nb * p.tpc);
  p.stages = kWgStages;
  if (std::min(occ_regs, (220 * 1024) / (stage * kWgStages + 1024)) <= 1)  // one CTA per SM anyway: deepen the ring
    p.stages = std::max(kWgStages, std::min(kWgMaxStages, (220 * 1024 - 1024) / stage));
  pl->smem = stage * p.stages + 1024;
  // Split the pixel range so that ONE wave of CTAs covers the machine (every CTA pays pipeline fill and a full accumulator
  // write-back, so extra waves are pure overhead); occupancy is bounded by registers and shared memory.
  int occ = std::min(occ_regs, (220 * 1024) / pl->smem);
  if (occ < 1) occ = 1;
  int splits = (occ * sm_count()) / base;  // floor: a partial second wave would double the tail
  if (splits > p.num_blocks / 8) splits = p.num_blocks / 8;  // at least 8 pixel blocks per CTA
  const long long wbytes = 4LL * p.cout * p.num_taps * p.cin;
  const long long max_splits = (128LL << 20) / wbytes;
  if (splits > max_splits) splits = static_cast<int>(max_splits);
  if (splits < 1) splits = 1;
  p.blocks_per_split = ceil_div(p.num_blocks, splits);
  pl->splits = ceil_div(p.num_blocks, p.blocks_per_split);
  return 0;
}
}  // namespace

extern "C" int64_t yb200_conv2d_wgrad_workspace(const yb200_act* x, const yb200_act* dz, int ksize, int stride) {
  WgradPlan pl;
  int rc = plan_wgrad(x, dz, ksize, stride, &pl);
  if (rc) return rc;
  return pl.workspace_bytes();
}

template <int BN, int TPC>
static int launch_wgrad_inst(const CUtensorMap& tmDz, const CUtensorMap& tmX, const WgradPlan& pl, dim3 grid, cudaStream_t st) {
  static PerDevice<int> smem_limit(0);
  YB_CHECK_CUDA(raise_smem_limit(smem_limit, pl.smem, wgrad_gemm_kernel<BN, TPC>));
  launch_k_opt(false, wgrad_gemm_kernel<BN, TPC>, grid, kWgThreads, pl.smem, st, tmDz, tmX, pl.p);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

static int launch_wgrad(const CUtensorMap& tmDz, const CUtensorMap& tmX, const WgradPlan& pl, dim3 grid, cudaStream_t st) {
  const int bn = pl.p.bn, tpc = pl.p.tpc;
#define YB_CASE(BN, TPC) \
  if (bn == BN && tpc == TPC) return launch_wgrad_inst<BN, TPC>(tmDz, tmX, pl, grid, st);
  YB_CASE(16, 1) YB_CASE(16, 3)
  YB_CASE(32, 1) YB_CASE(32, 3)
  YB_CASE(64, 1) YB_CASE(64, 3)
  YB_CASE(128, 1)
#undef YB_CASE
  return fail(YB200_ERR_UNSUPPORTED, "conv2d_wgrad: no kernel for a %d-wide cin tile with %d taps per CTA", bn, tpc);
}

static int wgrad_impl(const yb200_act* x, const yb200_act* dz, int ksize, int stride, int cin_real, int group, float* grad_oihw, int accumulate,
                      void* workspace, int64_t workspace_bytes, void* stream) {
  WgradPlan pl;
  int rc = plan_wgrad(x, dz, ksize, stride, &pl, group);
  if (rc) return rc;
  YB_REQUIRE(grad_oihw && workspace, YB200_ERR_INVALID, "conv2d_wgrad: null pointer");
  YB_REQUIRE(cin_real > 0 && cin_real <= x->c, YB200_ERR_INVALID, "conv2d_wgrad: cin_real %d vs padded %d", cin_real, x->c);
  YB_REQUIRE(workspace_bytes >= pl.workspace_bytes(), YB200_ERR_INVALID, "conv2d_wgrad: workspace %lld < %lld bytes", (long long)workspace_bytes,
             pl.workspace_bytes());
  pl.p.ws = static_cast<float*>(workspace);
  cudaStream_t st = as_stream(stream);
  CUtensorMap tmDz, tmX;
  if ((rc = make_act_map(&tmDz, *dz, false, pl.p.kc_a, pl.tw, pl.th, pl.tn))) return rc;
  if ((rc = make_act_map(&tmX, *x, stride == 2, pl.p.kc_b, pl.tw, pl.th, pl.tn))) return rc;
  dim3 grid(pl.p.cout_tiles * pl.p.cin_tiles * pl.p.tap_groups, pl.splits);
  if ((rc = launch_wgrad(tmDz, tmX, pl, grid, st))) return rc;
  const long long total = 1LL * pl.p.cout * pl.p.num_taps * pl.p.cin;
  const int blocks = static_cast<int>(std::min<long long>((total + 31) / 32, 16 * sm_count()));
  launch_k_opt(false, wgrad_reduce_kernel, blocks, 256, 0, st, pl.p.ws, grad_oihw, pl.splits, pl.p.cout, pl.p.num_taps, pl.p.cin, cin_real, accumulate);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int yb200_conv2d_wgrad(const yb200_act* x, const yb200_act* dz, int ksize, int stride, int cin_real, float* grad_oihw,
                                  int accumulate, void* workspace, int64_t workspace_bytes, void* stream) {
  return wgrad_impl(x, dz, ksize, stride, cin_real, 0, grad_oihw, accumulate, workspace, workspace_bytes, stream);
}

extern "C" int yb200_conv2d_wgrad_grouped(const yb200_act* x, const yb200_act* dz, int ksize, int stride, int cin_real, int group, float* grad_oihw,
                                          int accumulate, void* workspace, int64_t workspace_bytes, void* stream) {
  YB_REQUIRE(group > 1, YB200_ERR_INVALID, "conv2d_wgrad_grouped: group %d (use yb200_conv2d_wgrad)", group);
  return wgrad_impl(x, dz, ksize, stride, cin_real, group, grad_oihw, accumulate, workspace, workspace_bytes, stream);
}
