// Implicit-GEMM convolution on wgmma (sm_90a).
//
//   D[128 pixels, BLOCK_N channels] = sum over (tap, cin-block)  A_tap[128 px, BLOCK_K] * B_tap[BLOCK_N, BLOCK_K]^T
//
// A is the NHWC bf16 activation tensor seen through a 5-D TMA map (c, w, p, h, n): a "tap" is a
// coordinate offset of the 128-pixel box (TW x TH x TN), so zero padding is TMA out-of-bounds fill and
// stride-2 convolutions are taps on the space-to-depth view (p = row parity, column parity folded into c).
// B is the packed weight matrix [rows][taps*K] (K-major).  Two consumer warpgroups hold the fp32 accumulators
// of one 128 x BLOCK_N output tile in registers (64 rows each), fed by a TMA->smem mbarrier ring.
//
// Used for: conv forward (F3/F2/F8 of SURVEY.md par.8a), data-gradient (same kernel, transposed tap table)
// and the 1x1 prediction convolutions (fp32 + bias epilogue).
#pragma once
#include <cuda_fp16.h>

#include "sm90.cuh"

namespace yb {

constexpr int kMaxTaps = 54;  // 9 spatial taps x up to 6 operand-split terms (strict mode, conv_api.cu)

enum EpiMode : int {
  EPI_BF16 = 0,       // out = bf16(acc [+ addend])                          (data gradients)
  EPI_F16 = 1,        // out = fp16(acc)                                     (pre-BatchNorm conv output, eval mode)
  EPI_F16_STATS = 2,  // out = fp16(acc) + per-channel sum / sum-of-squares of the stored values (fp64 atomics)
  EPI_F32_BIAS = 3,   // out = acc + bias[c]   (fp32, arbitrary element strides)
  EPI_BF16_BN_SILU = 4,  // out = bf16(SiLU(acc*scale[c] + shift[c]) [+ addend]): eval-mode BatchNorm folded into the conv
                         // (the fold of utils/checkpoint.py:11-43 applied as an epilogue), residual added after the activation
  EPI_BF16_AFFINE = 5,   // out = bf16(acc*scale[c] + shift[c] [+ addend]); scale / shift may be null (1 / 0): Linear / Conv bias,
                         // ConvNeXt layer scale + residual (convnext.py:54-59)
  EPI_BF16_BIAS_GELU = 6,  // u = bf16(acc + shift[c]) -> aux_out (optional), out = bf16(GELU(u)), exact erf form (convnext.py:52-53)
  EPI_BF16_GELU_BWD = 7,   // out = bf16(acc * GELU'(u)), u read from aux_in; optional per-channel sums of the stored values -> stat_sum
                           // (gradient of the Linear bias that produced u)
  EPI_BF16_BIAS_RELU = 8,  // out = bf16(max(acc + shift[c], 0)): Linear + ReLU of the transformer FFN (detr_backbone.py:167)
  EPI_BF16_RELU_BWD = 9,   // out = bf16(aux_in > 0 ? acc : 0) (aux_in = the ReLU output); optional column sums -> stat_sum
};

__device__ __forceinline__ bool epi_has_stats(int mode, const double* stat_sum) {
  return mode == EPI_F16_STATS || ((mode == EPI_BF16_GELU_BWD || mode == EPI_BF16_RELU_BWD) && stat_sum != nullptr);
}
// Phi(u) = 0.5 (1 + erf(u / sqrt 2)) through Abramowitz-Stegun 7.1.26 (|error| < 1.5e-7, far below the bf16 resolution of the stored
// result): one MUFU.RCP, one MUFU.EX2 and 7 FMAs instead of erff's branchy polynomial -- the GEMMs that carry these epilogues have
// K = C and N = 4C, so they are bound by epilogue instruction issue, not by the tensor pipe.  e = exp(-u^2 / 2) is shared with GELU'.
__device__ __forceinline__ float gelu_phi(float u, float& e) {
  const float z = fabsf(u) * 0.70710678118654752f;
  const float t = __fdividef(1.f, fmaf(0.3275911f, z, 1.f));
  const float poly = t * fmaf(t, fmaf(t, fmaf(t, fmaf(t, 1.061405429f, -1.453152027f), 1.421413741f), -0.284496736f), 0.254829592f);
  e = __expf(-z * z);
  const float q = 0.5f * poly * e;
  return u >= 0.f ? 1.f - q : q;
}
__device__ __forceinline__ float gelu_erf(float u) {
  float e;
  return u * gelu_phi(u, e);
}
__device__ __forceinline__ float gelu_erf_grad(float u) {
  float e;
  const float phi = gelu_phi(u, e);
  return fmaf(u * 0.3989422804014327f, e, phi);
}

struct ConvTap {
  int c0;  // coordinate offset in the innermost (channel) dimension of the A map
  int dw;  // offset in w
  int p;   // coordinate in the parity dimension
  int dh;  // offset in h
  int kb;  // column offset of this tap inside the B matrix
  int ks;  // > 0: only the first ks 16-wide K steps of each k-block of this tap carry non-zero operands (persistent kernel: the rest is skipped)
};

struct ConvGemmParams {
  int tiles_w, tiles_h, tiles_n;
  int log_tw, log_th;          // tile = (1<<log_tw) x (1<<log_th) x (128 >> (log_tw+log_th)) pixels
  int num_taps, cin_blocks;    // K loop = num_taps * cin_blocks blocks of BLOCK_K
  int n_valid, h_valid, w_valid;  // pixel-grid extents (tile-space); pixels outside are neither stored nor counted
  int cout;                    // valid output channels (columns >= cout are dropped)
  int epi_mode;
  // output element (n, y, x, c) lives at out[n*out_sn + (y*out_mh+ph)*out_sh + (x*out_mw+pw)*out_sw + c*out_sc]; (ph, pw) is the
  // output-parity phase of the work item when num_phases == 4, else (0, 0)
  long long out_sn, out_sh, out_sw;
  int out_sc, out_mh, out_mw;
  void* out;
  const __nv_bfloat16* addend;  // optional, bf16, same (n,y,x) -> offset mapping with its own strides, channel stride 1
  long long add_sn, add_sh, add_sw;
  const float* bias;
  const float* scale;  // EPI_BF16_BN_SILU: per-channel scale / shift (gamma/sqrt(var+eps), beta - mean*scale)
  const float* shift;
  double* stat_sum;
  double* stat_sq;
  int stat_fold;  // > 0: column c accumulates into statistic c % stat_fold (pixel-grouped views: several columns are the same channel)
  // num_phases == 4: ONE launch computes the four output-parity classes of a stride-2 data gradient.  Work item wi = 4 * tile + phase;
  // phase (ph, pw) = (wi >> 1 & 1, wi & 1) uses taps[phase_tap[phase] .. phase_tap[phase + 1]) and writes pixel (2y + ph, 2x + pw).  The four
  // phases of a tile run on neighbouring CTAs at about the same time, so the gradient tile they share comes from HBM once (four separate
  // launches read the whole tensor four times).
  int num_phases;
  int phase_tap[5];
  int b_img_rows; // > 0: per-image weights -- the tile of image n reads weight rows n * b_img_rows + column (tiles must not span images)
  int xpose;      // EPI_F32_BIAS with channel-contiguous rows: transpose each 32 x 32 chunk through shared memory (kXposeBytes behind the ring)
  const __nv_bfloat16* aux_in;  // EPI_BF16_GELU_BWD: pre-activation u, same geometry as `out`
  __nv_bfloat16* aux_out;       // EPI_BF16_BIAS_GELU: where u is stored (may be null), same geometry as `out`
  ConvTap taps[kMaxTaps];
};

__device__ __forceinline__ void conv_decode_work(const ConvGemmParams& p, int wi, int& m, int& tap0, int& ntaps, int& oph, int& opw) {
  if (p.num_phases == 4) {
    m = wi >> 2;
    const int ph = wi & 3;
    tap0 = p.phase_tap[ph];
    ntaps = p.phase_tap[ph + 1] - tap0;
    oph = ph >> 1;
    opw = ph & 1;
  } else {
    m = wi; tap0 = 0; ntaps = p.num_taps; oph = opw = 0;
  }
}

template <int BLOCK_N, int BLOCK_K>
struct ConvGemmCfg {
  static constexpr int kSwizzle = BLOCK_K * 2;  // bytes of one K-row: 32 / 64 / 128
  static constexpr int kABytes = 128 * BLOCK_K * 2;
  static constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static_assert(BLOCK_K == 16 || BLOCK_K == 32 || BLOCK_K == 64, "BLOCK_K");
  static_assert(BLOCK_N == 16 || BLOCK_N == 32 || BLOCK_N == 64 || BLOCK_N == 128, "BLOCK_N");
  static_assert(kABytes % (8 * kSwizzle) == 0 && kStageBytes % (8 * kSwizzle) == 0, "tiles must start on a swizzle-pattern boundary");
};

__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  __half2 v = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ void store_bf16x8(__nv_bfloat16* dst, const float* v) {
  uint4 u;
  u.x = pack_bf16x2(v[0], v[1]);
  u.y = pack_bf16x2(v[2], v[3]);
  u.z = pack_bf16x2(v[4], v[5]);
  u.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(dst) = u;
}

// Per-column parameters (scale | shift / bias) of the CTA's column tile are staged in shared memory once per CTA; the epilogue reads
// them with 16-byte broadcast loads (per-element __ldg plus a null test per element made the parameterised epilogues 2-3x slower
// than the plain one).  Columns beyond cout hold (1, 0).
template <int BLOCK_N>
__device__ __forceinline__ void stage_col_params(const ConvGemmParams& p, int col0, float (*s_col)[BLOCK_N]) {
  const float* sh = p.shift ? p.shift : p.bias;
  for (int i = threadIdx.x; i < BLOCK_N; i += blockDim.x) {
    const bool ok = col0 + i < p.cout;
    s_col[0][i] = (ok && p.scale) ? p.scale[col0 + i] : 1.f;
    s_col[1][i] = (ok && sh) ? sh[col0 + i] : 0.f;
  }
}

// EXT = false: the YOLOX training / inference modes only (EPI_BF16 .. EPI_BF16_BN_SILU); EXT = true adds the ConvNeXt / transformer
// modes.  Two instantiations per kernel keep the hot YOLOX kernels free of the extra modes' registers and code.
// fp32 rows with a pitch that is not a multiple of 16 bytes (the [B, A, 85] prediction tensor): a lane-per-pixel store touches 32 different
// sectors per instruction.  With the per-warp scratch each store instruction writes 32 consecutive floats of ONE pixel row instead.
constexpr int kXposeWarpFloats = 32 * 33 + 64;              // 32 x 32 chunk (pitch 33: conflict free both ways) + 32 row offsets (8 B each)
constexpr int kXposeBytes = 8 * kXposeWarpFloats * 4;       // eight epilogue warps

// One chunk (CH columns of one accumulator row per lane) of the staging-tile epilogue: EPI_F32_BIAS and, with EXT, the ConvNeXt /
// transformer modes (the 16-bit YOLOX modes store from the accumulator fragments: conv_gemm_persistent_kernel).
//   part_sum: this warp's shared-memory slots for the chunk's columns (column sums of EPI_BF16_GELU_BWD / EPI_BF16_RELU_BWD); `accumulate`
//   adds to them (sums over all tiles of the CTA) instead of overwriting.
template <int CH, bool EXT = true>
__device__ __forceinline__ void conv_epilogue_chunk(const ConvGemmParams& p, float (&v)[CH], bool valid, long long pix_off, long long add_off,
                                                    int cbase, int lane, float* part_sum, bool accumulate, const float* col_scale,
                                                    const float* col_shift, float* xp = nullptr) {
  if (p.epi_mode == EPI_F32_BIAS) {
    if (xp != nullptr) {
      long long* s_off = reinterpret_cast<long long*>(xp + 32 * 33);
#pragma unroll
      for (int i = 0; i < CH; ++i) xp[lane * 33 + i] = v[i] + col_shift[i];
      s_off[lane] = valid ? pix_off : -1;
      __syncwarp();
      float* o = reinterpret_cast<float*>(p.out) + cbase + lane;
      const bool colok = lane < CH && cbase + lane < p.cout;
#pragma unroll 8
      for (int r = 0; r < 32; ++r) {
        const long long off = s_off[r];
        if (off >= 0 && colok) o[off] = xp[r * 33 + lane];
      }
      __syncwarp();
      return;
    }
    if (valid) {
      float* o = reinterpret_cast<float*>(p.out) + pix_off;
#pragma unroll
      for (int i = 0; i < CH; ++i)
        if (cbase + i < p.cout) o[(long long)(cbase + i) * p.out_sc] = v[i] + col_shift[i];
    }
    return;
  }
  if constexpr (EXT) {
    if (p.epi_mode == EPI_BF16_AFFINE) {
      if (p.scale != nullptr) {
  #pragma unroll
        for (int i = 0; i < CH; i += 4) {
          const float4 sc = *reinterpret_cast<const float4*>(col_scale + i);
          v[i] *= sc.x; v[i + 1] *= sc.y; v[i + 2] *= sc.z; v[i + 3] *= sc.w;
        }
      }
      if (p.shift != nullptr) {
  #pragma unroll
        for (int i = 0; i < CH; i += 4) {
          const float4 sh = *reinterpret_cast<const float4*>(col_shift + i);
          v[i] += sh.x; v[i + 1] += sh.y; v[i + 2] += sh.z; v[i + 3] += sh.w;
        }
      }
    }
    if (p.epi_mode == EPI_BF16_BIAS_RELU) {
  #pragma unroll
      for (int i = 0; i < CH; i += 4) {
        const float4 sh = *reinterpret_cast<const float4*>(col_shift + i);
        v[i] = fmaxf(v[i] + sh.x, 0.f); v[i + 1] = fmaxf(v[i + 1] + sh.y, 0.f);
        v[i + 2] = fmaxf(v[i + 2] + sh.z, 0.f); v[i + 3] = fmaxf(v[i + 3] + sh.w, 0.f);
      }
    }
    if (p.epi_mode == EPI_BF16_RELU_BWD && valid) {
      const __nv_bfloat16* a = p.aux_in + pix_off + cbase;
  #pragma unroll
      for (int i = 0; i < CH; i += 8) {
        if (cbase + i < p.cout) {
          const uint4 u = *reinterpret_cast<const uint4*>(a + i);
          // bf16 sign / zero test on the raw bits: positive and non-zero
          v[i + 0] = (u.x & 0xFFFFu) - 1u < 0x7FFFu ? v[i + 0] : 0.f; v[i + 1] = (u.x >> 16) - 1u < 0x7FFFu ? v[i + 1] : 0.f;
          v[i + 2] = (u.y & 0xFFFFu) - 1u < 0x7FFFu ? v[i + 2] : 0.f; v[i + 3] = (u.y >> 16) - 1u < 0x7FFFu ? v[i + 3] : 0.f;
          v[i + 4] = (u.z & 0xFFFFu) - 1u < 0x7FFFu ? v[i + 4] : 0.f; v[i + 5] = (u.z >> 16) - 1u < 0x7FFFu ? v[i + 5] : 0.f;
          v[i + 6] = (u.w & 0xFFFFu) - 1u < 0x7FFFu ? v[i + 6] : 0.f; v[i + 7] = (u.w >> 16) - 1u < 0x7FFFu ? v[i + 7] : 0.f;
        }
      }
    }
    if (p.epi_mode == EPI_BF16_BIAS_GELU) {
  #pragma unroll
      for (int i = 0; i < CH; i += 4) {
        const float4 sh = *reinterpret_cast<const float4*>(col_shift + i);
        v[i] = bf16_round(v[i] + sh.x); v[i + 1] = bf16_round(v[i + 1] + sh.y);
        v[i + 2] = bf16_round(v[i + 2] + sh.z); v[i + 3] = bf16_round(v[i + 3] + sh.w);
      }
      if (p.aux_out != nullptr && valid) {
        __nv_bfloat16* o = p.aux_out + pix_off + cbase;
  #pragma unroll
        for (int i = 0; i < CH; i += 8)
          if (cbase + i < p.cout) store_bf16x8(o + i, v + i);
      }
  #pragma unroll
      for (int i = 0; i < CH; ++i) v[i] = gelu_erf(v[i]);
    }
    if (p.epi_mode == EPI_BF16_GELU_BWD && valid) {
      const __nv_bfloat16* a = p.aux_in + pix_off + cbase;
  #pragma unroll
      for (int i = 0; i < CH; i += 8) {
        if (cbase + i < p.cout) {
          const uint4 u = *reinterpret_cast<const uint4*>(a + i);
          v[i + 0] *= gelu_erf_grad(bf16_lo(u.x)); v[i + 1] *= gelu_erf_grad(bf16_hi(u.x));
          v[i + 2] *= gelu_erf_grad(bf16_lo(u.y)); v[i + 3] *= gelu_erf_grad(bf16_hi(u.y));
          v[i + 4] *= gelu_erf_grad(bf16_lo(u.z)); v[i + 5] *= gelu_erf_grad(bf16_hi(u.z));
          v[i + 6] *= gelu_erf_grad(bf16_lo(u.w)); v[i + 7] *= gelu_erf_grad(bf16_hi(u.w));
        }
      }
    }
      if (p.addend != nullptr && valid) {
      const __nv_bfloat16* a = p.addend + add_off + cbase;
#pragma unroll
      for (int i = 0; i < CH; i += 8) {
        if (cbase + i < p.cout) {
          const uint4 u = *reinterpret_cast<const uint4*>(a + i);
          v[i + 0] += bf16_lo(u.x); v[i + 1] += bf16_hi(u.x);
          v[i + 2] += bf16_lo(u.y); v[i + 3] += bf16_hi(u.y);
          v[i + 4] += bf16_lo(u.z); v[i + 5] += bf16_hi(u.z);
          v[i + 6] += bf16_lo(u.w); v[i + 7] += bf16_hi(u.w);
        }
      }
    }
    // round once (one packed conversion per two values); the column sums describe exactly the values that are stored
    uint32_t pk[CH / 2];
#pragma unroll
    for (int i = 0; i < CH; i += 2) pk[i >> 1] = pack_bf16x2(v[i], v[i + 1]);
    if (valid) {
      __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + pix_off + cbase;
#pragma unroll
      for (int i = 0; i < CH; i += 8)
        if (cbase + i < p.cout) *reinterpret_cast<uint4*>(o + i) = make_uint4(pk[i >> 1], pk[(i >> 1) + 1], pk[(i >> 1) + 2], pk[(i >> 1) + 3]);
    }
    if ((p.epi_mode == EPI_BF16_GELU_BWD || p.epi_mode == EPI_BF16_RELU_BWD) && p.stat_sum != nullptr) {
#pragma unroll
      for (int i = 0; i < CH; i += 2) {
        v[i] = valid ? bf16_lo(pk[i >> 1]) : 0.f;
        v[i + 1] = valid ? bf16_hi(pk[i >> 1]) : 0.f;
      }
      float cs;
      if constexpr (CH == 32) cs = warp_colsum32(v, lane);
      else cs = warp_colsum16(v, lane);
      if (lane < CH) part_sum[lane] = accumulate ? part_sum[lane] + cs : cs;  // each (warp, column) slot has exactly one writer
    }
  }
}

// ================================================================================================
// Persistent kernel: each CTA walks a strided list of 128-pixel tiles for ONE column tile.
//   warps 0-3, 4-7  two consumer warpgroups.  Warpgroup g computes rows [64 g, 64 g + 64) of the tile with wgmma (accumulator in
//                   registers) and then runs the epilogue of those rows.  The mode selects one of two epilogues, because the output
//                   format forces it:
//                   - TMA store (the 16-bit modes EPI_BF16, EPI_F16, EPI_F16_STATS, EPI_BF16_BN_SILU of EXT = false): the mode's arithmetic
//                     on the accumulator fragment, stmatrix into a swizzled 16-bit tile, one bulk tensor store of the warpgroup's 64 rows
//                     (ConvTmaEpiCfg, ConvOutMaps); an addend tile arrives by TMA into the same buffer and is read with ldmatrix
//                   - staging tile (EPI_F32_BIAS, whose [B, A, 85] rows a tensor map cannot address, and the EXT modes): the accumulator
//                     passes through a per-warpgroup fp32 tile in shared memory, kCols columns per round, so that every epilogue lane owns
//                     one pixel row, as conv_epilogue_chunk expects
//   warp 8          TMA producer: the ring runs ahead across tile boundaries, so the loads of tile i+1 overlap the epilogue of tile i
// Per-channel statistics are accumulated in shared memory over all tiles of the CTA (one fp64 atomic per channel and CTA instead of per
// tile); barrier setup and descriptor prefetch are paid once.
// grid.x = n_tiles * groups;  CTA b: column tile b % n_tiles, pixel tiles (b / n_tiles) + i * groups.
// ================================================================================================
constexpr int kMaxStagesP = 8;      // ring slots; one slot holds kb_per_slot consecutive k-blocks under a single mbarrier
constexpr int kConvThreadsP = 288;  // two consumer warpgroups + one producer warp

template <int BLOCK_N>
struct ConvEpiCfg {
  // accumulator columns staged per round: up to 32 at BN <= 64 (two CTAs per SM: 96 registers per thread), 64 above
  static constexpr int kCols = BLOCK_N <= 64 ? (BLOCK_N < 32 ? BLOCK_N : 32) : 64;
  static_assert(BLOCK_N % kCols == 0, "staging rounds must cover the column tile");
  static constexpr int kPitch = kCols + 4;                    // floats per staged row: 16-byte aligned, conflict-free row reads
  static constexpr int kHalves = BLOCK_N >= 32 ? 2 : 1;       // warps per 32-row quadrant, each taking kCols / kHalves columns of a round
  static constexpr int kChunk = kCols / kHalves;              // 16 or 32 columns per conv_epilogue_chunk
  static constexpr int kStageBytes = 2 * 64 * kPitch * 4;     // both warpgroups
};

// Output tile of the TMA-store epilogue: a warpgroup's 64 rows x BLOCK_N 16-bit columns as boxes of at most 64 columns (a swizzled box row
// is at most 128 bytes), each in the swizzle of its row width (32 / 64 / 128 bytes: stmatrix and ldmatrix are then free of bank conflicts).
// The buffers live in the bytes of the fp32 staging tile, so shared memory and CTAs per SM are the same on both paths: two per warpgroup
// where they fit (BN 16 / 32), else one.
template <int BLOCK_N>
struct ConvTmaEpiCfg {
  static constexpr int kBoxCols = BLOCK_N < 64 ? BLOCK_N : 64;
  static constexpr int kBoxes = BLOCK_N / kBoxCols;
  static constexpr int kRowBytes = 2 * kBoxCols;  // = the swizzle span
  static constexpr int kBoxBytes = 64 * kRowBytes;
  static constexpr int kBufBytes = kBoxes * kBoxBytes;
  static constexpr int kBufs = 2 * 2 * kBufBytes <= ConvEpiCfg<BLOCK_N>::kStageBytes ? 2 : 1;
  static_assert(2 * kBufs * kBufBytes <= ConvEpiCfg<BLOCK_N>::kStageBytes, "output tiles must fit in the staging tile's bytes");
};

// Tensor maps of the TMA-store epilogue: the 16-bit output view and the addend as (c, x, y, n) over the pixel grid of the work items, with
// the view's own extents, so that TMA clipping drops the columns beyond the view's channels and the pixels beyond the valid grid.  A
// four-phase data gradient has one map per output-parity phase (ph, pw) at index 2 ph + pw; other launches use index 0.
struct ConvOutMaps {
  CUtensorMap out[4];
  CUtensorMap add[4];
};

__host__ __device__ constexpr int conv_min_ctas(int block_n, int block_k) { return (block_n >= 128 || block_k == 16) ? 1 : 2; }

// The 64-row half of a (tw, th, tn) pixel tile that warpgroup g stores: the outermost dimension longer than one pixel is halved.  Offsets of
// half 1 in (x, y, n); the TMA box is the tile with that dimension halved (conv_api.cu).
__host__ __device__ inline void conv_half_offset(int log_tw, int log_th, int& dx, int& dy, int& dn) {
  const int log_tn = 7 - log_tw - log_th;
  dx = dy = dn = 0;
  if (log_tn > 0) dn = 1 << (log_tn - 1);
  else if (log_th > 0) dy = 1 << (log_th - 1);
  else dx = 1 << (log_tw - 1);
}

// EXT: false = YOLOX training / inference epilogues, true = + ConvNeXt / transformer epilogues
template <int BLOCK_N, int BLOCK_K, bool EXT>
// two CTAs per SM (96 registers per thread: five of their 18 warps share one 16 K-register SM sub-partition) where that fits without
// spilling; one CTA per SM (168 registers) for BN 128 and for BLOCK_K 16 (the deep k-block slots); conv_min_ctas
__global__ void __launch_bounds__(kConvThreadsP, conv_min_ctas(BLOCK_N, BLOCK_K))
conv_gemm_persistent_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                            const __grid_constant__ ConvGemmParams p, const __grid_constant__ ConvOutMaps om, int num_stages, int kb_per_slot,
                            int n_tiles, int m_tiles) {
  using Cfg = ConvGemmCfg<BLOCK_N, BLOCK_K>;
  using Epi = ConvEpiCfg<BLOCK_N>;
  using TE = ConvTmaEpiCfg<BLOCK_N>;
  static_assert(Cfg::kStageBytes % (8 * TE::kRowBytes) == 0, "output tiles must start on a swizzle-pattern boundary");
  constexpr int CH = Epi::kChunk;
  extern __shared__ uint8_t smem_dyn[];
  __shared__ __align__(8) uint64_t s_bar[2 * kMaxStagesP + 4];  // ring full / empty, then the addend tiles [warpgroup][buffer]
  __shared__ float s_part[4][2][BLOCK_N];
  __shared__ __align__(16) float s_col[2][BLOCK_N];

  const int warp = warp_id_uniform();
  const int lane = threadIdx.x & 31;
  const uint32_t smem_base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  uint8_t* const smem_al = smem_dyn + (smem_base - smem_u32(smem_dyn));
  const int ring_bytes = num_stages * kb_per_slot * Cfg::kStageBytes;
  const uint32_t bar_full = smem_u32(&s_bar[0]);
  const uint32_t bar_empty = smem_u32(&s_bar[kMaxStagesP]);
  const uint32_t bar_add = smem_u32(&s_bar[2 * kMaxStagesP]);
  const bool tma_epi = !EXT && p.epi_mode != EPI_F32_BIAS;

  const int n_tile = blockIdx.x % n_tiles;
  const int group = blockIdx.x / n_tiles;
  const int groups = gridDim.x / n_tiles;
  const int col0 = n_tile * BLOCK_N;
  const int log_tw = p.log_tw, log_th = p.log_th;

  if (threadIdx.x == 0) {
    for (int s = 0; s < num_stages; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, 2);  // one arrival per consumer warpgroup
    }
    for (int s = 0; s < 4; ++s) mbar_init(bar_add + 8 * s, 1);
    mbar_fence_init();
  }
  for (int i = threadIdx.x; i < 4 * 2 * BLOCK_N; i += blockDim.x) (&s_part[0][0][0])[i] = 0.f;
  pdl_sync();  // everything above touches only this CTA's shared memory: it overlaps the tail of the previous kernel
  stage_col_params<BLOCK_N>(p, col0, s_col);
  __syncthreads();

  if (warp == 8) {
    // ===================== TMA producer =====================
    if (elect_one()) {
      tma_prefetch_desc(&tmA);
      tma_prefetch_desc(&tmB);
      int stage = 0;
      uint32_t phase = 0;
      for (int wi = group; wi < m_tiles; wi += groups) {  // m_tiles counts work items (pixel tiles x phases)
        int m, tap, ntaps, oph, opw;
        conv_decode_work(p, wi, m, tap, ntaps, oph, opw);
        const int num_kb = ntaps * p.cin_blocks;
        int t = m;
        const int tw = t % p.tiles_w;
        t /= p.tiles_w;
        const int th = t % p.tiles_h;
        const int tn = t / p.tiles_h;
        const int w0 = tw << log_tw, h0 = th << log_th, n0 = tn << (7 - log_tw - log_th);
        int cb = 0;
        for (int kb = 0; kb < num_kb; kb += kb_per_slot) {  // num_kb is a multiple of kb_per_slot
          mbar_wait(bar_empty + 8 * stage, phase ^ 1u);
          const uint32_t full = bar_full + 8 * stage;
          mbar_expect_tx(full, Cfg::kStageBytes * kb_per_slot);
          for (int j = 0; j < kb_per_slot; ++j) {
            const uint32_t sa = smem_base + (stage * kb_per_slot + j) * Cfg::kStageBytes;
            const ConvTap& tp = p.taps[tap];
            tma_load_5d(sa, &tmA, full, tp.c0 + cb * BLOCK_K, w0 + tp.dw, tp.p, h0 + tp.dh, n0);
            tma_load_2d(sa + Cfg::kABytes, &tmB, full, tp.kb + cb * BLOCK_K, col0 + n0 * p.b_img_rows);
            if (++cb == p.cin_blocks) { cb = 0; ++tap; }
          }
          if (++stage == num_stages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else if (warp < 8) {
    // ===================== consumer warpgroups: MMA, then the epilogue of their 64 rows =====================
    const int g = warp >> 2;         // rows [64 g, 64 g + 64) of the tile
    const int wl = warp & 3;
    const int q = 2 * g + (wl & 1);  // 32-row quadrant whose epilogue (staging path) or statistics (both paths) this warp runs
    const int half = wl >> 1;        // which part of each staged round of columns
    const int mrow = q * 32 + lane;
    const int xl = mrow & ((1 << log_tw) - 1);
    const int yl = (mrow >> log_tw) & ((1 << log_th) - 1);
    const int nl = mrow >> (log_tw + log_th);
    float* const stg = reinterpret_cast<float*>(smem_al + ring_bytes) + g * 64 * Epi::kPitch;
    float* xp = nullptr;
    if (p.xpose) xp = reinterpret_cast<float*>(smem_al + ring_bytes + Epi::kStageBytes) + warp * kXposeWarpFloats;
    // TMA path: the leader thread of the warpgroup issues, commits and waits for its bulk copies (bulk async-groups are per thread)
    const bool leader = (threadIdx.x & 127) == 0;
    const bool add_tile = tma_epi && p.addend != nullptr;
    const uint32_t obuf = smem_base + ring_bytes + g * TE::kBufs * TE::kBufBytes;
    // stmatrix / ldmatrix rows of this lane: lanes 8j .. 8j + 7 address matrix j = rows + 8 (j & 1), column block + (j >> 1); the 16-byte
    // chunk index is XORed with address bits 7 and up (the TMA swizzle of kRowBytes-wide rows)
    const int srow = 16 * wl + (lane & 7) + 8 * ((lane >> 3) & 1);
    const uint32_t srow_off = srow * TE::kRowBytes;
    const uint32_t schunk = (lane >> 4) ^ ((srow_off >> 7) & (TE::kRowBytes / 16 - 1));
    int hx, hy, hn;
    conv_half_offset(log_tw, log_th, hx, hy, hn);
    hx *= g; hy *= g; hn *= g;
    if (tma_epi && leader) {
      tma_prefetch_desc(&om.out[0]);
      if (add_tile) tma_prefetch_desc(&om.add[0]);
    }
    constexpr uint32_t lcode = gmma_layout_code(Cfg::kSwizzle);
    constexpr uint32_t sbo = 8 * Cfg::kSwizzle;  // 8 rows of one swizzle atom
    float acc[BLOCK_N / 2];
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;  // defined on every path into the first wgmma (which overwrites it: scale-d 0)
    wgmma_fence_operand(acc);
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;  // tiles of this CTA so far
    for (int wi = group; wi < m_tiles; wi += groups, ++it) {
      int m, tap, ntaps, oph, opw;
      conv_decode_work(p, wi, m, tap, ntaps, oph, opw);
      const int num_kb = ntaps * p.cin_blocks;
      int t = m;
      const int tw = t % p.tiles_w;
      t /= p.tiles_w;
      const int th = t % p.tiles_h;
      const int tn = t / p.tiles_h;
      const int w0 = tw << log_tw, h0 = th << log_th, n0 = tn << (7 - log_tw - log_th);
      const int pm = p.num_phases == 4 ? 2 * oph + opw : 0;
      const int slot = TE::kBufs == 2 ? (it & 1) : 0;
      const uint32_t buf = obuf + slot * TE::kBufBytes;
      const uint32_t abar = bar_add + 8 * (2 * g + slot);
      if (add_tile && leader) {
        // the addend tile goes to the buffer that this tile's output will occupy; its latency hides behind the main loop
        if (TE::kBufs == 1) bulk_wait_read<0>();  // the previous tile's store has read the buffer
        mbar_expect_tx(abar, TE::kBufBytes);
#pragma unroll
        for (int b = 0; b < TE::kBoxes; ++b) tma_load_4d(buf + b * TE::kBoxBytes, &om.add[pm], abar, col0 + 64 * b, w0 + hx, h0 + hy, n0 + hn);
      }
      int j = 0, prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {  // one wgmma group per k-block; ring slots hold kb_per_slot of them
        if (j == 0) mbar_wait(bar_full + 8 * stage, phase);
        const uint32_t sa = smem_base + (stage * kb_per_slot + j) * Cfg::kStageBytes + g * 64 * Cfg::kSwizzle;
        const uint32_t sb = smem_base + (stage * kb_per_slot + j) * Cfg::kStageBytes + Cfg::kABytes;
        wgmma_fence_operand(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / 16; ++k)
          Wgmma<BLOCK_N>::template mma<0, 0>(acc, gmma_desc(sa + k * 32, 16, sbo, lcode), gmma_desc(sb + k * 32, 16, sbo, lcode), (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs have completed
        wgmma_fence_operand(acc);
        // first k-block of a slot: every k-block of the previous slot has completed, hand that slot back to the producer
        mbar_arrive_if(bar_empty + 8 * prev, j == 0 && prev >= 0 && (threadIdx.x & 127) == 0);
        if (++j == kb_per_slot) {
          j = 0;
          prev = stage;
          if (++stage == num_stages) { stage = 0; phase ^= 1u; }
        }
      }
      wgmma_wait<0>();
      wgmma_fence_operand(acc);
      mbar_arrive_if(bar_empty + 8 * prev, (threadIdx.x & 127) == 0);

      if (tma_epi) {
        if (TE::kBufs == 1 && !add_tile) {  // the previous tile's store has read the buffer (with an addend: implied by its arrival)
          if (leader) bulk_wait_read<0>();
          named_bar_sync(1 + g, 128);
        }
        // fragment: acc[4 i + e] is row 16 wl + lane / 4 + 8 (e >> 1), column 8 i + 2 (lane % 4) + (e & 1) of the warpgroup's rows
        if (p.epi_mode == EPI_BF16_BN_SILU) {
#pragma unroll
          for (int i = 0; i < BLOCK_N / 8; ++i) {
            const float2 sc = *reinterpret_cast<const float2*>(&s_col[0][8 * i + 2 * (lane & 3)]);
            const float2 sh = *reinterpret_cast<const float2*>(&s_col[1][8 * i + 2 * (lane & 3)]);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float u = fmaf(acc[4 * i + e], (e & 1) ? sc.y : sc.x, (e & 1) ? sh.y : sh.x);
              acc[4 * i + e] = bf16_round(__fdividef(u, 1.f + __expf(-u)));  // rounded before the residual add, as a materialised activation
            }
          }
        }
        if (add_tile) {
          mbar_wait(abar, (it / TE::kBufs) & 1);
#pragma unroll
          for (int i = 0; i < BLOCK_N / 8; i += 2) {
            uint32_t a[4];
            ldmatrix_x4(buf + (i >> 3) * TE::kBoxBytes + srow_off + (((i & 7) ^ schunk) << 4), a[0], a[1], a[2], a[3]);
#pragma unroll
            for (int r = 0; r < 4; ++r) {
              acc[4 * i + 2 * r] += bf16_lo(a[r]);
              acc[4 * i + 2 * r + 1] += bf16_hi(a[r]);
            }
          }
        }
        // round once: pk[2 i] holds row lane / 4 and pk[2 i + 1] row lane / 4 + 8 of column pair 8 i + 2 (lane % 4)
        uint32_t pk[BLOCK_N / 4];
        if (p.epi_mode == EPI_F16 || p.epi_mode == EPI_F16_STATS) {
#pragma unroll
          for (int i = 0; i < BLOCK_N / 4; ++i) pk[i] = pack_f16x2(acc[2 * i], acc[2 * i + 1]);
        } else {
#pragma unroll
          for (int i = 0; i < BLOCK_N / 4; ++i) pk[i] = pack_bf16x2(acc[2 * i], acc[2 * i + 1]);
        }
#pragma unroll
        for (int i = 0; i < BLOCK_N / 8; i += 2)
          stmatrix_x4(buf + (i >> 3) * TE::kBoxBytes + srow_off + (((i & 7) ^ schunk) << 4), pk[2 * i], pk[2 * i + 1], pk[2 * i + 2], pk[2 * i + 3]);
        fence_proxy_async_smem();
        // two buffers: the previous tile's store has read the other one before any thread passes this barrier, so the next tile may fill it
        if (TE::kBufs == 2 && leader) bulk_wait_read<0>();
        named_bar_sync(1 + g, 128);
        if (leader) {
#pragma unroll
          for (int b = 0; b < TE::kBoxes; ++b) tma_store_4d(&om.out[pm], buf + b * TE::kBoxBytes, col0 + 64 * b, w0 + hx, h0 + hy, n0 + hn);
          bulk_commit();
        }
        if (p.epi_mode == EPI_F16_STATS) {
          // Σ and Σ² of the stored values, read back from the output tile (the store only reads it as well; the next write to this buffer
          // follows a barrier that every thread passes after these reads), in exactly the order of the staging path: one pixel row per lane
          // and 16 or 32 columns per warp, a butterfly over the 32 rows of a quadrant, per-quadrant sums over the CTA's tiles.  The sums are
          // then the same fp32 additions as on the parent's path, and a training step computes the same BatchNorm statistics bit for bit.
          const bool valid = w0 + xl < p.w_valid && h0 + yl < p.h_valid && n0 + nl < p.n_valid;
          const uint32_t row = (wl & 1) * 32 + lane;  // this lane's row of the warpgroup's tile
          const uint32_t rxor = ((row * TE::kRowBytes) >> 7) & (TE::kRowBytes / 16 - 1);
#pragma unroll 1
          for (int r = 0; r < BLOCK_N / Epi::kCols; ++r) {
            const int c = r * Epi::kCols + half * CH;
            if (half < Epi::kHalves && col0 + c < p.cout) {
              float v[CH], sq[CH];
#pragma unroll
              for (int i = 0; i < CH; i += 8) {
                const int cc = c + i;
                uint4 u;
                asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
                             : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w)
                             : "r"(buf + (cc / TE::kBoxCols) * TE::kBoxBytes + row * TE::kRowBytes + ((((cc % TE::kBoxCols) >> 3) ^ rxor) << 4))
                             : "memory");
                const uint32_t w4[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  __half2 hv;
                  *reinterpret_cast<uint32_t*>(&hv) = w4[j];
                  const float2 fv = __half22float2(hv);
                  v[i + 2 * j] = valid ? fv.x : 0.f;
                  v[i + 2 * j + 1] = valid ? fv.y : 0.f;
                }
              }
#pragma unroll
              for (int i = 0; i < CH; ++i) sq[i] = v[i] * v[i];
              float cs, cq;
              if constexpr (CH == 32) { cs = warp_colsum32(v, lane); cq = warp_colsum32(sq, lane); }
              else { cs = warp_colsum16(v, lane); cq = warp_colsum16(sq, lane); }
              if (lane < CH) {  // each (quadrant, column) slot has exactly one writer
                s_part[q][0][c + lane] += cs;
                s_part[q][1][c + lane] += cq;
              }
            }
          }
        }
      } else {
        const int x = w0 + xl, y = h0 + yl, n = n0 + nl;
        const bool valid = (x < p.w_valid) && (y < p.h_valid) && (n < p.n_valid);
        const long long pix_off = (long long)n * p.out_sn + (long long)(y * p.out_mh + oph) * p.out_sh +
                                  (long long)(x * p.out_mw + opw) * p.out_sw;
        const long long add_off = (long long)n * p.add_sn + (long long)(y * p.out_mh + oph) * p.add_sh +
                                  (long long)(x * p.out_mw + opw) * p.add_sw;
        float* const r0 = stg + (16 * wl + (lane >> 2)) * Epi::kPitch + 2 * (lane & 3);  // this thread's fragment rows in the staging tile
        float* const r1 = r0 + 8 * Epi::kPitch;
        const float* const row_src = stg + ((wl & 1) * 32 + lane) * Epi::kPitch + half * CH;
#pragma unroll 1
        for (int r = 0; r < BLOCK_N / Epi::kCols; ++r) {
          named_bar_sync(1 + g, 128);  // every row of the previous round has been read
#pragma unroll
          for (int i = 0; i < BLOCK_N / 8; ++i) {
            if (i / (Epi::kCols / 8) == r) {
              const int c = (i % (Epi::kCols / 8)) * 8;
              *reinterpret_cast<float2*>(r0 + c) = make_float2(acc[4 * i], acc[4 * i + 1]);
              *reinterpret_cast<float2*>(r1 + c) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
            }
          }
          named_bar_sync(1 + g, 128);
          const int c = r * Epi::kCols + half * CH;  // tile column of this warp's chunk
          // chunks at or beyond the last valid output channel are dead (cout not a multiple of the column tile)
          if (half < Epi::kHalves && col0 + c < p.cout) {
            float v[CH];
#pragma unroll
            for (int i = 0; i < CH; i += 4) {
              const float4 f = *reinterpret_cast<const float4*>(row_src + i);
              v[i] = f.x; v[i + 1] = f.y; v[i + 2] = f.z; v[i + 3] = f.w;
            }
            conv_epilogue_chunk<CH, EXT>(p, v, valid, pix_off, add_off, col0 + c, lane, &s_part[q][0][c], true, &s_col[0][c], &s_col[1][c], xp);
          }
        }
      }
    }
    if (tma_epi && leader) bulk_wait_all();  // the stores have completed before the CTA's shared memory is released
  }

  __syncthreads();
  if (EXT ? epi_has_stats(p.epi_mode, p.stat_sum) : p.epi_mode == EPI_F16_STATS) {
    for (int e = threadIdx.x; e < BLOCK_N && col0 + e < p.cout; e += blockDim.x) {  // BLOCK_N may exceed the thread count
      const float s1 = (s_part[0][0][e] + s_part[1][0][e]) + (s_part[2][0][e] + s_part[3][0][e]);
      const float s2 = (s_part[0][1][e] + s_part[1][1][e]) + (s_part[2][1][e] + s_part[3][1][e]);
      const int ch = p.stat_fold > 0 ? (col0 + e) % p.stat_fold : col0 + e;
      atomicAdd(p.stat_sum + ch, static_cast<double>(s1));
      if (p.stat_sq != nullptr) atomicAdd(p.stat_sq + ch, static_cast<double>(s2));
    }
  }
}

}  // namespace yb
