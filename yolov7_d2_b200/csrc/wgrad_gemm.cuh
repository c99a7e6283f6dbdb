// Weight-gradient GEMM on wgmma (sm_90a).
//
//   dW_tap[co, ci] = sum over pixels  dz[px, co] * x_tap[px, ci]
//
// Both operands are NHWC bf16 tensors, i.e. the contraction index (pixel) is the *slow* index of each
// smem tile: "MN-major" descriptors for both wgmma operands.  dz tiles are dense 64-pixel boxes; x tiles are the same boxes
// displaced by the tap (identical TMA maps / tap tables as the forward kernel), so zero padding and stride-2
// need no extra code.  One CTA owns (cout tile of 128) x (cin tile of BN) x (tap group) x (pixel range); two consumer warpgroups
// (64 cout rows each) keep one fp32 accumulator per tap in registers; partial tiles go to a split-K workspace reduced by
// wgrad_reduce_kernel (deterministic, no atomics).
#pragma once
#include "sm90.cuh"
#include "conv_gemm.cuh"

namespace yb {

constexpr int kWgPix = 64;       // pixels per K block (4 wgmma K-steps)
constexpr int kWgThreads = 288;  // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int kWgStages = 3;     // default ring depth (keeps two CTAs per SM on the small layers)
constexpr int kWgMaxStages = 6;  // one-CTA-per-SM plans (the pixel-grouped stem: 40 KB stages) take as many as fit: the kernel is latency bound otherwise

struct WgradParams {
  int tiles_w, tiles_h, tiles_n;  // 64-pixel tiles over the dz pixel grid
  int log_tw, log_th;
  int num_blocks;                 // total pixel blocks = tiles_w*tiles_h*tiles_n
  int blocks_per_split;
  int cout, cin;                  // logical sizes (cin = padded K per tap)
  int kc_a, ma;                   // dz channel box width (<=64) and number of boxes per 128-row tile
  int kc_b, nb;                   // x channel box width (<=64) and boxes per BN tile
  int bn;                         // cin tile width = kc_b*nb
  int tpc, tap_groups, num_taps;  // taps per CTA, groups, total taps
  int stages;                     // ring depth (kWgStages .. kWgMaxStages)
  int cin_tiles, cout_tiles;
  int dz_c0;                      // channel offset of dz slice inside its buffer
  float* ws;                      // [split][cout][num_taps][cin] fp32
  ConvTap taps[kMaxTaps];         // x taps (c0, dw, p, dh).  ks > 0 (pixel-grouped stem, yb200_conv2d_wgrad_grouped): only the first 16 * ks channels
                                  // of this tap's x box matter (the box starts at the one neighbour pixel that does): the epilogue stores those
                                  // accumulator columns at input channel kb (a multiple of 8), zeros elsewhere
};

// one CTA-resident accumulator of 64 x BN fp32 per tap and warpgroup: TPC * BN / 2 registers per thread
template <int BN, int TPC>
__global__ void __launch_bounds__(kWgThreads, TPC * BN <= 96 ? 2 : 1)
wgrad_gemm_kernel(const __grid_constant__ CUtensorMap tmDz, const __grid_constant__ CUtensorMap tmX,
                  const __grid_constant__ WgradParams p) {
  pdl_sync();
  extern __shared__ uint8_t smem_dyn[];
  __shared__ __align__(8) uint64_t s_bar[2 * kWgMaxStages];
  const int num_stages = p.stages;

  const int warp = warp_id_uniform();
  const int lane = threadIdx.x & 31;
  const uint32_t smem_base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  const uint32_t bar_full = smem_u32(&s_bar[0]);
  const uint32_t bar_empty = smem_u32(&s_bar[kWgMaxStages]);

  // work decomposition: blockIdx.x = ((cout_tile * cin_tiles + cin_tile) * tap_groups + group), blockIdx.y = split
  int w = blockIdx.x;
  const int group = w % p.tap_groups;
  w /= p.tap_groups;
  const int cin_tile = w % p.cin_tiles;
  const int cout_tile = w / p.cin_tiles;
  const int split = blockIdx.y;
  const int tap0 = group * p.tpc;
  const int ntap = min(p.tpc, p.num_taps - tap0);
  const int blk_begin = split * p.blocks_per_split;
  const int blk_end = min(p.num_blocks, blk_begin + p.blocks_per_split);
  const int nblk = blk_end - blk_begin;

  const uint32_t a_box_bytes = kWgPix * p.kc_a * 2;
  const uint32_t b_box_bytes = kWgPix * p.kc_b * 2;
  const uint32_t a_bytes = a_box_bytes * p.ma;
  const uint32_t b_tap_bytes = b_box_bytes * p.nb;
  const uint32_t stage_bytes = a_bytes + b_tap_bytes * p.tpc;  // constant stride even for a short last group

  if (threadIdx.x == 0) {
    for (int s = 0; s < num_stages; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, 2);  // one arrival per consumer warpgroup
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (elect_one()) {
      tma_prefetch_desc(&tmDz);
      tma_prefetch_desc(&tmX);
      int stage = 0;
      uint32_t phase = 0;
      for (int b = 0; b < nblk; ++b) {
        int t = blk_begin + b;
        const int tw = t % p.tiles_w;
        t /= p.tiles_w;
        const int th = t % p.tiles_h;
        const int tn = t / p.tiles_h;
        const int w0 = tw << p.log_tw, h0 = th << p.log_th, n0 = tn << (6 - p.log_tw - p.log_th);
        mbar_wait(bar_empty + 8 * stage, phase ^ 1u);
        const uint32_t sa = smem_base + stage * stage_bytes;
        const uint32_t full = bar_full + 8 * stage;
        mbar_expect_tx(full, a_bytes + b_tap_bytes * ntap);
        for (int j = 0; j < p.ma; ++j)
          tma_load_5d(sa + j * a_box_bytes, &tmDz, full, p.dz_c0 + cout_tile * 128 + j * p.kc_a, w0, 0, h0, n0);
        for (int ti = 0; ti < ntap; ++ti) {
          const ConvTap& tp = p.taps[tap0 + ti];
          const uint32_t sb = sa + a_bytes + ti * b_tap_bytes;
          for (int j = 0; j < p.nb; ++j)
            tma_load_5d(sb + j * b_box_bytes, &tmX, full, tp.c0 + cin_tile * p.bn + j * p.kc_b, w0 + tp.dw, tp.p,
                        h0 + tp.dh, n0);
        }
        if (++stage == num_stages) { stage = 0; phase ^= 1u; }
      }
    }
  } else if (warp < 8) {
    const int g = warp >> 2;                     // cout rows [64 g, 64 g + 64) of the tile
    const int rows = p.ma * p.kc_a;              // cout rows of this tile's boxes (128, or the whole slice when narrower)
    const bool active = 64 * g < rows;
    const uint32_t lcode_a = gmma_layout_code(p.kc_a * 2);
    const uint32_t lcode_b = gmma_layout_code(p.kc_b * 2);
    const uint32_t row_a = p.kc_a * 2, row_b = p.kc_b * 2;
    // MN-major canonical layout: LBO = byte distance between channel boxes, SBO = 8 pixel rows.  When the cout tile is narrower than
    // 64 rows the extra rows alias box 0 (LBO 0): they only produce accumulator rows that are never stored.
    const uint32_t lbo_a = rows >= 64 ? a_box_bytes : 0u;
    const uint32_t a_off = static_cast<uint32_t>(64 * g / p.kc_a) * a_box_bytes;
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    if (!active) {  // no rows of this tile in this warpgroup: hand the slots back, nothing else
      for (int b = 0; b < nblk; ++b) {
        mbar_wait(bar_full + 8 * stage, phase);
        mbar_arrive_if(bar_empty + 8 * prev, prev >= 0 && (threadIdx.x & 127) == 0);
        prev = stage;
        if (++stage == num_stages) { stage = 0; phase ^= 1u; }
      }
      mbar_arrive_if(bar_empty + 8 * prev, prev >= 0 && (threadIdx.x & 127) == 0);
      return;
    }
    float acc[TPC][BN / 2];
#pragma unroll
    for (int ti = 0; ti < TPC; ++ti)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[ti][i] = 0.f;
#pragma unroll
    for (int ti = 0; ti < TPC; ++ti) wgmma_fence_operand(acc[ti]);  // opaque zeros: not rematerialised between the wgmma of a stage
    for (int b = 0; b < nblk; ++b) {
      mbar_wait(bar_full + 8 * stage, phase);
      const uint32_t sa = smem_base + stage * stage_bytes;
      wgmma_fence();
      // every tap slot of the stage, also those of a short last tap group: their products land in accumulators that are never stored
#pragma unroll
      for (int ti = 0; ti < TPC; ++ti) {
        const uint32_t sb = sa + a_bytes + ti * b_tap_bytes;
#pragma unroll
        for (int k = 0; k < kWgPix / 16; ++k)
          Wgmma<BN>::template mma<1, 1>(acc[ti], gmma_desc(sa + a_off + k * 16 * row_a, lbo_a, 8 * row_a, lcode_a),
                                        gmma_desc(sb + k * 16 * row_b, b_box_bytes, 8 * row_b, lcode_b), 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();  // the previous block's MMAs have completed: hand its slot back to the producer
      mbar_arrive_if(bar_empty + 8 * prev, prev >= 0 && (threadIdx.x & 127) == 0);
      prev = stage;
      if (++stage == num_stages) { stage = 0; phase ^= 1u; }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int ti = 0; ti < TPC; ++ti) wgmma_fence_operand(acc[ti]);
    mbar_arrive_if(bar_empty + 8 * prev, prev >= 0 && (threadIdx.x & 127) == 0);

    // accumulator fragment -> split-K workspace: thread rows r and r + 8, columns 8 i + 2 (lane % 4) + {0, 1}
    const int r = 64 * g + 16 * (warp & 3) + (lane >> 2);
    const int cpair = 2 * (lane & 3);
    float* wsb = p.ws + (long long)split * p.cout * p.num_taps * p.cin;
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int row = r + 8 * hr;
      const int co = cout_tile * 128 + row;
      if (row >= rows || co >= p.cout) continue;
#pragma unroll
      for (int ti = 0; ti < TPC; ++ti) {
        if (ti >= ntap) continue;
        float* dst = wsb + ((long long)co * p.num_taps + tap0 + ti) * p.cin + cin_tile * BN + cpair;
        const int ks = p.taps[tap0 + ti].ks, shift = p.taps[tap0 + ti].kb;
        if (ks == 0) {
#pragma unroll
          for (int i = 0; i < BN / 8; ++i)
            *reinterpret_cast<float2*>(dst + 8 * i) = make_float2(acc[ti][4 * i + 2 * hr], acc[ti][4 * i + 2 * hr + 1]);
        } else {  // sparse tap: accumulator columns [0, 16 ks) belong at input channels [shift, shift + 16 ks)
#pragma unroll
          for (int i = 0; i < BN / 8; ++i)
            if (8 * i < shift || 8 * i >= shift + 16 * ks) *reinterpret_cast<float2*>(dst + 8 * i) = make_float2(0.f, 0.f);
#pragma unroll
          for (int i = 0; i < BN / 8; ++i)
            if (8 * i < 16 * ks && shift + 8 * i < BN)
              *reinterpret_cast<float2*>(dst + shift + 8 * i) = make_float2(acc[ti][4 * i + 2 * hr], acc[ti][4 * i + 2 * hr + 1]);
        }
      }
    }
  }
}

// Sum the split-K partials and scatter into the reference's OIHW fp32 gradient layout
// (torch.nn.Conv2d.weight.grad: [Cout][Cin][kh][kw]); padded input channels (ci >= cin_real) are dropped.
// accumulate != 0 adds to the existing gradient (gradient accumulation across micro-batches).
// block = (32 outputs, 8 split lanes): the serial chain over splits is 8x shorter; partials are combined in a fixed order
__global__ void __launch_bounds__(256)
wgrad_reduce_kernel(const float* __restrict__ ws, float* __restrict__ grad_oihw, int splits, int cout, int num_taps, int cin_pad,
                    int cin_real, int accumulate) {
  pdl_sync();
  __shared__ float part[8][33];
  const unsigned total = static_cast<unsigned>(cout) * num_taps * cin_pad;
  const unsigned tc = static_cast<unsigned>(num_taps) * cin_pad;
  const int ox = threadIdx.x & 31, sl = threadIdx.x >> 5;
  for (unsigned base = blockIdx.x * 32u; base < total; base += gridDim.x * 32u) {
    const unsigned i = base + ox;
    float acc = 0.f;
    if (i < total) {
      // four independent loads in flight per thread (the kernel is latency bound: one 4-byte load per thread and iteration otherwise);
      // fixed association order, so the result does not depend on the launch
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
      int s = sl;
      for (; s + 24 < splits; s += 32) {
        a0 += ws[static_cast<size_t>(s) * total + i];
        a1 += ws[static_cast<size_t>(s + 8) * total + i];
        a2 += ws[static_cast<size_t>(s + 16) * total + i];
        a3 += ws[static_cast<size_t>(s + 24) * total + i];
      }
      for (; s < splits; s += 8) a0 += ws[static_cast<size_t>(s) * total + i];
      acc = (a0 + a1) + (a2 + a3);
    }
    part[sl][ox] = acc;
    __syncthreads();
    if (sl == 0 && i < total) {
      const float v = ((part[0][ox] + part[1][ox]) + (part[2][ox] + part[3][ox])) + ((part[4][ox] + part[5][ox]) + (part[6][ox] + part[7][ox]));
      const unsigned co = i / tc;
      const unsigned r = i - co * tc;
      const unsigned tap = r / cin_pad;
      const unsigned ci = r - tap * cin_pad;
      if (ci < static_cast<unsigned>(cin_real)) {
        float* g = grad_oihw + (static_cast<size_t>(co) * cin_real + ci) * num_taps + tap;
        *g = accumulate ? (*g + v) : v;
      }
    }
    __syncthreads();
  }
}

}  // namespace yb
