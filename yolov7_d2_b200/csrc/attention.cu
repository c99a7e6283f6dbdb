// Multi-head attention core on wgmma (SURVEY.md par.8a row T1): the part of nn.MultiheadAttention between in_proj and out_proj
//   out[b, i, h] = softmax_j( scale * <q[b,i,h], k[b,j,h]> + key_padding_mask[b,j] ) . v[b,j,h]
// as used by TransformerEncoderLayer / TransformerDecoderLayer (yolov7/modeling/backbone/detr_backbone.py:140,157-161,200-236: d_model 256,
// 8 heads x 32, sequences of 1050 tokens at 800x1333).  Head dimension 32 is compiled in.
//
// One CTA per (128-query tile, head, image); flash-attention style streaming over 128-key tiles:
//   warp 4     TMA producer: Q tile once, K / V tiles double-buffered (5-D NHWC maps, out-of-range tokens zero-filled)
//   warps 0-3  one warpgroup: S = Q K^T (wgmma 64x128x16, K-major operands, 64 query rows at a time) staged as fp32 rows in shared memory,
//              online softmax with one query row per thread (running max / sum in the exp2 domain), P written as bf16 into a 128B-swizzled
//              K-major tile, O_j = P V (wgmma 64x32x16, V as MN-major B operand straight from its token-major tile) staged the same way and
//              folded into the running output kept in registers (acc = (acc + O_j) * alpha)
// With 32-wide heads the kernel is bound by MUFU.EX2 (128 x 128 exponentials per tile against 2 MFLOP of MMA).
#include "host_common.cuh"
#include "sm90.cuh"

using namespace yb;

namespace {

constexpr int kAttD = 32;          // head dimension
constexpr int kAttTile = 128;      // queries per CTA, keys per step
constexpr int kAttThreads = 160;   // one compute warpgroup + one producer warp
constexpr int kQBytes = kAttTile * kAttD * 2;       // 8 KB, 64-byte rows (swizzle 64)
constexpr int kKVBytes = kAttTile * kAttD * 2;
constexpr int kPBytes = kAttTile * kAttTile * 2;    // 32 KB: two K-blocks of [128 rows][64 keys] with 128-byte rows (swizzle 128)
constexpr int kSPitch = kAttTile + 4;               // fp32 row pitch of a staged score tile (16-byte aligned, conflict-free row reads)
constexpr int kOPitch = kAttD + 4;                  // fp32 row pitch of a staged [128][32] output tile
constexpr int kSBytes = kAttTile * kSPitch * 4;     // 66 KB: staged S (forward), later the staged O_j
constexpr int kAttSmem = kQBytes + 4 * kKVBytes + kPBytes + kSBytes + 1024;

__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Dropout (nn.MultiheadAttention(dropout=p) on the attention probabilities, nn.Dropout on the residual branches / the FFN, detr_backbone.py:140-152,
// 200-214): a counter-based hash instead of torch's Philox stream -- keep(element) = (mix32(seed-derived key ^ index * golden) >> 8) >= p * 2^24 -- so the
// backward kernels regenerate the mask of the forward from (seed, indices) alone.  thr24 == 0 disables it (p = 0 / eval: not a single extra instruction).
struct DropParams {
  uint32_t seed, thr24;
  float inv_keep;
};
__host__ __device__ __forceinline__ uint32_t mix32(uint32_t h) {
  h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16;
  return h;
}
// per-row key of the attention mask: (seed, image * heads + head, query index)
__device__ __forceinline__ uint32_t drop_row_key(uint32_t seed, uint32_t bh, uint32_t q) { return mix32(seed ^ mix32(bh * 0x9E3779B1u + q + 0x7F4A7C15u)); }
__device__ __forceinline__ float drop_factor(uint32_t row_key, uint32_t col, const DropParams& d) {
  return (mix32(row_key ^ (col * 0x9E3779B1u)) >> 8) >= d.thr24 ? d.inv_keep : 0.f;
}

struct AttnParams {
  DropParams drop;
  int lq, lk, heads;
  int q_coff, k_coff, v_coff;   // channel offsets of head 0 inside the q / k / v buffers
  float scale_log2;             // softmax scale * log2(e)
  const uint8_t* mask;          // [B][lk], 1 = ignore, may be null
  __nv_bfloat16* out;           // [B][lq][out_pitch], head h at channel out_coff + 32 h
  int out_pitch, out_coff;
  float* lse;                   // [B][heads][lq] natural-log sum-exp of the scaled scores, may be null
};

template <bool DROP>  // the dropout-free instantiation is the kernel as it was (the extra integer work and registers cost the p = 0 path 35 % when the
                      // choice was a run-time branch inside the softmax loop)
__global__ void __launch_bounds__(kAttThreads, 1)
attention_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                     const __grid_constant__ AttnParams p) {
  pdl_sync();
  extern __shared__ uint8_t smem_dyn[];
  __shared__ __align__(8) uint64_t s_bar[5];  // q_full, kv_full[2], kv_empty[2]
  __shared__ __align__(16) float s_bias[2][kAttTile];

  const int warp = warp_id_uniform();
  const int q0 = blockIdx.x * kAttTile, h = blockIdx.y, b = blockIdx.z;
  const uint32_t base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  const uint32_t sQ = base, sK = base + kQBytes, sV = sK + 2 * kKVBytes, sP = sV + 2 * kKVBytes;
  float* const sS = reinterpret_cast<float*>(smem_dyn + (sP + kPBytes - smem_u32(smem_dyn)));
  const uint32_t bar_q = smem_u32(&s_bar[0]), bar_kv_full = smem_u32(&s_bar[1]), bar_kv_empty = smem_u32(&s_bar[3]);
  const int ntiles = (p.lk + kAttTile - 1) / kAttTile;

  if (threadIdx.x == 0) {
    mbar_init(bar_q, 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(bar_kv_full + 8 * s, 1);
      mbar_init(bar_kv_empty + 8 * s, 1);
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (elect_one()) {
      tma_prefetch_desc(&tmQ);
      tma_prefetch_desc(&tmK);
      tma_prefetch_desc(&tmV);
      mbar_expect_tx(bar_q, kQBytes);
      tma_load_5d(sQ, &tmQ, bar_q, p.q_coff + h * kAttD, q0, 0, 0, b);
      for (int j = 0; j < ntiles; ++j) {
        const int st = j & 1;
        mbar_wait(bar_kv_empty + 8 * st, ((j >> 1) & 1) ^ 1);
        mbar_expect_tx(bar_kv_full + 8 * st, 2 * kKVBytes);
        tma_load_5d(sK + st * kKVBytes, &tmK, bar_kv_full + 8 * st, p.k_coff + h * kAttD, j * kAttTile, 0, 0, b);
        tma_load_5d(sV + st * kKVBytes, &tmV, bar_kv_full + 8 * st, p.v_coff + h * kAttD, j * kAttTile, 0, 0, b);
      }
    }
  } else if (warp < 4) {
    const int row = threadIdx.x;  // query row of this thread inside the tile
    const int tid = threadIdx.x;
    const uint32_t l64 = gmma_layout_code(64), l128 = gmma_layout_code(128);
    const float* const srow = sS + row * kSPitch;
    float m = -INFINITY, l = 0.f;
    uint32_t drop_key = 0;
    if constexpr (DROP) drop_key = drop_row_key(p.drop.seed, static_cast<uint32_t>(b * p.heads + h), static_cast<uint32_t>(q0 + row));
    float acc[kAttD];
#pragma unroll
    for (int i = 0; i < kAttD; ++i) acc[i] = 0.f;
    mbar_wait(bar_q, 0);
    for (int j = 0; j < ntiles; ++j) {
      const int st = j & 1;
      {  // additive mask of this key tile: 0 or -inf (padding keys and keys beyond lk)
        const int key = j * kAttTile + tid;
        const bool dead = key >= p.lk || (p.mask != nullptr && p.mask[static_cast<size_t>(b) * p.lk + key] != 0);
        s_bias[j & 1][tid] = dead ? -INFINITY : 0.f;
      }
      named_bar_sync(1, kAttTile);  // also: every thread is done with the previous tile's staged O_j
      const float* bias = s_bias[j & 1];
      mbar_wait(bar_kv_full + 8 * st, (j >> 1) & 1);
      // S = Q K^T, 64 query rows per wgmma, staged as fp32 rows
#pragma unroll 1
      for (int hf = 0; hf < 2; ++hf) {
        float sacc[kAttTile / 2];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kAttD / 16; ++k)
          Wgmma<kAttTile>::mma<0, 0>(sacc, gmma_desc(sQ + hf * 64 * (kAttD * 2) + k * 32, 16, 512, l64),
                                     gmma_desc(sK + st * kKVBytes + k * 32, 16, 512, l64), k != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_operand(sacc);
        wg_acc_to_smem<kAttTile>(sacc, sS + hf * 64 * kSPitch, kSPitch);
      }
      named_bar_sync(1, kAttTile);
      // pass 1: row maximum of the scaled, masked scores
      float mx = m;
#pragma unroll 1
      for (int c = 0; c < kAttTile; c += 32) {
        float r[32];
        lds_row32(srow + c, r);
#pragma unroll
        for (int i = 0; i < 32; i += 4) {  // 16-byte broadcast loads of the mask bias: per-element LDS made the LSU the busiest pipe
          const float4 bb = *reinterpret_cast<const float4*>(bias + c + i);
          mx = fmaxf(mx, fmaf(r[i], p.scale_log2, bb.x));
          mx = fmaxf(mx, fmaf(r[i + 1], p.scale_log2, bb.y));
          mx = fmaxf(mx, fmaf(r[i + 2], p.scale_log2, bb.z));
          mx = fmaxf(mx, fmaf(r[i + 3], p.scale_log2, bb.w));
        }
      }
      const float m_safe = mx == -INFINITY ? 0.f : mx;  // every key so far is masked: keep everything at zero without NaNs
      const float alpha = ex2(m - m_safe);               // m = -inf -> 0
      if (j > 0) {  // the previous tile's P V product is already folded into acc
#pragma unroll
        for (int i = 0; i < kAttD; ++i) acc[i] *= alpha;
      }
      l *= alpha;
      m = mx;
      // pass 2: probabilities -> bf16 P tile (K-major, 128-byte rows, 16-byte chunks XOR-swizzled with the row index)
      float rowsum = 0.f;
#pragma unroll 1
      for (int c = 0; c < kAttTile; c += 32) {
        float r[32];
        lds_row32(srow + c, r);
        uint32_t pk[16];
#pragma unroll
        for (int i = 0; i < 32; i += 4) {
          const float4 bb = *reinterpret_cast<const float4*>(bias + c + i);
          const float p0 = ex2(fmaf(r[i], p.scale_log2, bb.x - m_safe));
          const float p1 = ex2(fmaf(r[i + 1], p.scale_log2, bb.y - m_safe));
          const float p2 = ex2(fmaf(r[i + 2], p.scale_log2, bb.z - m_safe));
          const float p3 = ex2(fmaf(r[i + 3], p.scale_log2, bb.w - m_safe));
          rowsum += (p0 + p1) + (p2 + p3);  // the normaliser is the sum of the UNDROPPED probabilities: dropout(softmax(S)) V
          if constexpr (DROP) {
            const uint32_t col = static_cast<uint32_t>(j * kAttTile + c + i);
            pk[i >> 1] = pack_bf16x2(p0 * drop_factor(drop_key, col, p.drop), p1 * drop_factor(drop_key, col + 1, p.drop));
            pk[(i >> 1) + 1] = pack_bf16x2(p2 * drop_factor(drop_key, col + 2, p.drop), p3 * drop_factor(drop_key, col + 3, p.drop));
          } else {
            pk[i >> 1] = pack_bf16x2(p0, p1);
            pk[(i >> 1) + 1] = pack_bf16x2(p2, p3);
          }
        }
        const uint32_t blk = sP + (c >> 6) * (kAttTile * 128) + row * 128;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int chunk = ((c & 32) >> 3) + q;  // 16-byte chunk inside the 128-byte row
          const uint32_t addr = blk + (((chunk ^ (row & 7))) << 4);
          asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(pk[4 * q]), "r"(pk[4 * q + 1]), "r"(pk[4 * q + 2]), "r"(pk[4 * q + 3])
                       : "memory");
        }
      }
      l += rowsum;
      fence_proxy_async();  // generic-proxy writes of P must be visible to the tensor core (async proxy)
      named_bar_sync(1, kAttTile);
      // O_j = P V (64 query rows per wgmma), staged over the scores (no longer read) and folded into acc
      float o[2][kAttD / 2];
      wgmma_fence();
#pragma unroll
      for (int hf = 0; hf < 2; ++hf)
#pragma unroll
        for (int kk = 0; kk < kAttTile / 16; ++kk)
          Wgmma<kAttD>::mma<0, 1>(o[hf], gmma_desc(sP + (kk >> 2) * (kAttTile * 128) + hf * 64 * 128 + (kk & 3) * 32, 16, 1024, l128),
                                  gmma_desc(sV + st * kKVBytes + kk * 16 * (kAttD * 2), kKVBytes, 8 * (kAttD * 2), l64), kk != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operand(o[0]);
      wgmma_fence_operand(o[1]);
      if (threadIdx.x == 0) mbar_arrive(bar_kv_empty + 8 * st);
      wg_acc_to_smem<kAttD>(o[0], sS, kOPitch);
      wg_acc_to_smem<kAttD>(o[1], sS + 64 * kOPitch, kOPitch);
      named_bar_sync(1, kAttTile);
      {
        float ov[kAttD];
        lds_row32(sS + row * kOPitch, ov);
#pragma unroll
        for (int i = 0; i < kAttD; ++i) acc[i] += ov[i];
      }
    }
    const int qi = q0 + row;
    if (qi < p.lq) {
      const float inv = l > 0.f ? 1.f / l : 0.f;  // a fully masked row gives zeros (torch gives NaN)
      __nv_bfloat16* dst = p.out + (static_cast<size_t>(b) * p.lq + qi) * p.out_pitch + p.out_coff + h * kAttD;
#pragma unroll
      for (int i = 0; i < kAttD; i += 8) {
        uint4 u;
        u.x = pack_bf16x2(acc[i] * inv, acc[i + 1] * inv);
        u.y = pack_bf16x2(acc[i + 2] * inv, acc[i + 3] * inv);
        u.z = pack_bf16x2(acc[i + 4] * inv, acc[i + 5] * inv);
        u.w = pack_bf16x2(acc[i + 6] * inv, acc[i + 7] * inv);
        *reinterpret_cast<uint4*>(dst + i) = u;
      }
      if (p.lse != nullptr) p.lse[(static_cast<size_t>(b) * p.heads + h) * p.lq + qi] = l > 0.f ? (m + log2f(l)) * 0.6931471805599453f : -INFINITY;
    }
  }
}

// ================================================================================================================================
// Backward of the attention core.  With P = softmax(S), S = scale * Q K^T + mask, O = P V and D_i = <dO_i, O_i>:
//   dV = P^T dO,   dP = dO V^T,   dS = P o (dP - D) * scale,   dQ = dS K,   dK = dS^T Q
// P is recomputed from the saved log-sum-exp (fp32 per query row).  Two kernels, no atomics (bit-reproducible):
//   attention_bwd_kv_kernel  one CTA per (128-key tile, head, image), streams over query tiles, dK / dV accumulate in registers
//   attention_bwd_q_kernel   one CTA per (128-query tile, head, image), streams over key tiles, dQ accumulates in registers
// Operand forms: S and dP are K-major x K-major wgmmas on the TMA tiles, 64 query rows at a time, staged as fp32 rows in shared memory;
// P / dS are written by the compute threads as bf16 [query][key] tiles (128-byte rows, swizzle 128) and consumed either K-major (dQ = dS K)
// or MN-major (dV = P^T dO, dK = dS^T Q: the contraction index is the tile row); dO / Q / K enter those products as MN-major B operands
// straight from their token-major tiles.
// ================================================================================================================================
struct AttnBwdParams {
  DropParams drop;
  int lq, lk, heads;
  int q_coff, k_coff, v_coff, do_coff;
  float scale, scale_log2;
  const uint8_t* mask;
  const float* lse;    // [B][heads][lq], natural log
  const float* dsum;   // [B][heads][lq], D = <dO, O>
  __nv_bfloat16 *dq, *dk, *dv;
  int dq_pitch, dq_coff, dk_pitch, dk_coff, dv_pitch, dv_coff;
};

constexpr int kBwdStage = 64 * kSPitch * 4;  // one staged [64 query rows][128 keys] fp32 tile (S or dP)
constexpr int kBwdSmemKV = 2 * kKVBytes + 4 * kQBytes + 2 * kPBytes + 2 * kBwdStage + 1024;  // K, V | Q x2, dO x2 | P, dS | staged S, dP
constexpr int kBwdSmemQ = 2 * kQBytes + 4 * kKVBytes + kPBytes + 2 * kBwdStage + 1024;       // Q, dO | K x2, V x2 | dS | staged S, dP

// D[b][h][q] = sum_d dO[b][q][h][d] * O[b][q][h][d]
__global__ void attention_bwd_prep_kernel(const __nv_bfloat16* __restrict__ o, int o_pitch, int o_coff, const __nv_bfloat16* __restrict__ d_o, int do_pitch,
                                          int do_coff, int batch, int lq, int heads, float* __restrict__ dsum) {
  pdl_sync();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(batch) * lq * heads) return;
  const int h = static_cast<int>(i % heads);
  const long long t = i / heads;  // b * lq + q
  const int q = static_cast<int>(t % lq), b = static_cast<int>(t / lq);
  const __nv_bfloat16* po = o + t * o_pitch + o_coff + h * kAttD;
  const __nv_bfloat16* pd = d_o + t * do_pitch + do_coff + h * kAttD;
  float acc = 0.f;
#pragma unroll
  for (int c = 0; c < kAttD; c += 8) {
    const uint4 a = *reinterpret_cast<const uint4*>(po + c), g = *reinterpret_cast<const uint4*>(pd + c);
    acc += bf16_lo(a.x) * bf16_lo(g.x) + bf16_hi(a.x) * bf16_hi(g.x) + bf16_lo(a.y) * bf16_lo(g.y) + bf16_hi(a.y) * bf16_hi(g.y) +
           bf16_lo(a.z) * bf16_lo(g.z) + bf16_hi(a.z) * bf16_hi(g.z) + bf16_lo(a.w) * bf16_lo(g.w) + bf16_hi(a.w) * bf16_hi(g.w);
  }
  dsum[(static_cast<size_t>(b) * heads + h) * lq + q] = acc;
}

// one 32-column chunk of P and dS for one query row: reads S and dP from their staged rows, writes both bf16 tiles ([query][key], swizzle 128)
// With dropout D (0 or 1/(1-p) per element): O = (D o P) V, so the tile written for dV = (D o P)^T dO is the dropped one, dP = D o (dO V^T) and
// dS = P o (dP - <dO, O>) -- the row term <dO, O> (attention_bwd_prep_kernel) already contains D through O.
template <bool DROP>
__device__ __forceinline__ void bwd_chunk(const float* srow, const float* dprow, int c, int row, const float* bias, float lse_log2, float dsum,
                                          float scale, float scale_log2, uint32_t sP, uint32_t sDS, bool write_p, const DropParams& drop, uint32_t drop_key,
                                          int key0) {
  float r[32], g[32];
  lds_row32(srow + c, r);
  lds_row32(dprow + c, g);
  uint32_t pk[16], dk[16];
#pragma unroll
  for (int i = 0; i < 32; i += 4) {
    const float4 bb = *reinterpret_cast<const float4*>(bias + c + i);
    const float p0 = ex2(fmaf(r[i], scale_log2, bb.x - lse_log2));
    const float p1 = ex2(fmaf(r[i + 1], scale_log2, bb.y - lse_log2));
    const float p2 = ex2(fmaf(r[i + 2], scale_log2, bb.z - lse_log2));
    const float p3 = ex2(fmaf(r[i + 3], scale_log2, bb.w - lse_log2));
    float f0 = 1.f, f1 = 1.f, f2 = 1.f, f3 = 1.f;
    if constexpr (DROP) {
      const uint32_t col = static_cast<uint32_t>(key0 + c + i);
      f0 = drop_factor(drop_key, col, drop); f1 = drop_factor(drop_key, col + 1, drop);
      f2 = drop_factor(drop_key, col + 2, drop); f3 = drop_factor(drop_key, col + 3, drop);
    }
    pk[i >> 1] = pack_bf16x2(p0 * f0, p1 * f1);
    pk[(i >> 1) + 1] = pack_bf16x2(p2 * f2, p3 * f3);
    dk[i >> 1] = pack_bf16x2(p0 * (g[i] * f0 - dsum) * scale, p1 * (g[i + 1] * f1 - dsum) * scale);
    dk[(i >> 1) + 1] = pack_bf16x2(p2 * (g[i + 2] * f2 - dsum) * scale, p3 * (g[i + 3] * f3 - dsum) * scale);
  }
  const uint32_t off = (c >> 6) * (kAttTile * 128) + row * 128;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int chunk = ((c & 32) >> 3) + q;
    const uint32_t sw = off + (((chunk ^ (row & 7))) << 4);
    if (write_p)
      asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(sP + sw), "r"(pk[4 * q]), "r"(pk[4 * q + 1]), "r"(pk[4 * q + 2]), "r"(pk[4 * q + 3]) : "memory");
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(sDS + sw), "r"(dk[4 * q]), "r"(dk[4 * q + 1]), "r"(dk[4 * q + 2]), "r"(dk[4 * q + 3]) : "memory");
  }
}

__device__ __forceinline__ void store_row32(__nv_bfloat16* dst, const float (&o)[32]) {
#pragma unroll
  for (int i = 0; i < kAttD; i += 8) {
    uint4 u;
    u.x = pack_bf16x2(o[i], o[i + 1]);
    u.y = pack_bf16x2(o[i + 2], o[i + 3]);
    u.z = pack_bf16x2(o[i + 4], o[i + 5]);
    u.w = pack_bf16x2(o[i + 6], o[i + 7]);
    *reinterpret_cast<uint4*>(dst + i) = u;
  }
}

// S and dP of query rows [64 hf, 64 hf + 64) of the tiles at sQ / sDO against the key tiles at sK / sV, staged as fp32 rows
__device__ __forceinline__ void bwd_scores_half(uint32_t sQ, uint32_t sDO, uint32_t sK, uint32_t sV, int hf, float* stS, float* stDP) {
  const uint32_t l64 = gmma_layout_code(64);
  float acc[kAttTile / 2];
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < kAttD / 16; ++k)
    Wgmma<kAttTile>::mma<0, 0>(acc, gmma_desc(sQ + hf * 64 * (kAttD * 2) + k * 32, 16, 512, l64), gmma_desc(sK + k * 32, 16, 512, l64), k != 0 ? 1u : 0u);
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_operand(acc);
  wg_acc_to_smem<kAttTile>(acc, stS, kSPitch);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < kAttD / 16; ++k)
    Wgmma<kAttTile>::mma<0, 0>(acc, gmma_desc(sDO + hf * 64 * (kAttD * 2) + k * 32, 16, 512, l64), gmma_desc(sV + k * 32, 16, 512, l64), k != 0 ? 1u : 0u);
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_operand(acc);
  wg_acc_to_smem<kAttTile>(acc, stDP, kSPitch);
}

// a [128][32] accumulator held as two 64-row warpgroup fragments -> row `row` of it in `o` (through the staging area at st)
__device__ __forceinline__ void acc_row32(const float (&a)[2][kAttD / 2], float* st, int row, float (&o)[32]) {
  named_bar_sync(1, kAttTile);  // the staging area is free
  wg_acc_to_smem<kAttD>(a[0], st, kOPitch);
  wg_acc_to_smem<kAttD>(a[1], st + 64 * kOPitch, kOPitch);
  named_bar_sync(1, kAttTile);
  lds_row32(st + row * kOPitch, o);
}

template <bool DROP>
__global__ void __launch_bounds__(kAttThreads, 1)
attention_bwd_kv_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                        const __grid_constant__ CUtensorMap tmDO, const __grid_constant__ AttnBwdParams p) {
  pdl_sync();
  extern __shared__ uint8_t smem_dyn[];
  __shared__ __align__(8) uint64_t s_bar[5];  // kv_full, qdo_full[2], qdo_empty[2]
  __shared__ __align__(16) float s_bias[kAttTile];

  const int warp = warp_id_uniform();
  const int k0 = blockIdx.x * kAttTile, h = blockIdx.y, b = blockIdx.z;
  const uint32_t base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  const uint32_t sK = base, sV = sK + kKVBytes, sQ = sV + kKVBytes, sDO = sQ + 2 * kQBytes, sP = sDO + 2 * kQBytes, sDS = sP + kPBytes;
  float* const stS = reinterpret_cast<float*>(smem_dyn + (sDS + kPBytes - smem_u32(smem_dyn)));
  float* const stDP = stS + 64 * kSPitch;
  const uint32_t bar_kv = smem_u32(&s_bar[0]), bar_full = smem_u32(&s_bar[1]), bar_empty = smem_u32(&s_bar[3]);
  const int ntiles = (p.lq + kAttTile - 1) / kAttTile;

  if (threadIdx.x == 0) {
    mbar_init(bar_kv, 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, 1);
    }
    mbar_fence_init();
  }
  if (threadIdx.x < kAttTile) {  // additive mask of this CTA's key tile
    const int key = k0 + threadIdx.x;
    const bool dead = key >= p.lk || (p.mask != nullptr && p.mask[static_cast<size_t>(b) * p.lk + key] != 0);
    s_bias[threadIdx.x] = dead ? -INFINITY : 0.f;
  }
  __syncthreads();

  if (warp == 4) {
    if (elect_one()) {
      mbar_expect_tx(bar_kv, 2 * kKVBytes);
      tma_load_5d(sK, &tmK, bar_kv, p.k_coff + h * kAttD, k0, 0, 0, b);
      tma_load_5d(sV, &tmV, bar_kv, p.v_coff + h * kAttD, k0, 0, 0, b);
      for (int i = 0; i < ntiles; ++i) {
        const int st = i & 1;
        mbar_wait(bar_empty + 8 * st, ((i >> 1) & 1) ^ 1);
        mbar_expect_tx(bar_full + 8 * st, 2 * kQBytes);
        tma_load_5d(sQ + st * kQBytes, &tmQ, bar_full + 8 * st, p.q_coff + h * kAttD, i * kAttTile, 0, 0, b);
        tma_load_5d(sDO + st * kQBytes, &tmDO, bar_full + 8 * st, p.do_coff + h * kAttD, i * kAttTile, 0, 0, b);
      }
    }
  } else if (warp < 4) {
    const int t = threadIdx.x;
    const int rl = t & 63, cbeg = (t >> 6) * 64;  // staged row of this thread and the 64 columns of it that it converts
    const uint32_t l64 = gmma_layout_code(64), l128 = gmma_layout_code(128);
    float dv[2][kAttD / 2], dk[2][kAttD / 2];  // [key half]: keys [64 g, 64 g + 64) of the tile
#pragma unroll
    for (int g = 0; g < 2; ++g)
#pragma unroll
      for (int i = 0; i < kAttD / 2; ++i) { dv[g][i] = 0.f; dk[g][i] = 0.f; }
    mbar_wait(bar_kv, 0);
    for (int i = 0; i < ntiles; ++i) {
      const int st = i & 1;
      mbar_wait(bar_full + 8 * st, (i >> 1) & 1);
#pragma unroll 1
      for (int hf = 0; hf < 2; ++hf) {
        const int row = 64 * hf + rl;
        const int qi = i * kAttTile + row;
        const size_t stat = (static_cast<size_t>(b) * p.heads + h) * p.lq + qi;
        float lse_log2 = qi < p.lq ? p.lse[stat] * 1.4426950408889634f : INFINITY;  // rows beyond lq: p = 0
        if (lse_log2 == -INFINITY) lse_log2 = INFINITY;                                 // fully masked query: zero gradients instead of NaN
        const float dsum = qi < p.lq ? p.dsum[stat] : 0.f;
        uint32_t drop_key = 0;
        if constexpr (DROP) drop_key = drop_row_key(p.drop.seed, static_cast<uint32_t>(b * p.heads + h), static_cast<uint32_t>(qi));
        bwd_scores_half(sQ + st * kQBytes, sDO + st * kQBytes, sK, sV, hf, stS, stDP);
        named_bar_sync(1, kAttTile);
#pragma unroll 1
        for (int c = cbeg; c < cbeg + 64; c += 32)
          bwd_chunk<DROP>(stS + rl * kSPitch, stDP + rl * kSPitch, c, row, s_bias, lse_log2, dsum, p.scale, p.scale_log2, sP, sDS, true, p.drop, drop_key, k0);
        fence_proxy_async();          // P / dS writes -> visible to the tensor core
        named_bar_sync(1, kAttTile);  // and the staged tiles are free again
      }
      wgmma_fence();
#pragma unroll
      for (int g = 0; g < 2; ++g)
#pragma unroll
        for (int kk = 0; kk < kAttTile / 16; ++kk) {  // contraction over the 128 query rows of the tile, 16 at a time
          const uint64_t a_p = gmma_desc(sP + g * (kAttTile * 128) + kk * 16 * 128, kAttTile * 128, 8 * 128, l128);
          const uint64_t a_ds = gmma_desc(sDS + g * (kAttTile * 128) + kk * 16 * 128, kAttTile * 128, 8 * 128, l128);
          const uint64_t b_do = gmma_desc(sDO + st * kQBytes + kk * 16 * (kAttD * 2), kQBytes, 8 * (kAttD * 2), l64);
          const uint64_t b_q = gmma_desc(sQ + st * kQBytes + kk * 16 * (kAttD * 2), kQBytes, 8 * (kAttD * 2), l64);
          Wgmma<kAttD>::mma<1, 1>(dv[g], a_p, b_do, 1u);
          Wgmma<kAttD>::mma<1, 1>(dk[g], a_ds, b_q, 1u);
        }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operand(dv[0]); wgmma_fence_operand(dv[1]);
      wgmma_fence_operand(dk[0]); wgmma_fence_operand(dk[1]);
      if (t == 0) mbar_arrive(bar_empty + 8 * st);
    }
    const int key = k0 + t;  // accumulator row = key index
    float o[32];
    acc_row32(dv, stS, t, o);
    if (key < p.lk) store_row32(p.dv + (static_cast<size_t>(b) * p.lk + key) * p.dv_pitch + p.dv_coff + h * kAttD, o);
    acc_row32(dk, stS, t, o);
    if (key < p.lk) store_row32(p.dk + (static_cast<size_t>(b) * p.lk + key) * p.dk_pitch + p.dk_coff + h * kAttD, o);
  }
}

template <bool DROP>
__global__ void __launch_bounds__(kAttThreads, 1)
attention_bwd_q_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                       const __grid_constant__ CUtensorMap tmDO, const __grid_constant__ AttnBwdParams p) {
  pdl_sync();
  extern __shared__ uint8_t smem_dyn[];
  __shared__ __align__(8) uint64_t s_bar[5];  // qdo_full, kv_full[2], kv_empty[2]
  __shared__ __align__(16) float s_bias[2][kAttTile];

  const int warp = warp_id_uniform();
  const int q0 = blockIdx.x * kAttTile, h = blockIdx.y, b = blockIdx.z;
  const uint32_t base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  const uint32_t sQ = base, sDO = sQ + kQBytes, sK = sDO + kQBytes, sV = sK + 2 * kKVBytes, sDS = sV + 2 * kKVBytes;
  float* const stS = reinterpret_cast<float*>(smem_dyn + (sDS + kPBytes - smem_u32(smem_dyn)));
  float* const stDP = stS + 64 * kSPitch;
  const uint32_t bar_q = smem_u32(&s_bar[0]), bar_full = smem_u32(&s_bar[1]), bar_empty = smem_u32(&s_bar[3]);
  const int ntiles = (p.lk + kAttTile - 1) / kAttTile;

  if (threadIdx.x == 0) {
    mbar_init(bar_q, 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, 1);
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (elect_one()) {
      mbar_expect_tx(bar_q, 2 * kQBytes);
      tma_load_5d(sQ, &tmQ, bar_q, p.q_coff + h * kAttD, q0, 0, 0, b);
      tma_load_5d(sDO, &tmDO, bar_q, p.do_coff + h * kAttD, q0, 0, 0, b);
      for (int j = 0; j < ntiles; ++j) {
        const int st = j & 1;
        mbar_wait(bar_empty + 8 * st, ((j >> 1) & 1) ^ 1);
        mbar_expect_tx(bar_full + 8 * st, 2 * kKVBytes);
        tma_load_5d(sK + st * kKVBytes, &tmK, bar_full + 8 * st, p.k_coff + h * kAttD, j * kAttTile, 0, 0, b);
        tma_load_5d(sV + st * kKVBytes, &tmV, bar_full + 8 * st, p.v_coff + h * kAttD, j * kAttTile, 0, 0, b);
      }
    }
  } else if (warp < 4) {
    const int t = threadIdx.x, tid = t;
    const int rl = t & 63, cbeg = (t >> 6) * 64;  // staged row of this thread and the 64 columns of it that it converts
    const uint32_t l64 = gmma_layout_code(64), l128 = gmma_layout_code(128);
    // per-row terms of the two query rows this thread converts (rows rl and 64 + rl of the tile)
    float lse_log2[2], dsum[2];
    uint32_t drop_key[2] = {0u, 0u};
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const int qi = q0 + 64 * hf + rl;
      const size_t stat = (static_cast<size_t>(b) * p.heads + h) * p.lq + qi;
      lse_log2[hf] = qi < p.lq ? p.lse[stat] * 1.4426950408889634f : INFINITY;
      if (lse_log2[hf] == -INFINITY) lse_log2[hf] = INFINITY;
      dsum[hf] = qi < p.lq ? p.dsum[stat] : 0.f;
      if constexpr (DROP) drop_key[hf] = drop_row_key(p.drop.seed, static_cast<uint32_t>(b * p.heads + h), static_cast<uint32_t>(qi));
    }
    float dq[2][kAttD / 2];  // [query half]
#pragma unroll
    for (int g = 0; g < 2; ++g)
#pragma unroll
      for (int i = 0; i < kAttD / 2; ++i) dq[g][i] = 0.f;
    mbar_wait(bar_q, 0);
    for (int j = 0; j < ntiles; ++j) {
      const int st = j & 1;
      {
        const int key = j * kAttTile + tid;
        const bool dead = key >= p.lk || (p.mask != nullptr && p.mask[static_cast<size_t>(b) * p.lk + key] != 0);
        s_bias[j & 1][tid] = dead ? -INFINITY : 0.f;
      }
      mbar_wait(bar_full + 8 * st, (j >> 1) & 1);
#pragma unroll 1
      for (int hf = 0; hf < 2; ++hf) {
        bwd_scores_half(sQ, sDO, sK + st * kKVBytes, sV + st * kKVBytes, hf, stS, stDP);
        named_bar_sync(1, kAttTile);  // staged tiles (and, on the first half, the mask bias) complete
#pragma unroll 1
        for (int c = cbeg; c < cbeg + 64; c += 32)
          bwd_chunk<DROP>(stS + rl * kSPitch, stDP + rl * kSPitch, c, 64 * hf + rl, s_bias[j & 1], lse_log2[hf], dsum[hf], p.scale, p.scale_log2, sDS, sDS,
                          false, p.drop, drop_key[hf], j * kAttTile);
        fence_proxy_async();
        named_bar_sync(1, kAttTile);
      }
      wgmma_fence();
#pragma unroll
      for (int g = 0; g < 2; ++g)
#pragma unroll
        for (int kk = 0; kk < kAttTile / 16; ++kk) {
          const uint64_t da = gmma_desc(sDS + (kk >> 2) * (kAttTile * 128) + g * 64 * 128 + (kk & 3) * 32, 16, 1024, l128);
          const uint64_t db = gmma_desc(sK + st * kKVBytes + kk * 16 * (kAttD * 2), kKVBytes, 8 * (kAttD * 2), l64);
          Wgmma<kAttD>::mma<0, 1>(dq[g], da, db, 1u);  // A = dS (K-major), B = K tile (MN-major): as P V in the forward kernel
        }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_operand(dq[0]);
      wgmma_fence_operand(dq[1]);
      if (t == 0) mbar_arrive(bar_empty + 8 * st);
    }
    const int qi = q0 + t;
    float o[32];
    acc_row32(dq, stS, t, o);
    if (qi < p.lq) store_row32(p.dq + (static_cast<size_t>(b) * p.lq + qi) * p.dq_pitch + p.dq_coff + h * kAttD, o);
  }
}

// a token sequence: a [B][1][L][E] view with E = heads x 32
int check_tokens(const yb200_act* a, const char* name) {
  if (const int rc = check_act(a, name)) return rc;
  YB_REQUIRE(a->h == 1 && a->c % kAttD == 0, YB200_ERR_INVALID, "%s: expected a [B][1][L][heads x 32] view (got %dx%dx%dx%d)", name, a->n, a->h,
             a->w, a->c);
  return 0;
}

}  // namespace

static int make_drop(float p_drop, uint32_t seed, DropParams* d, const char* who) {
  YB_REQUIRE(p_drop >= 0.f && p_drop < 1.f, YB200_ERR_INVALID, "%s: dropout probability %g outside [0, 1)", who, p_drop);
  d->seed = seed;
  d->thr24 = static_cast<uint32_t>(static_cast<double>(p_drop) * 16777216.0);
  d->inv_keep = 1.f / (1.f - p_drop);
  return 0;
}
static int attention_fwd_impl(const yb200_act* q, const yb200_act* k, const yb200_act* v, const uint8_t* key_padding_mask, float scale,
                              const yb200_act* out, float* lse, float p_drop, uint32_t seed, void* stream);
extern "C" int yb200_attention_fwd(const yb200_act* q, const yb200_act* k, const yb200_act* v, const uint8_t* key_padding_mask, float scale,
                                   const yb200_act* out, float* lse, void* stream) {
  return attention_fwd_impl(q, k, v, key_padding_mask, scale, out, lse, 0.f, 0u, stream);
}
extern "C" int yb200_attention_fwd_dropout(const yb200_act* q, const yb200_act* k, const yb200_act* v, const uint8_t* key_padding_mask, float scale,
                                           const yb200_act* out, float* lse, float p_drop, uint32_t seed, void* stream) {
  return attention_fwd_impl(q, k, v, key_padding_mask, scale, out, lse, p_drop, seed, stream);
}
static int attention_fwd_impl(const yb200_act* q, const yb200_act* k, const yb200_act* v, const uint8_t* key_padding_mask, float scale,
                              const yb200_act* out, float* lse, float p_drop, uint32_t seed, void* stream) {
  int rc;
  if ((rc = check_tokens(q, "attention_fwd q"))) return rc;
  if ((rc = check_tokens(k, "attention_fwd k"))) return rc;
  if ((rc = check_tokens(v, "attention_fwd v"))) return rc;
  if ((rc = check_tokens(out, "attention_fwd out"))) return rc;
  YB_REQUIRE(k->n == q->n && v->n == q->n && out->n == q->n && k->w == v->w && out->w == q->w && k->c == q->c && v->c == q->c && out->c == q->c,
             YB200_ERR_INVALID, "attention_fwd: shapes q %dx%dx%d k %dx%dx%d v %dx%dx%d out %dx%dx%d", q->n, q->w, q->c, k->n, k->w, k->c, v->n, v->w, v->c,
             out->n, out->w, out->c);
  CUtensorMap tmQ, tmK, tmV;
  if ((rc = make_act_map(&tmQ, *q, false, kAttD, kAttTile, 1, 1))) return rc;
  if ((rc = make_act_map(&tmK, *k, false, kAttD, kAttTile, 1, 1))) return rc;
  if ((rc = make_act_map(&tmV, *v, false, kAttD, kAttTile, 1, 1))) return rc;
  AttnParams p;
  if ((rc = make_drop(p_drop, seed, &p.drop, "attention_fwd"))) return rc;
  p.lq = q->w; p.lk = k->w; p.heads = q->c / kAttD;
  p.q_coff = q->c_off; p.k_coff = k->c_off; p.v_coff = v->c_off;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.mask = key_padding_mask;
  p.out = static_cast<__nv_bfloat16*>(out->ptr);
  p.out_pitch = out->c_pitch; p.out_coff = out->c_off;
  p.lse = lse;
  static PerDevice<int> smem_limit(0);
  YB_CHECK_CUDA(raise_smem_limit(smem_limit, kAttSmem, attention_fwd_kernel<false>, attention_fwd_kernel<true>));
  dim3 grid(ceil_div(p.lq, kAttTile), p.heads, q->n);
  if (p.drop.thr24 != 0)
    launch_k(attention_fwd_kernel<true>, grid, kAttThreads, kAttSmem, as_stream(stream), tmQ, tmK, tmV, p);
  else
    launch_k(attention_fwd_kernel<false>, grid, kAttThreads, kAttSmem, as_stream(stream), tmQ, tmK, tmV, p);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int64_t yb200_attention_bwd_workspace(const yb200_act* q) {
  if (!q || q->n <= 0 || q->w <= 0 || q->c <= 0 || q->c % kAttD != 0) return YB200_ERR_INVALID;
  return 4LL * q->n * (q->c / kAttD) * q->w;
}

static int attention_bwd_impl(const yb200_act* q, const yb200_act* k, const yb200_act* v, const yb200_act* out, const yb200_act* dout,
                              const uint8_t* key_padding_mask, float scale, const float* lse, const yb200_act* dq, const yb200_act* dk,
                              const yb200_act* dv, void* workspace, float p_drop, uint32_t seed, void* stream);
extern "C" int yb200_attention_bwd(const yb200_act* q, const yb200_act* k, const yb200_act* v, const yb200_act* out, const yb200_act* dout,
                                   const uint8_t* key_padding_mask, float scale, const float* lse, const yb200_act* dq, const yb200_act* dk,
                                   const yb200_act* dv, void* workspace, void* stream) {
  return attention_bwd_impl(q, k, v, out, dout, key_padding_mask, scale, lse, dq, dk, dv, workspace, 0.f, 0u, stream);
}
extern "C" int yb200_attention_bwd_dropout(const yb200_act* q, const yb200_act* k, const yb200_act* v, const yb200_act* out, const yb200_act* dout,
                                           const uint8_t* key_padding_mask, float scale, const float* lse, const yb200_act* dq, const yb200_act* dk,
                                           const yb200_act* dv, void* workspace, float p_drop, uint32_t seed, void* stream) {
  return attention_bwd_impl(q, k, v, out, dout, key_padding_mask, scale, lse, dq, dk, dv, workspace, p_drop, seed, stream);
}
static int attention_bwd_impl(const yb200_act* q, const yb200_act* k, const yb200_act* v, const yb200_act* out, const yb200_act* dout,
                              const uint8_t* key_padding_mask, float scale, const float* lse, const yb200_act* dq, const yb200_act* dk,
                              const yb200_act* dv, void* workspace, float p_drop, uint32_t seed, void* stream) {
  int rc;
  const yb200_act* all[8] = {q, k, v, out, dout, dq, dk, dv};
  const char* names[8] = {"attention_bwd q", "attention_bwd k", "attention_bwd v", "attention_bwd out", "attention_bwd dout", "attention_bwd dq", "attention_bwd dk",
                          "attention_bwd dv"};
  for (int i = 0; i < 8; ++i)
    if ((rc = check_tokens(all[i], names[i]))) return rc;
  YB_REQUIRE(lse && workspace, YB200_ERR_INVALID, "attention_bwd: null lse / workspace");
  const yb200_act* qlike[3] = {out, dout, dq};
  for (const yb200_act* t : qlike) YB_REQUIRE(t->n == q->n && t->w == q->w && t->c == q->c, YB200_ERR_INVALID, "attention_bwd: query-side shapes differ");
  const yb200_act* klike[4] = {k, v, dk, dv};
  for (const yb200_act* t : klike) YB_REQUIRE(t->n == q->n && t->w == k->w && t->c == q->c, YB200_ERR_INVALID, "attention_bwd: key-side shapes differ");
  CUtensorMap tmQ, tmK, tmV, tmDO;
  if ((rc = make_act_map(&tmQ, *q, false, kAttD, kAttTile, 1, 1))) return rc;
  if ((rc = make_act_map(&tmK, *k, false, kAttD, kAttTile, 1, 1))) return rc;
  if ((rc = make_act_map(&tmV, *v, false, kAttD, kAttTile, 1, 1))) return rc;
  if ((rc = make_act_map(&tmDO, *dout, false, kAttD, kAttTile, 1, 1))) return rc;
  AttnBwdParams p;
  if ((rc = make_drop(p_drop, seed, &p.drop, "attention_bwd"))) return rc;
  p.lq = q->w; p.lk = k->w; p.heads = q->c / kAttD;
  p.q_coff = q->c_off; p.k_coff = k->c_off; p.v_coff = v->c_off; p.do_coff = dout->c_off;
  p.scale = scale; p.scale_log2 = scale * 1.4426950408889634f;
  p.mask = key_padding_mask;
  p.lse = lse;
  p.dsum = static_cast<const float*>(workspace);
  p.dq = static_cast<__nv_bfloat16*>(dq->ptr); p.dq_pitch = dq->c_pitch; p.dq_coff = dq->c_off;
  p.dk = static_cast<__nv_bfloat16*>(dk->ptr); p.dk_pitch = dk->c_pitch; p.dk_coff = dk->c_off;
  p.dv = static_cast<__nv_bfloat16*>(dv->ptr); p.dv_pitch = dv->c_pitch; p.dv_coff = dv->c_off;
  static PerDevice<int> kv_limit(0), q_limit(0);
  YB_CHECK_CUDA(raise_smem_limit(kv_limit, kBwdSmemKV, attention_bwd_kv_kernel<false>, attention_bwd_kv_kernel<true>));
  YB_CHECK_CUDA(raise_smem_limit(q_limit, kBwdSmemQ, attention_bwd_q_kernel<false>, attention_bwd_q_kernel<true>));
  cudaStream_t st = as_stream(stream);
  const long long rows = 1LL * q->n * q->w * p.heads;
  launch_k(attention_bwd_prep_kernel, static_cast<int>((rows + 255) / 256), 256, 0, st, static_cast<const __nv_bfloat16*>(out->ptr), out->c_pitch, out->c_off,
                                                                                  static_cast<const __nv_bfloat16*>(dout->ptr), dout->c_pitch, dout->c_off, q->n,
                                                                                  q->w, p.heads, static_cast<float*>(workspace));
  if (p.drop.thr24 != 0) {
    launch_k(attention_bwd_kv_kernel<true>, dim3(ceil_div(p.lk, kAttTile), p.heads, q->n), kAttThreads, kBwdSmemKV, st, tmQ, tmK, tmV, tmDO, p);
    launch_k(attention_bwd_q_kernel<true>, dim3(ceil_div(p.lq, kAttTile), p.heads, q->n), kAttThreads, kBwdSmemQ, st, tmQ, tmK, tmV, tmDO, p);
  } else {
    launch_k(attention_bwd_kv_kernel<false>, dim3(ceil_div(p.lk, kAttTile), p.heads, q->n), kAttThreads, kBwdSmemKV, st, tmQ, tmK, tmV, tmDO, p);
    launch_k(attention_bwd_q_kernel<false>, dim3(ceil_div(p.lq, kAttTile), p.heads, q->n), kAttThreads, kBwdSmemQ, st, tmQ, tmK, tmV, tmDO, p);
  }
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}


// ------------------------------------------------------------------------------------------------
// nn.Dropout on a [B][1][L][C] bf16 activation (dropout / dropout1 / dropout2 / dropout3 of the transformer layers, detr_backbone.py:147-152, 207-214):
//   out = residual + x * keep(seed, element) / (1 - p) * extra_scale        (residual may be null; extra_scale = 1 except in the FFN backward)
// with the same counter-based hash as the attention kernels; `element` is the logical index ((b * L + l) * C + c), so views with different channel
// pitches share a mask and the backward pass (the same call on the gradient, same seed) regenerates it.
// ------------------------------------------------------------------------------------------------
namespace {
__global__ void dropout_bf16_kernel(const __nv_bfloat16* __restrict__ x, int x_pitch, const __nv_bfloat16* __restrict__ res, int res_pitch,
                                    __nv_bfloat16* __restrict__ out, int out_pitch, long long rows, int c, DropParams d, float extra_scale) {
  pdl_sync();
  const int cv = c / 8;
  const long long total = rows * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cv;
    const int c8 = static_cast<int>(i - r * cv) * 8;
    const uint4 xv = *reinterpret_cast<const uint4*>(x + r * x_pitch + c8);
    uint4 rv = make_uint4(0u, 0u, 0u, 0u);
    if (res) rv = *reinterpret_cast<const uint4*>(res + r * res_pitch + c8);
    const uint32_t xs[4] = {xv.x, xv.y, xv.z, xv.w}, rs[4] = {rv.x, rv.y, rv.z, rv.w};
    uint32_t o[4];
    const uint32_t e0 = static_cast<uint32_t>(r * c + c8);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float f0 = (mix32(d.seed ^ ((e0 + 2 * k) * 0x9E3779B1u)) >> 8) >= d.thr24 ? d.inv_keep * extra_scale : 0.f;
      const float f1 = (mix32(d.seed ^ ((e0 + 2 * k + 1) * 0x9E3779B1u)) >> 8) >= d.thr24 ? d.inv_keep * extra_scale : 0.f;
      o[k] = pack_bf16x2(fmaf(bf16_lo(xs[k]), f0, bf16_lo(rs[k])), fmaf(bf16_hi(xs[k]), f1, bf16_hi(rs[k])));
    }
    *reinterpret_cast<uint4*>(out + r * out_pitch + c8) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}
}  // namespace

extern "C" int yb200_dropout(const yb200_act* x, const yb200_act* residual, const yb200_act* out, float p_drop, uint32_t seed, float extra_scale,
                             void* stream) {
  int rc;
  if ((rc = check_tokens(x, "dropout x"))) return rc;
  if ((rc = check_tokens(out, "dropout out"))) return rc;
  if (residual && (rc = check_tokens(residual, "dropout residual"))) return rc;
  YB_REQUIRE(out->n == x->n && out->w == x->w && out->c == x->c && (!residual || (residual->n == x->n && residual->w == x->w && residual->c == x->c)),
             YB200_ERR_INVALID, "dropout: shapes differ");
  YB_REQUIRE(1LL * x->n * x->w * x->c < (1LL << 32), YB200_ERR_UNSUPPORTED, "dropout: more than 2^32 elements");
  DropParams d;
  if ((rc = make_drop(p_drop, seed, &d, "dropout"))) return rc;
  const long long rows = 1LL * x->n * x->w;
  const long long total = rows * (x->c / 8);
  const int blocks = static_cast<int>(std::min<long long>((total + 255) / 256, 16LL * sm_count()));
  launch_k(dropout_bf16_kernel, blocks, 256, 0, as_stream(stream), static_cast<const __nv_bfloat16*>(x->ptr) + x->c_off, x->c_pitch,
           residual ? static_cast<const __nv_bfloat16*>(residual->ptr) + residual->c_off : nullptr, residual ? residual->c_pitch : 0,
           static_cast<__nv_bfloat16*>(out->ptr) + out->c_off, out->c_pitch, rows, x->c, d, extra_scale);
  YB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
