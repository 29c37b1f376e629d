// Causal GQA flash attention for sm_90a on wgmma tensor cores (SURVEY.md K3 / M7).
//
// Input is the fused, already-roped projection qkv [B*S, (H+2*KVH)*HD] (bf16); 2-D TMA maps with {64 x 128|64}-element
// boxes serve Q, K and V.  Every GEMM is a wgmma with fp32 accumulators in registers; the softmax probabilities P and
// the score gradients dS go back into the tensor core as register A operands (the wgmma accumulator layout of 16
// columns is exactly the m64k16 A-fragment layout), so they never touch shared memory.
//
//  forward   CTA = (q tile of 128, head, batch), two warpgroups of 64 q rows.  Per kv tile of 128:
//            S = Q K^T, online softmax in registers (rows are shared by 4 lanes), O += P V with V consumed as an
//            MN-major operand.  K/V are double-buffered; thread 0 issues the TMA loads.
//  backward  two kernels:  dK/dV: CTA = (kv tile 128, kv head, batch), streams (Q_i, dO_i) tiles of 64 rows of every
//            head of the GQA group, computes S^T = K Q^T and dP^T = V dO^T, accumulates dV += P^T dO and dK += dS^T Q
//            in registers (GQA group summed in the accumulator, no atomics);  dQ: CTA = (q tile 128, head, batch),
//            streams (K_j, V_j) tiles of 64, dQ += dS K.  The score GEMMs are recomputed in both kernels in exchange
//            for a deterministic, atomic-free dQ.
#include "common.cuh"
#include "tensormap.h"
#include "wgmma.cuh"

namespace b200 {

constexpr int ATT_THREADS = 256;
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;

// D += A * B with N = HD (64 or 128), A from registers
template <int HD, int TB>
B200_DEVINL void mma_rs_hd(float (&d)[HD / 2], const uint32_t (&a)[4], uint64_t bdesc) {
  if constexpr (HD == 128) wgmma_bf16_rs_n128<TB>(d, a, bdesc, 1);
  else wgmma_bf16_rs_n64<TB>(d, a, bdesc, 1);
}

// accumulator columns [16 kk, 16 kk + 16) of a thread -> m64k16 A fragment
template <int NREG>
B200_DEVINL void acc_to_frag(const float (&v)[NREG], int kk, uint32_t (&a)[4]) {
  a[0] = pack_bf16x2(v[8 * kk + 0], v[8 * kk + 1]);
  a[1] = pack_bf16x2(v[8 * kk + 2], v[8 * kk + 3]);
  a[2] = pack_bf16x2(v[8 * kk + 4], v[8 * kk + 5]);
  a[3] = pack_bf16x2(v[8 * kk + 6], v[8 * kk + 7]);
}

B200_DEVINL float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
B200_DEVINL float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// ============================================================================================ forward
template <int HD>
struct FwdCfg {
  static constexpr int NCH = HD / 64;
  static constexpr int TILE_BYTES = 128 * HD * 2;   // 128 rows, NCH chunks of 64 columns (16 KiB each)
  static constexpr int SMEM = TILE_BYTES * (1 + 2 + 2) + 1024 + 256;
};

template <int HD>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tm, __nv_bfloat16* __restrict__ o, float* __restrict__ lse,
                int S, int H, int KVH, float scale_log2, int n_qt) {
  using C = FwdCfg<HD>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + C::TILE_BYTES;          // [2 stages]
  uint8_t* sV = sK + 2 * C::TILE_BYTES;      // [2 stages]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + 2 * C::TILE_BYTES);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;              // [2]

  const int wg = threadIdx.x >> 7, w4 = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int qt = n_qt - 1 - blockIdx.x;      // heavy tiles first
  const int h = blockIdx.y, b = blockIdx.z;
  const int kvh = h / (H / KVH);
  const int row0 = b * S + qt * 128;
  const int n_kv = min(qt + 1, (S + 127) / 128);

  auto load_kv = [&](int j) {
    const int st = j & 1;
    const int krow = b * S + j * 128;
    mbar_arrive_expect_tx(&kv_full[st], 2 * C::TILE_BYTES);
    for (int c = 0; c < C::NCH; ++c) {
      tma_load_2d(sK + st * C::TILE_BYTES + c * 16384, &tm, &kv_full[st], (H + kvh) * HD + 64 * c, krow);
      tma_load_2d(sV + st * C::TILE_BYTES + c * 16384, &tm, &kv_full[st], (H + KVH + kvh) * HD + 64 * c, krow);
    }
  };
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm);
    mbar_init(q_full, 1);
    mbar_init(&kv_full[0], 1);
    mbar_init(&kv_full[1], 1);
    fence_barrier_init();
    mbar_arrive_expect_tx(q_full, C::TILE_BYTES);
    for (int c = 0; c < C::NCH; ++c) tma_load_2d(sQ + c * 16384, &tm, q_full, h * HD + 64 * c, row0);
    for (int j = 0; j < 2 && j < n_kv; ++j) load_kv(j);
  }
  __syncthreads();

  const int r_lo = qt * 128 + wg * 64 + w4 * 16 + (lane >> 2);   // sequence index of the thread's rows r_lo, r_lo + 8
  const int cq = 2 * (lane & 3);
  const uint64_t qd = make_smem_desc(smem_u32(sQ) + wg * 8192, 0, 1024);
  float oacc[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) oacc[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  mbar_wait(q_full, 0);
  for (int j = 0; j < n_kv; ++j) {
    const int st = j & 1;
    mbar_wait(&kv_full[st], (j >> 1) & 1);
    const uint64_t kd = make_smem_desc(smem_u32(sK + st * C::TILE_BYTES), 0, 1024);
    const uint64_t vd = make_smem_desc(smem_u32(sV + st * C::TILE_BYTES), 16384, 1024);
    float s[64];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) {
      const uint32_t off = ((kk >> 2) * 16384 + (kk & 3) * 32) >> 4;
      wgmma_bf16_ss_n128<0, 0>(s, qd + off, kd + off, kk != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    // masking only on the diagonal / ragged last tile
    const int kv0 = j * 128;
    if (j == qt || kv0 + 128 > S) {
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const int kv = kv0 + 8 * (i >> 2) + cq + (i & 1);
        const int q = r_lo + 8 * ((i >> 1) & 1);
        if (kv > q || kv >= S) s[i] = -INFINITY;
      }
    }
    float corr[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * hh], s[4 * jj + 2 * hh + 1]));
      const float m_new = fmaxf(m_run[hh], quad_max(mx) * scale_log2);
      corr[hh] = exp2f(m_run[hh] - m_new);
      m_run[hh] = m_new;
      float ls = 0.f;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int i = 4 * jj + 2 * hh + e;
          s[i] = exp2f(fmaf(s[i], scale_log2, -m_new));
          ls += s[i];
        }
      }
      l_run[hh] = l_run[hh] * corr[hh] + ls;
    }
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) oacc[i] *= corr[(i >> 1) & 1];
    uint32_t pa[8][4];                         // P as A fragments, all packed before the MMA batch starts
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) acc_to_frag(s, kk, pa[kk]);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) mma_rs_hd<HD, 1>(oacc, pa[kk], vd + ((kk * 2048) >> 4));   // 16 kv rows per step
    wgmma_commit();
    wgmma_wait<0>();
    named_bar_sync(1, ATT_THREADS);          // both warpgroups are done with this K/V stage
    if (threadIdx.x == 0 && j + 2 < n_kv) load_kv(j + 2);
  }

#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int q = r_lo + 8 * hh;
    const float l = quad_sum(l_run[hh]);
    if (q < S) {
      const float inv_l = 1.f / l;
      __nv_bfloat16* orow = o + (static_cast<size_t>(b) * S + q) * (H * HD) + h * HD;
#pragma unroll
      for (int jj = 0; jj < HD / 8; ++jj)
        *reinterpret_cast<uint32_t*>(orow + 8 * jj + cq) =
            pack_bf16x2(oacc[4 * jj + 2 * hh] * inv_l, oacc[4 * jj + 2 * hh + 1] * inv_l);
      if ((lane & 3) == 0) lse[(static_cast<size_t>(b) * H + h) * S + q] = (m_run[hh] + log2f(l)) * LN2;
    }
  }
}

// ===================================================================================== backward prep
// -delta[b,h,s] = -sum_d dO[b,s,h,d] * O[b,s,h,d]  and  -lse * log2(e)  (both planes NEGATED: the backward kernels use
// them as the addend of an FFMA).  HD/8 lanes per (row, head), one 16-byte load of dO and of O per lane.
template <int HD>
__global__ void __launch_bounds__(256) attn_delta_kernel(const __nv_bfloat16* __restrict__ dout, const __nv_bfloat16* __restrict__ o,
                                                         float* __restrict__ delta, const float* __restrict__ lse,
                                                         float* __restrict__ lse2, int B, int S, int H, int ld) {
  constexpr int G = HD / 8;                              // lanes per (row, head)
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long item = gid / G;                        // (b*S + s) * H + h
  const int sub = (int)(gid % G);
  const bool live = item < (long long)B * S * H;
  float acc = 0.f;
  if (live) {
    const uint4 x = *reinterpret_cast<const uint4*>(dout + item * HD + sub * 8);
    const uint4 y = *reinterpret_cast<const uint4*>(o + item * HD + sub * 8);
    const uint32_t xs[4] = {x.x, x.y, x.z, x.w}, ys[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 a = unpack_bf16x2(xs[i]), c = unpack_bf16x2(ys[i]);
      acc = fmaf(a.x, c.x, fmaf(a.y, c.y, acc));
    }
  }
#pragma unroll
  for (int m = G / 2; m > 0; m >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, m);
  if (live && sub == 0) {
    const int h = (int)(item % H);
    const long long bs = item / H;
    const int b = (int)(bs / S), sq = (int)(bs % S);
    delta[((size_t)b * H + h) * ld + sq] = -acc;
    if (lse2) lse2[((size_t)b * H + h) * ld + sq] = -lse[((size_t)b * H + h) * S + sq] * LOG2E;
  }
}

// ============================================================================================ backward
enum { MODE_DKDV = 0, MODE_DQ = 1 };

template <int HD>
struct BwdCfg {
  static constexpr int NCH = HD / 64;
  static constexpr int X_BYTES = 128 * HD * 2;     // resident 128-row tile: NCH chunks of 16 KiB
  static constexpr int Y_BYTES = 64 * HD * 2;      // streamed 64-row tile: NCH chunks of 8 KiB
  static constexpr int SMEM = 2 * X_BYTES + 2 * 2 * Y_BYTES + 1024 + 256;
};

// MODE_DKDV: X1 = K, X2 = V (128 kv rows), streamed Y1 = Q, Y2 = dO (64 q rows);  S^T = X1 Y1^T, dP^T = X2 Y2^T,
//            acc1 (dV) += P^T Y2, acc2 (dK) += dS^T Y1.
// MODE_DQ:   X1 = Q, X2 = dO (128 q rows), streamed Y1 = K, Y2 = V (64 kv rows);  S = X1 Y1^T, dP = X2 Y2^T,
//            acc2 (dQ) += dS Y1.
template <int HD, int MODE>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                const float* __restrict__ lse2g, const float* __restrict__ delta, __nv_bfloat16* __restrict__ dqkv,
                int S, int H, int KVH, float scale, int n_t128, int ld, const float* __restrict__ rope) {
  using C = BwdCfg<HD>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sX1 = smem;
  uint8_t* sX2 = sX1 + C::X_BYTES;
  uint8_t* sY = sX2 + C::X_BYTES;            // [2 stages][Y1 | Y2]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sY + 4 * C::Y_BYTES);
  uint64_t* x_full = bars;
  uint64_t* y_full = bars + 1;               // [2]

  const int wg = threadIdx.x >> 7, w4 = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int G = H / KVH;
  const int b = blockIdx.z;
  const float scale_log2 = scale * LOG2E;
  const int n_t64 = (S + 63) / 64;
  int t128, head_lo, head_n, kvh;
  if constexpr (MODE == MODE_DKDV) {
    t128 = blockIdx.x; kvh = blockIdx.y; head_lo = kvh * G; head_n = G;
  } else {
    t128 = n_t128 - 1 - blockIdx.x; head_lo = blockIdx.y; head_n = 1; kvh = blockIdx.y / G;
  }
  // streamed 64-row tiles: dK/dV -> q tiles from the diagonal to the end; dQ -> kv tiles up to the diagonal
  const int s_lo = (MODE == MODE_DKDV) ? 2 * t128 : 0;
  const int s_hi = (MODE == MODE_DKDV) ? n_t64 : min(2 * t128 + 2, n_t64);
  const int per_head = s_hi - s_lo;
  const int n_iter = per_head * head_n;
  const int xrow0 = b * S + t128 * 128;

  auto load_y = [&](int it) {
    const int st = it & 1;
    const int hh = head_lo + it / per_head;
    const int yrow = b * S + (s_lo + it % per_head) * 64;
    uint8_t* y1 = sY + st * 2 * C::Y_BYTES;
    uint8_t* y2 = y1 + C::Y_BYTES;
    mbar_arrive_expect_tx(&y_full[st], 2 * C::Y_BYTES);
    for (int c = 0; c < C::NCH; ++c) {
      if constexpr (MODE == MODE_DKDV) {
        tma_load_2d(y1 + c * 8192, &tm_qkv, &y_full[st], hh * HD + 64 * c, yrow);
        tma_load_2d(y2 + c * 8192, &tm_do, &y_full[st], hh * HD + 64 * c, yrow);
      } else {
        tma_load_2d(y1 + c * 8192, &tm_qkv, &y_full[st], (H + kvh) * HD + 64 * c, yrow);
        tma_load_2d(y2 + c * 8192, &tm_qkv, &y_full[st], (H + KVH + kvh) * HD + 64 * c, yrow);
      }
    }
  };
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_qkv); tma_prefetch_desc(&tm_do);
    mbar_init(x_full, 1);
    mbar_init(&y_full[0], 1);
    mbar_init(&y_full[1], 1);
    fence_barrier_init();
    mbar_arrive_expect_tx(x_full, 2 * C::X_BYTES);
    for (int c = 0; c < C::NCH; ++c) {
      for (int half = 0; half < 2; ++half) {   // 128 rows as two 64-row boxes
        uint8_t* d1 = sX1 + c * 16384 + half * 8192;
        uint8_t* d2 = sX2 + c * 16384 + half * 8192;
        const int r = xrow0 + 64 * half;
        if constexpr (MODE == MODE_DKDV) {
          tma_load_2d(d1, &tm_qkv, x_full, (H + kvh) * HD + 64 * c, r);
          tma_load_2d(d2, &tm_qkv, x_full, (H + KVH + kvh) * HD + 64 * c, r);
        } else {
          tma_load_2d(d1, &tm_qkv, x_full, head_lo * HD + 64 * c, r);
          tma_load_2d(d2, &tm_do, x_full, head_lo * HD + 64 * c, r);
        }
      }
    }
    for (int it = 0; it < 2 && it < n_iter; ++it) load_y(it);
  }
  __syncthreads();

  const int x_lo = t128 * 128 + wg * 64 + w4 * 16 + (lane >> 2);   // sequence index of the thread's rows x_lo, x_lo + 8
  const int cq = 2 * (lane & 3);
  const uint64_t x1d = make_smem_desc(smem_u32(sX1) + wg * 8192, 0, 1024);
  const uint64_t x2d = make_smem_desc(smem_u32(sX2) + wg * 8192, 0, 1024);
  float acc1[MODE == MODE_DKDV ? HD / 2 : 1];
  float acc2[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) acc2[i] = 0.f;
#pragma unroll
  for (int i = 0; i < (MODE == MODE_DKDV ? HD / 2 : 1); ++i) acc1[i] = 0.f;
  float row_nl[2] = {0.f, 0.f}, row_nd[2] = {0.f, 0.f};
  if constexpr (MODE == MODE_DQ) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const size_t sidx = ((size_t)b * H + head_lo) * ld + min(x_lo + 8 * hh, S - 1);
      row_nl[hh] = lse2g[sidx];
      row_nd[hh] = delta[sidx];
    }
  }

  mbar_wait(x_full, 0);
  for (int it = 0; it < n_iter; ++it) {
    const int st = it & 1;
    const int hh_head = head_lo + it / per_head;
    const int y0 = (s_lo + it % per_head) * 64;        // first streamed sequence index
    const uint32_t y1a = smem_u32(sY + st * 2 * C::Y_BYTES), y2a = y1a + C::Y_BYTES;
    // streamed-index statistics (dK/dV: the q columns of this thread)
    float col_nl[16], col_nd[16];
    if constexpr (MODE == MODE_DKDV) {
      const size_t base = ((size_t)b * H + hh_head) * ld;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int y = min(y0 + 8 * (i >> 1) + cq + (i & 1), S - 1);
        col_nl[i] = lse2g[base + y];
        col_nd[i] = delta[base + y];
      }
    }
    mbar_wait(&y_full[st], (it >> 1) & 1);
    const uint64_t y1d = make_smem_desc(y1a, 0, 1024), y2d = make_smem_desc(y2a, 0, 1024);
    float s[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) {
      const uint32_t ox = ((kk >> 2) * 16384 + (kk & 3) * 32) >> 4, oy = ((kk >> 2) * 8192 + (kk & 3) * 32) >> 4;
      wgmma_bf16_ss_n64<0, 0>(s, x1d + ox, y1d + oy, kk != 0);
    }
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) {
      const uint32_t ox = ((kk >> 2) * 16384 + (kk & 3) * 32) >> 4, oy = ((kk >> 2) * 8192 + (kk & 3) * 32) >> 4;
      wgmma_bf16_ss_n64<0, 0>(dp, x2d + ox, y2d + oy, kk != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    // P and dS (unscaled) in place of S and dP
    // only tiles that touch the causal diagonal or cross the sequence end need per-element masking
    const bool diag = (MODE == MODE_DKDV) ? (y0 < t128 * 128 + 128) : (y0 + 64 > t128 * 128);
    const bool need_mask = diag || (y0 + 64 > S) || (t128 * 128 + 128 > S);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int x = x_lo + 8 * ((i >> 1) & 1);
      const int y = y0 + 8 * (i >> 2) + cq + (i & 1);
      float nl, nd;
      if constexpr (MODE == MODE_DKDV) { nl = col_nl[2 * (i >> 2) + (i & 1)]; nd = col_nd[2 * (i >> 2) + (i & 1)]; }
      else { nl = row_nl[(i >> 1) & 1]; nd = row_nd[(i >> 1) & 1]; }
      bool masked = false;
      if (need_mask) masked = (MODE == MODE_DKDV) ? (x > y || y >= S || x >= S) : (y > x || y >= S || x >= S);
      const float pv = masked ? 0.f : exp2f(fmaf(s[i], scale_log2, nl));
      s[i] = pv;
      dp[i] = masked ? 0.f : pv * (dp[i] + nd);
    }
    // Y1 / Y2 as MN-major B operands: 16 streamed rows per step, 64-column chunks 8 KiB apart
    const uint64_t y1t = make_smem_desc(y1a, 8192, 1024), y2t = make_smem_desc(y2a, 8192, 1024);
    uint32_t pa[4][4], da[4][4];               // P and dS as A fragments, all packed before the MMA batch starts
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      if constexpr (MODE == MODE_DKDV) acc_to_frag(s, kk, pa[kk]);
      acc_to_frag(dp, kk, da[kk]);
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      if constexpr (MODE == MODE_DKDV) mma_rs_hd<HD, 1>(acc1, pa[kk], y2t + ((kk * 2048) >> 4));
      mma_rs_hd<HD, 1>(acc2, da[kk], y1t + ((kk * 2048) >> 4));
    }
    wgmma_commit();
    wgmma_wait<0>();
    named_bar_sync(1, ATT_THREADS);          // both warpgroups are done with this stage
    if (threadIdx.x == 0 && it + 2 < n_iter) load_y(it + 2);
  }

  // epilogue: acc2 = dK | dQ (times the softmax scale, with the INVERSE rotary embedding of the row's position: the
  // forward RoPE lives in the QKV GEMM epilogue, so what leaves here is the gradient of the un-rotated projection;
  // table [S][HD/2][cos, sin]); acc1 = dV
  const int Wd = (H + 2 * KVH) * HD;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int x = x_lo + 8 * hh;
    if (x >= S) continue;
    __nv_bfloat16* drow = dqkv + ((size_t)b * S + x) * Wd;
    const int col2 = (MODE == MODE_DKDV) ? (H + kvh) * HD : head_lo * HD;
    const float* trow = rope ? rope + (size_t)x * HD : nullptr;
#pragma unroll
    for (int jj = 0; jj < HD / 8; ++jj) {
      const int c = 8 * jj + cq;
      float f0 = acc2[4 * jj + 2 * hh] * scale, f1 = acc2[4 * jj + 2 * hh + 1] * scale;
      if (trow) {
        const float2 cs = *reinterpret_cast<const float2*>(trow + c);
        const float a0 = f0, a1 = f1;
        f0 = a0 * cs.x + a1 * cs.y;
        f1 = a1 * cs.x - a0 * cs.y;
      }
      *reinterpret_cast<uint32_t*>(drow + col2 + c) = pack_bf16x2(f0, f1);
      if constexpr (MODE == MODE_DKDV)
        *reinterpret_cast<uint32_t*>(drow + (H + KVH + kvh) * HD + c) =
            pack_bf16x2(acc1[4 * jj + 2 * hh], acc1[4 * jj + 2 * hh + 1]);
    }
  }
}

template <int HD>
static int launch_fwd(const void* qkv, void* o, float* lse, int B, int S, int H, int KVH, float scale, cudaStream_t st) {
  using C = FwdCfg<HD>;
  CUtensorMap tm;
  const int W = (H + 2 * KVH) * HD;
  if (make_tmap_2d_bf16(&tm, qkv, (uint64_t)W, (uint64_t)B * S, (uint64_t)W, 64, 128)) return -3;
  auto kern = attn_fwd_kernel<HD>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  const int n_qt = (S + 127) / 128;
  kern<<<dim3(n_qt, H, B), ATT_THREADS, C::SMEM, st>>>(tm, (__nv_bfloat16*)o, lse, S, H, KVH, scale * LOG2E, n_qt);
  return (int)cudaGetLastError();
}

template <int HD>
static int launch_bwd(const void* dout, const void* qkv, const void* o, const float* lse, void* dqkv, float* delta,
                      int B, int S, int H, int KVH, float scale, const float* rope, cudaStream_t st) {
  using C = BwdCfg<HD>;
  const int W = (H + 2 * KVH) * HD;
  CUtensorMap q64, d64;
  if (make_tmap_2d_bf16(&q64, qkv, (uint64_t)W, (uint64_t)B * S, (uint64_t)W, 64, 64)) return -3;
  if (make_tmap_2d_bf16(&d64, dout, (uint64_t)H * HD, (uint64_t)B * S, (uint64_t)H * HD, 64, 64)) return -3;
  // rows padded to a multiple of 128; plane 0 = -delta, plane 1 = -lse * log2(e)
  const int ld = ((S + 127) / 128) * 128;
  float* lse2 = delta + (size_t)B * H * ld;
  {
    const long long lanes = (long long)B * S * H * (HD / 8);
    const long long blocks = (lanes + 255) / 256;
    attn_delta_kernel<HD><<<(unsigned)blocks, 256, 0, st>>>((const __nv_bfloat16*)dout, (const __nv_bfloat16*)o, delta,
                                                            lse, lse2, B, S, H, ld);
  }
  auto j1 = attn_bwd_kernel<HD, MODE_DKDV>;
  auto j2 = attn_bwd_kernel<HD, MODE_DQ>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(j1, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM);
    if (e != cudaSuccess) return (int)e;
    e = cudaFuncSetAttribute(j2, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  const int n_t = (S + 127) / 128;
  j1<<<dim3(n_t, KVH, B), ATT_THREADS, C::SMEM, st>>>(q64, d64, lse2, delta, (__nv_bfloat16*)dqkv, S, H, KVH, scale, n_t,
                                                      ld, rope);
  j2<<<dim3(n_t, H, B), ATT_THREADS, C::SMEM, st>>>(q64, d64, lse2, delta, (__nv_bfloat16*)dqkv, S, H, KVH, scale, n_t,
                                                    ld, rope);
  return (int)cudaGetLastError();
}

}  // namespace b200

extern "C" int b200_attn_fwd(const void* qkv, void* o, float* lse, int B, int S, int H, int KVH, int HD, float scale,
                             cudaStream_t st) {
  if (H % KVH) return -1;
  if (HD == 128) return b200::launch_fwd<128>(qkv, o, lse, B, S, H, KVH, scale, st);
  if (HD == 64) return b200::launch_fwd<64>(qkv, o, lse, B, S, H, KVH, scale, st);
  return -2;
}
// rope (optional): [S][HD/2][cos, sin] table; dq and dk leave the kernel with the inverse rotation applied
extern "C" int b200_attn_bwd(const void* dout, const void* qkv, const void* o, const float* lse, void* dqkv,
                             float* delta, int B, int S, int H, int KVH, int HD, float scale, const float* rope,
                             cudaStream_t st) {
  if (H % KVH) return -1;
  if (HD == 128) return b200::launch_bwd<128>(dout, qkv, o, lse, dqkv, delta, B, S, H, KVH, scale, rope, st);
  if (HD == 64) return b200::launch_bwd<64>(dout, qkv, o, lse, dqkv, delta, B, S, H, KVH, scale, rope, st);
  return -2;
}
