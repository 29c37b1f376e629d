// Causal GQA flash attention for sm_90a on wgmma tensor cores (SURVEY.md K3 / M7).
//
// Input is the fused, already-roped projection qkv [B*S, (H+2*KVH)*HD] (bf16); 2-D TMA maps with {64 x 128|64}-element
// boxes serve Q, K and V.  Every GEMM is a wgmma with fp32 accumulators in registers; the softmax probabilities P and
// the score gradients dS go back into the tensor core as register A operands (the wgmma accumulator layout of 16
// columns is exactly the m64k16 A-fragment layout), so they never touch shared memory.
//
// Every kernel is warp-specialised: warpgroup 0 is a TMA producer that keeps a ring of streamed tiles full (full / empty
// mbarriers per stage, no CTA-wide barrier per tile) and hands its registers to two consumer warpgroups of 64 rows each
// (setmaxnreg: 128 x 24 + 256 x 240 <= 64K).
//
//  forward   CTA = (head, batch, q tile of 128).  Per kv tile of 128: S = Q K^T, online softmax in registers (rows are
//            shared by 4 lanes), O += P V with V consumed as an MN-major operand.  S_{j+1} = Q K_{j+1}^T and P_j V_j are
//            issued before the softmax of tile j+1.
//  backward  two kernels:  dK/dV: CTA = (kv head, batch, kv tile 128), streams (Q_i, dO_i) tiles of 64 rows of every
//            head of the GQA group, computes S^T = K Q^T and dP^T = V dO^T, accumulates dV += P^T dO and dK += dS^T Q
//            in registers (GQA group summed in the accumulator, no atomics);  dQ: CTA = (head, batch, q tile 128),
//            streams (K_j, V_j) tiles of 64, dQ += dS K.  The score GEMMs are recomputed in both kernels in exchange
//            for a deterministic, atomic-free dQ.  S and dP are separate commit groups (exp2 of S runs while dP
//            computes), dV += P^T dO is issued before dS is formed, and the accumulate MMAs of tile i stay in flight
//            under the score GEMMs of tile i+1 (not at dK/dV hd 128, see CARRY);  the dK/dV kernel's -lse and -delta of
//            the streamed rows arrive in the stage by a 1-D bulk copy.
//  launch order: longest first.  The tile index is the slowest grid coordinate, so the heaviest tile of every (head,
//            batch) is issued before any lighter one (at B2 H16 KVH4 S4096 the dK/dV grid of 256 CTAs on 132 SMs otherwise
//            starts batch 1's diagonal tiles, 4x64 streamed tiles each, after ~90 light CTAs have finished).
//
// Document masking (DOC = true, packed training rows): a segment table seg [2][B*S] int32 holds, per position, the
// first (plane 0) and last (plane 1) position of its document within the row.  Key k is visible to query q when
// seg0[q] <= k <= q, equivalently k <= q <= seg1[k].  Both planes are non-decreasing, so the first row of a q tile has
// the smallest document start of the tile and the first row of a kv tile the smallest document end: whole tiles
// outside the document band are skipped, the rest are masked per element like the diagonal.  Each kernel takes the
// one plane it needs (forward and dQ: seg0; dK/dV: seg1), nullptr when DOC = false.
#include "common.cuh"
#include "tensormap.h"
#include "wgmma.cuh"

namespace b200 {

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

constexpr int PIPE_THREADS = 384;                       // producer warpgroup + two consumer warpgroups
constexpr int PRODUCER_REGS = 24, CONSUMER_REGS = 240;

template <int N>
B200_DEVINL void attn_regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
B200_DEVINL void attn_regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// 1-D bulk copy global -> shared (16-byte aligned, size a multiple of 16), completing on an mbarrier
B200_DEVINL void bulk_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ============================================================================================ forward
template <int HD>
struct FwdPipeCfg {
  static constexpr int NCH = HD / 64;
  static constexpr int TILE_BYTES = 128 * HD * 2;
  static constexpr int STAGES = 2;                      // K and V rings (released separately)
  static constexpr int SMEM = TILE_BYTES * (1 + 2 * STAGES) + 1024 + 256;
};

// grid (H, B, n_qt): q tile slowest, heavy to light
template <int HD, bool DOC>
__global__ void __launch_bounds__(PIPE_THREADS, 1)
attn_fwd_pipe_kernel(const __grid_constant__ CUtensorMap tm, __nv_bfloat16* __restrict__ o, float* __restrict__ lse,
                     int S, int H, int KVH, float scale_log2, int n_qt, const int* __restrict__ seg0) {
  using C = FwdPipeCfg<HD>;
  constexpr int ST = C::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + C::TILE_BYTES;          // [ST]
  uint8_t* sV = sK + ST * C::TILE_BYTES;     // [ST]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + ST * C::TILE_BYTES);
  uint64_t* q_full = bars;
  uint64_t* k_full = bars + 1;               // [ST] each
  uint64_t* v_full = k_full + ST;
  uint64_t* k_empty = v_full + ST;
  uint64_t* v_empty = k_empty + ST;

  const int wg = threadIdx.x >> 7, w4 = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int h = blockIdx.x, b = blockIdx.y;
  const int qt = n_qt - 1 - blockIdx.z;
  const int kvh = h / (H / KVH);
  const int row0 = b * S + qt * 128;
  const int n_kv = min(qt + 1, (S + 127) / 128);
  // DOC: kv tiles before the document of the tile's first row hold no visible key for any row of the tile
  const int* srow = DOC ? seg0 + static_cast<size_t>(b) * S : nullptr;
  const int j_lo = DOC ? srow[qt * 128] / 128 : 0;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < ST; ++s) {
      mbar_init(&k_full[s], 1);
      mbar_init(&v_full[s], 1);
      mbar_init(&k_empty[s], 8);             // one arrive per consumer warp
      mbar_init(&v_empty[s], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    attn_regs_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      tma_prefetch_desc(&tm);
      mbar_arrive_expect_tx(q_full, C::TILE_BYTES);
      for (int c = 0; c < C::NCH; ++c) tma_load_2d(sQ + c * 16384, &tm, q_full, h * HD + 64 * c, row0);
      for (int j = j_lo; j < n_kv; ++j) {
        const int st = (j - j_lo) % ST;
        const uint32_t ph = ((j - j_lo) / ST) & 1;
        const int krow = b * S + j * 128;
        mbar_wait(&k_empty[st], ph ^ 1);
        mbar_arrive_expect_tx(&k_full[st], C::TILE_BYTES);
        for (int c = 0; c < C::NCH; ++c)
          tma_load_2d(sK + st * C::TILE_BYTES + c * 16384, &tm, &k_full[st], (H + kvh) * HD + 64 * c, krow);
        mbar_wait(&v_empty[st], ph ^ 1);
        mbar_arrive_expect_tx(&v_full[st], C::TILE_BYTES);
        for (int c = 0; c < C::NCH; ++c)
          tma_load_2d(sV + st * C::TILE_BYTES + c * 16384, &tm, &v_full[st], (H + KVH + kvh) * HD + 64 * c, krow);
      }
    }
    asm volatile("exit;");                 // not return: a path that rejoins the consumers' caps them at 168 registers
  }
  attn_regs_inc<CONSUMER_REGS>();
  const int cw = wg - 1;                     // consumer warpgroup: q rows [64 cw, 64 cw + 64) of the tile

  const int r_lo = qt * 128 + cw * 64 + w4 * 16 + (lane >> 2);   // sequence index of the thread's rows r_lo, r_lo + 8
  const int cq = 2 * (lane & 3);
  int doc_lo[2] = {0, 0}, tile_doc_hi = 0;     // DOC: document start of the thread's rows and of the tile's last row
  if constexpr (DOC) {
    doc_lo[0] = srow[min(r_lo, S - 1)];
    doc_lo[1] = srow[min(r_lo + 8, S - 1)];
    tile_doc_hi = srow[min(qt * 128 + 127, S - 1)];
  }
  const uint64_t qd = make_smem_desc(smem_u32(sQ) + cw * 8192, 0, 1024);
  float oacc[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) oacc[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  auto issue_s = [&](int j, float (&s)[64]) {          // S_j = Q K_j^T, one commit group
    const int n = j - j_lo;
    mbar_wait(&k_full[n % ST], (n / ST) & 1);
    const uint64_t kd = make_smem_desc(smem_u32(sK + (n % ST) * C::TILE_BYTES), 0, 1024);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) {
      const uint32_t off = ((kk >> 2) * 16384 + (kk & 3) * 32) >> 4;
      wgmma_bf16_ss_n128<0, 0>(s, qd + off, kd + off, kk != 0);
    }
    wgmma_commit();
  };
  auto issue_pv = [&](int j, const uint32_t (&pa)[8][4]) {   // O += P_j V_j, one commit group
    const int n = j - j_lo;
    mbar_wait(&v_full[n % ST], (n / ST) & 1);
    const uint64_t vd = make_smem_desc(smem_u32(sV + (n % ST) * C::TILE_BYTES), 16384, 1024);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) mma_rs_hd<HD, 1>(oacc, pa[kk], vd + ((kk * 2048) >> 4));
    wgmma_commit();
  };
  auto release = [&](uint64_t* empty, int j) {
    if (lane == 0) mbar_arrive(&empty[(j - j_lo) % ST]);
  };
  // masking and online softmax of tile j: s -> P, m_run / l_run updated, corr = rescale of O.  Masking only on the
  // diagonal / ragged last tile (DOC: and on tiles that start before some row's document).
  auto softmax = [&](int j, float (&s)[64], float (&corr)[2]) {
    const int kv0 = j * 128;
    if (j == qt || kv0 + 128 > S || (DOC && kv0 < tile_doc_hi)) {
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const int kv = kv0 + 8 * (i >> 2) + cq + (i & 1);
        const int q = r_lo + 8 * ((i >> 1) & 1);
        if (kv > q || kv >= S || (DOC && kv < doc_lo[(i >> 1) & 1])) s[i] = -INFINITY;
      }
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * hh], s[4 * jj + 2 * hh + 1]));
      const float m_new = fmaxf(m_run[hh], quad_max(mx) * scale_log2);
      // DOC: a row whose document starts after this tile has seen no key yet (m_new = -inf); subtracting 0 instead
      // keeps exp2(-inf - m) at 0 rather than NaN.  Plain causal rows always see key 0 in the first tile.
      const float m_sub = (DOC && m_new == -INFINITY) ? 0.f : m_new;
      corr[hh] = exp2f(m_run[hh] - m_sub);
      m_run[hh] = m_new;
      float ls = 0.f;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int i = 4 * jj + 2 * hh + e;
          s[i] = exp2f(fmaf(s[i], scale_log2, -m_sub));
          ls += s[i];
        }
      }
      l_run[hh] = l_run[hh] * corr[hh] + ls;
    }
  };

  mbar_wait(q_full, 0);
  float s[64], corr[2];
  uint32_t pa[8][4];                           // P_j as A fragments
  issue_s(j_lo, s);
  wgmma_wait<0>();
  release(k_empty, j_lo);
  softmax(j_lo, s, corr);
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) oacc[i] *= corr[(i >> 1) & 1];
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) acc_to_frag(s, kk, pa[kk]);
  for (int j = j_lo + 1; j < n_kv; ++j) {
    issue_s(j, s);
    issue_pv(j - 1, pa);
    wgmma_wait<1>();                           // S_j has landed; P_{j-1} V_{j-1} may still run
    release(k_empty, j);
    softmax(j, s, corr);
    wgmma_wait<0>();
    release(v_empty, j - 1);
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) oacc[i] *= corr[(i >> 1) & 1];
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) acc_to_frag(s, kk, pa[kk]);
  }
  issue_pv(n_kv - 1, pa);
  wgmma_wait<0>();

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

// ============================================================================================ backward
enum { MODE_DKDV = 0, MODE_DQ = 1 };

template <int HD>
struct BwdPipeCfg {
  static constexpr int NCH = HD / 64;
  static constexpr int X_BYTES = 128 * HD * 2;
  static constexpr int Y_BYTES = 64 * HD * 2;
  static constexpr int STAGES = 3;
  static constexpr int STAT_BYTES = 2 * 64 * 4;         // dK/dV: -lse * log2(e) | -delta of the 64 streamed rows
  static constexpr int SMEM = 2 * X_BYTES + STAGES * (2 * Y_BYTES + STAT_BYTES) + 1024 + 256;
};

// MODE_DKDV: X1 = K, X2 = V (128 kv rows), streamed Y1 = Q, Y2 = dO (64 q rows);  S^T = X1 Y1^T, dP^T = X2 Y2^T,
//            acc1 (dV) += P^T Y2, acc2 (dK) += dS^T Y1.
// MODE_DQ:   X1 = Q, X2 = dO (128 q rows), streamed Y1 = K, Y2 = V (64 kv rows);  S = X1 Y1^T, dP = X2 Y2^T,
//            acc2 (dQ) += dS Y1.
// DOC: seg_plane = seg1 (document ends) for MODE_DKDV, seg0 (document starts) for MODE_DQ.
// grid (KVH, B, n_t) for dK/dV (kv tile slowest; tile 0, on the diagonal of the whole sequence, streams the most q
// tiles), (H, B, n_t) for dQ (q tile slowest, heavy to light).
template <int HD, int MODE, bool DOC>
__global__ void __launch_bounds__(PIPE_THREADS, 1)
attn_bwd_pipe_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_do,
                     const float* __restrict__ lse2g, const float* __restrict__ delta, __nv_bfloat16* __restrict__ dqkv,
                     int S, int H, int KVH, float scale, int n_t128, int ld, const float* __restrict__ rope,
                     const int* __restrict__ seg_plane) {
  using C = BwdPipeCfg<HD>;
  constexpr int ST = C::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sX1 = smem;
  uint8_t* sX2 = sX1 + C::X_BYTES;
  uint8_t* sY = sX2 + C::X_BYTES;            // [ST][Y1 | Y2]
  float* sStat = reinterpret_cast<float*>(sY + ST * 2 * C::Y_BYTES);   // [ST][-lse*log2e | -delta][64]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sStat + ST * 128);
  uint64_t* x_full = bars;
  uint64_t* y_full = bars + 1;               // [ST]
  uint64_t* y_empty = y_full + ST;           // [ST]

  const int wg = threadIdx.x >> 7, w4 = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int G = H / KVH;
  const int b = blockIdx.y;
  const float scale_log2 = scale * LOG2E;
  const int n_t64 = (S + 63) / 64;
  int t128, head_lo, head_n, kvh;
  if constexpr (MODE == MODE_DKDV) {
    t128 = blockIdx.z; kvh = blockIdx.x; head_lo = kvh * G; head_n = G;
  } else {
    t128 = n_t128 - 1 - blockIdx.z; head_lo = blockIdx.x; head_n = 1; kvh = blockIdx.x / G;
  }
  // DOC: the document bound of the tile's first and last resident row (dK/dV: end, dQ: start)
  const int* srow = DOC ? seg_plane + static_cast<size_t>(b) * S : nullptr;
  const int tile_doc_first = DOC ? srow[t128 * 128] : 0;
  const int tile_doc_last = DOC ? srow[min(t128 * 128 + 127, S - 1)] : 0;
  // streamed 64-row tiles: dK/dV -> q tiles from the diagonal to the end (DOC: to the last document end of the tile);
  // dQ -> kv tiles up to the diagonal (DOC: from the first document start of the tile)
  const int s_lo = (MODE == MODE_DKDV) ? 2 * t128 : (DOC ? tile_doc_first / 64 : 0);
  const int s_hi = (MODE == MODE_DKDV) ? (DOC ? tile_doc_last / 64 + 1 : n_t64) : min(2 * t128 + 2, n_t64);
  const int per_head = s_hi - s_lo;
  const int n_iter = per_head * head_n;
  const int xrow0 = b * S + t128 * 128;

  if (threadIdx.x == 0) {
    mbar_init(x_full, 1);
    for (int s = 0; s < ST; ++s) {
      mbar_init(&y_full[s], 1);
      mbar_init(&y_empty[s], 8);             // one arrive per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    attn_regs_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      tma_prefetch_desc(&tm_qkv); tma_prefetch_desc(&tm_do);
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
      for (int it = 0; it < n_iter; ++it) {
        const int st = it % ST;
        const int hh = head_lo + it / per_head;
        const int y0 = (s_lo + it % per_head) * 64;
        uint8_t* y1 = sY + st * 2 * C::Y_BYTES;
        uint8_t* y2 = y1 + C::Y_BYTES;
        mbar_wait(&y_empty[st], ((it / ST) & 1) ^ 1);
        mbar_arrive_expect_tx(&y_full[st], 2 * C::Y_BYTES + (MODE == MODE_DKDV ? C::STAT_BYTES : 0));
        for (int c = 0; c < C::NCH; ++c) {
          if constexpr (MODE == MODE_DKDV) {
            tma_load_2d(y1 + c * 8192, &tm_qkv, &y_full[st], hh * HD + 64 * c, b * S + y0);
            tma_load_2d(y2 + c * 8192, &tm_do, &y_full[st], hh * HD + 64 * c, b * S + y0);
          } else {
            tma_load_2d(y1 + c * 8192, &tm_qkv, &y_full[st], (H + kvh) * HD + 64 * c, b * S + y0);
            tma_load_2d(y2 + c * 8192, &tm_qkv, &y_full[st], (H + KVH + kvh) * HD + 64 * c, b * S + y0);
          }
        }
        if constexpr (MODE == MODE_DKDV) {
          // rows are padded to ld (a multiple of 128): y0 + 64 <= ld, so the copy stays inside the row; entries past S
          // are never written by attn_delta_kernel, and every column past S is masked below
          const size_t base = ((size_t)b * H + hh) * ld + y0;
          bulk_load_1d(sStat + st * 128, lse2g + base, 256, &y_full[st]);
          bulk_load_1d(sStat + st * 128 + 64, delta + base, 256, &y_full[st]);
        }
      }
    }
    asm volatile("exit;");                 // not return: a path that rejoins the consumers' caps them at 168 registers
  }
  attn_regs_inc<CONSUMER_REGS>();
  const int cw = wg - 1;                     // consumer warpgroup: resident rows [64 cw, 64 cw + 64) of the tile

  const int x_lo = t128 * 128 + cw * 64 + w4 * 16 + (lane >> 2);   // sequence index of the thread's rows x_lo, x_lo + 8
  const int cq = 2 * (lane & 3);
  const uint64_t x1d = make_smem_desc(smem_u32(sX1) + cw * 8192, 0, 1024);
  const uint64_t x2d = make_smem_desc(smem_u32(sX2) + cw * 8192, 0, 1024);
  float acc1[MODE == MODE_DKDV ? HD / 2 : 1];
  float acc2[HD / 2];
#pragma unroll
  for (int i = 0; i < HD / 2; ++i) acc2[i] = 0.f;
#pragma unroll
  for (int i = 0; i < (MODE == MODE_DKDV ? HD / 2 : 1); ++i) acc1[i] = 0.f;
  float row_nl[2] = {0.f, 0.f}, row_nd[2] = {0.f, 0.f};
  int row_doc[2] = {0, 0};                   // DOC: document bound of the thread's resident rows
  if constexpr (DOC) {
    row_doc[0] = srow[min(x_lo, S - 1)];
    row_doc[1] = srow[min(x_lo + 8, S - 1)];
  }
  if constexpr (MODE == MODE_DQ) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const size_t sidx = ((size_t)b * H + head_lo) * ld + min(x_lo + 8 * hh, S - 1);
      row_nl[hh] = lse2g[sidx];
      row_nd[hh] = delta[sidx];
    }
  }

  // CARRY: the accumulate MMAs of tile i stay in flight under the score GEMMs of tile i+1.  Not at dK/dV hd 128: there
  // acc1 + acc2 (128 registers), S + dP (64) and the P / dS fragments still read by the in-flight MMAs (32) exceed the
  // 240-register budget, and ptxas would serialise every wgmma of the kernel; that instantiation retires the
  // accumulate group at the end of each tile instead.
  constexpr bool CARRY = !(MODE == MODE_DKDV && HD == 128);
  mbar_wait(x_full, 0);
  uint32_t pa[4][4], da[4][4];               // P and dS of the tile as A fragments (read by MMAs still in flight)
  for (int it = 0; it < n_iter; ++it) {
    const int st = it % ST;
    const int y0 = (s_lo + it % per_head) * 64;
    const uint32_t y1a = smem_u32(sY + st * 2 * C::Y_BYTES), y2a = y1a + C::Y_BYTES;
    mbar_wait(&y_full[st], (it / ST) & 1);
    const uint64_t y1d = make_smem_desc(y1a, 0, 1024), y2d = make_smem_desc(y2a, 0, 1024);
    float s[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) {
      const uint32_t ox = ((kk >> 2) * 16384 + (kk & 3) * 32) >> 4, oy = ((kk >> 2) * 8192 + (kk & 3) * 32) >> 4;
      wgmma_bf16_ss_n64<0, 0>(s, x1d + ox, y1d + oy, kk != 0);
    }
    wgmma_commit();
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) {
      const uint32_t ox = ((kk >> 2) * 16384 + (kk & 3) * 32) >> 4, oy = ((kk >> 2) * 8192 + (kk & 3) * 32) >> 4;
      wgmma_bf16_ss_n64<0, 0>(dp, x2d + ox, y2d + oy, kk != 0);
    }
    wgmma_commit();
    wgmma_wait<1>();                         // S has landed (CARRY: and so have the accumulate MMAs of the previous tile)
    if (CARRY && it > 0 && lane == 0) mbar_arrive(&y_empty[(it - 1) % ST]);
    // only tiles that touch the causal diagonal or cross the sequence end need per-element masking
    const bool diag = (MODE == MODE_DKDV) ? (y0 < t128 * 128 + 128) : (y0 + 64 > t128 * 128);
    // DOC: also tiles that reach past the first row's document end (dK/dV) or start before the last row's document (dQ)
    const bool doc_edge = DOC && ((MODE == MODE_DKDV) ? (y0 + 63 > tile_doc_first) : (y0 < tile_doc_last));
    const bool need_mask = diag || (y0 + 64 > S) || (t128 * 128 + 128 > S) || doc_edge;
    const float* stl = sStat + st * 128;
    uint32_t mbits = 0;
    // P in place of S
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int x = x_lo + 8 * ((i >> 1) & 1);
      const int y = y0 + 8 * (i >> 2) + cq + (i & 1);
      const float nl = (MODE == MODE_DKDV) ? stl[8 * (i >> 2) + cq + (i & 1)] : row_nl[(i >> 1) & 1];
      bool masked = false;
      if (need_mask) masked = (MODE == MODE_DKDV) ? (x > y || y >= S || x >= S) : (y > x || y >= S || x >= S);
      if constexpr (DOC) {
        const int bound = row_doc[(i >> 1) & 1];
        if (need_mask) masked = masked || ((MODE == MODE_DKDV) ? (y > bound) : (y < bound));
      }
      mbits |= (masked ? 1u : 0u) << i;
      s[i] = masked ? 0.f : exp2f(fmaf(s[i], scale_log2, nl));
    }
    // Y1 / Y2 as MN-major B operands: 16 streamed rows per step, 64-column chunks 8 KiB apart
    const uint64_t y1t = make_smem_desc(y1a, 8192, 1024), y2t = make_smem_desc(y2a, 8192, 1024);
    if constexpr (MODE == MODE_DKDV) {       // dV += P^T dO while dP is still computing
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) acc_to_frag(s, kk, pa[kk]);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) mma_rs_hd<HD, 1>(acc1, pa[kk], y2t + ((kk * 2048) >> 4));
      wgmma_commit();
      wgmma_wait<1>();                       // dP has landed
    } else {
      wgmma_wait<0>();
    }
    // dS (unscaled) in place of dP
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const float nd = (MODE == MODE_DKDV) ? stl[64 + 8 * (i >> 2) + cq + (i & 1)] : row_nd[(i >> 1) & 1];
      dp[i] = ((mbits >> i) & 1u) ? 0.f : s[i] * (dp[i] + nd);
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) acc_to_frag(dp, kk, da[kk]);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) mma_rs_hd<HD, 1>(acc2, da[kk], y1t + ((kk * 2048) >> 4));
    wgmma_commit();
    if constexpr (!CARRY) {
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(&y_empty[st]);
    }
  }
  wgmma_wait<0>();

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

template <int HD, bool DOC>
static int launch_fwd(const void* qkv, void* o, float* lse, int B, int S, int H, int KVH, float scale, const int* seg,
                      cudaStream_t st) {
  constexpr int SMEM = FwdPipeCfg<HD>::SMEM;
  CUtensorMap tm;
  const int W = (H + 2 * KVH) * HD;
  if (make_tmap_2d_bf16(&tm, qkv, (uint64_t)W, (uint64_t)B * S, (uint64_t)W, 64, 128)) return -3;
  auto kern = attn_fwd_pipe_kernel<HD, DOC>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  const int n_qt = (S + 127) / 128;
  kern<<<dim3(H, B, n_qt), PIPE_THREADS, SMEM, st>>>(tm, (__nv_bfloat16*)o, lse, S, H, KVH, scale * LOG2E, n_qt, seg);
  return (int)cudaGetLastError();
}

template <int HD, bool DOC>
static int launch_bwd(const void* dout, const void* qkv, const void* o, const float* lse, void* dqkv, float* delta,
                      int B, int S, int H, int KVH, float scale, const float* rope, const int* seg, cudaStream_t st) {
  constexpr int SMEM = BwdPipeCfg<HD>::SMEM;
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
  auto j1 = attn_bwd_pipe_kernel<HD, MODE_DKDV, DOC>;
  auto j2 = attn_bwd_pipe_kernel<HD, MODE_DQ, DOC>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(j1, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) return (int)e;
    e = cudaFuncSetAttribute(j2, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  const int n_t = (S + 127) / 128;
  const int* seg1 = DOC ? seg + (size_t)B * S : nullptr;   // dK/dV bounds its q range by document ends, dQ by starts
  j1<<<dim3(KVH, B, n_t), PIPE_THREADS, SMEM, st>>>(q64, d64, lse2, delta, (__nv_bfloat16*)dqkv, S, H, KVH, scale, n_t,
                                                      ld, rope, seg1);
  j2<<<dim3(H, B, n_t), PIPE_THREADS, SMEM, st>>>(q64, d64, lse2, delta, (__nv_bfloat16*)dqkv, S, H, KVH, scale, n_t, ld,
                                                    rope, seg);
  return (int)cudaGetLastError();
}

static int attn_fwd(const void* qkv, void* o, float* lse, int B, int S, int H, int KVH, int HD, float scale,
                    cudaStream_t st, const int* seg) {
  if (H % KVH) return -1;
  if (seg) {
    if (HD == 128) return launch_fwd<128, true>(qkv, o, lse, B, S, H, KVH, scale, seg, st);
    if (HD == 64) return launch_fwd<64, true>(qkv, o, lse, B, S, H, KVH, scale, seg, st);
    return -2;
  }
  if (HD == 128) return launch_fwd<128, false>(qkv, o, lse, B, S, H, KVH, scale, nullptr, st);
  if (HD == 64) return launch_fwd<64, false>(qkv, o, lse, B, S, H, KVH, scale, nullptr, st);
  return -2;
}

static int attn_bwd(const void* dout, const void* qkv, const void* o, const float* lse, void* dqkv, float* delta, int B,
                    int S, int H, int KVH, int HD, float scale, const float* rope, cudaStream_t st, const int* seg) {
  if (H % KVH) return -1;
  if (seg) {
    if (HD == 128) return launch_bwd<128, true>(dout, qkv, o, lse, dqkv, delta, B, S, H, KVH, scale, rope, seg, st);
    if (HD == 64) return launch_bwd<64, true>(dout, qkv, o, lse, dqkv, delta, B, S, H, KVH, scale, rope, seg, st);
    return -2;
  }
  if (HD == 128) return launch_bwd<128, false>(dout, qkv, o, lse, dqkv, delta, B, S, H, KVH, scale, rope, nullptr, st);
  if (HD == 64) return launch_bwd<64, false>(dout, qkv, o, lse, dqkv, delta, B, S, H, KVH, scale, rope, nullptr, st);
  return -2;
}

}  // namespace b200

// seg (optional): [2][B*S] int32 document table (first | last position of each position's document within its row);
// nullptr = plain causal attention
extern "C" int b200_attn_fwd(const void* qkv, void* o, float* lse, int B, int S, int H, int KVH, int HD, float scale,
                             cudaStream_t st, const int* seg) {
  return b200::attn_fwd(qkv, o, lse, B, S, H, KVH, HD, scale, st, seg);
}
// rope (optional): [S][HD/2][cos, sin] table; dq and dk leave the kernel with the inverse rotation applied
extern "C" int b200_attn_bwd(const void* dout, const void* qkv, const void* o, const float* lse, void* dqkv,
                             float* delta, int B, int S, int H, int KVH, int HD, float scale, const float* rope,
                             cudaStream_t st, const int* seg) {
  return b200::attn_bwd(dout, qkv, o, lse, dqkv, delta, B, S, H, KVH, HD, scale, rope, st, seg);
}
