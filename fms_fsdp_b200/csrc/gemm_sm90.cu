// Persistent warp-specialised bf16 GEMM for sm_90a:  C[M,N] (+)= A * B  with fp32 accumulation in registers.
//
//   TMA (cp.async.bulk.tensor, SWIZZLE_128B) -> 6-stage smem ring (mbarrier full / empty) -> wgmma m64n128k16 issued by
//   two consumer warpgroups (64 rows each of a 128 x 128 tile) -> register epilogue.
//
// One kernel serves the three GEMMs of a linear layer (SURVEY.md K1/K4/K6/K8 and their backward):
//   forward  y  = x  W^T : A K-major [M,K],  B K-major [N,K]            ("nt")
//   dgrad    dx = dy W   : A K-major [M,Nr], B MN-major (W is [Nr,K])   ("nn")
//   wgrad    dW = dy^T x : A MN-major (dy is [Mr,N]), B MN-major        ("tn")
// The MN-major cases use wgmma's transposed-operand smem layout, so no transposes are ever materialised.
// Epilogues: plain store, +residual, accumulate into C, RoPE on the QKV projection, SwiGLU (forward and backward),
// push of wgrad tiles to the owning rank, per-row/column scales of the e4m3 path; bf16 or fp32 output.
//
// Warp roles (384 threads): warpgroup 0 = producer (warp 0 lane 0 issues TMA; warps 2-3 are the comm warps of the fused
// all-gather), warpgroups 1-2 = consumers (wgmma + epilogue).
//
// gemm_wide_bf16 is the same pipeline on a 128 x 256 tile (wgmma m64n256k16) for the GEMMs without fused communication;
// use_wide picks the tile per launch.
#include "common.cuh"
#include "tensormap.h"
#include "wgmma.cuh"

namespace b200 {

constexpr int BM = 128, BN = 128, BK = 64;   // BK in bf16 elements = one 128-byte swizzle atom per row
constexpr int STAGES = 6;
constexpr int A_BYTES = BM * BK * 2;          // 16 KiB
constexpr int B_BYTES = BN * BK * 2;          // 16 KiB
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int THREADS = 384;
// push epilogue (bulk mode): each consumer warpgroup stages its 64 x 128 bf16 tile rows (row pitch 272 B: the 16-byte
// pad spreads the rows of a warp's fragment stores over the banks) so every 64-column row chunk leaves the SM as ONE
// 128-byte cp.async.bulk store; the ring gives up one stage to make room
constexpr int PUSH_PITCH = 272;
constexpr int PUSH_STAGE_BYTES = 2 * 64 * PUSH_PITCH;
template <int EPI>
__host__ __device__ constexpr int ring_stages() { return EPI == 4 /*EPI_PUSH*/ ? STAGES - 1 : STAGES; }
template <int EPI>
__host__ __device__ constexpr int smem_bytes() {   // ring + 1 KiB alignment slack + barriers (+ push staging)
  return ring_stages<EPI>() * STAGE_BYTES + 1024 + 256 + (EPI == 4 ? PUSH_STAGE_BYTES : 0);
}

enum { EPI_STORE = 0, EPI_RESIDUAL = 1, EPI_ACCUM = 2, EPI_ROPE = 3, EPI_PUSH = 4, EPI_SWIGLU = 5, EPI_SWIGLU_BWD = 6,
       EPI_SCALE = 7 };
// Grouped (mixture-of-experts) launches of the 128 x 128 kernel carry their mode in the high bits of the EPI template
// argument, so the instantiations that existed before them keep their names and their code.  Operands live in the
// expert-sorted row buffer of csrc/moe.cu; the expert weights are one tensor whose rows hold all experts.
//   GRP_M (forward nt, dgrad nn): m-tile mt belongs to expert p.grp_tile[mt] (-1: past the last segment, the tile is
//          skipped by producer and consumers alike); B's row (nt) or k (nn) coordinate is offset by e * p.grp_rows.
//   GRP_K (wgrad tn): problem b0 = expert e of p.nb0; its k-loop covers the rows [start, start + len) of the buffer
//          (p.grp_seg[e], p.grp_seg[nb0 + e]), rounded out to 64-row blocks that only add padding rows, which are zero;
//          C of expert e starts at e * p.sc0.
constexpr int EPI_MASK = 15, GRP_M = 16, GRP_K = 32;

// L2-friendly rasterisation: sweep all n-tiles for a band of GROUP_M m-tiles before moving to the next band, so the
// band's A rows stay L2-resident while B streams through once per band.
constexpr int GROUP_M = 16;
B200_DEVINL void tile_coords(int t, int m_tiles, int n_tiles, int& mt, int& nt) {
  const int per_band = GROUP_M * n_tiles;
  const int band = t / per_band;
  const int first_m = band * GROUP_M;
  const int band_m = min(GROUP_M, m_tiles - first_m);
  const int r = t - band * per_band;
  mt = first_m + r % band_m;
  nt = r / band_m;
}

// ---- fused all-gather (ag_gemm): the comm warps of the same persistent GEMM pull a unit's parameter shards from the
// peers over NVLink (16-byte ld.relaxed.sys on symmetric-heap addresses) into the local gathered buffer and publish
// per-chunk ready flags.  dependent=1: the B operand of THIS GEMM lives in that buffer, so the TMA producer acquires
// the flags of the chunks under each B tile before issuing its loads.  dependent=0: the gather is the NEXT unit's
// prefetch riding inside this GEMM.
constexpr int AG_CHUNK = 65536;       // bytes per ready flag
struct AgParams {
  const void* const* peer_shards;     // device table [world] of shard base addresses (own rank included)
  uint8_t* full;                      // local gathered buffer
  unsigned long long shard_bytes;
  unsigned long long begin, end;      // byte range of `full` to gather
  int world, rank;
  uint32_t* flags;                    // [ceil(total/AG_CHUNK)] epochs, local memory
  uint32_t epoch;
  int dependent;
  unsigned long long b_off;           // byte offset of the B matrix inside `full`
  unsigned long long b_row_bytes;     // bytes per stored B row (ldb * 2)
};

B200_DEVINL uint32_t ld_acquire_gpu(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
B200_DEVINL void st_release_gpu(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
B200_DEVINL uint4 ld_peer_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.relaxed.sys.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}
// block until chunks [lo, hi] of the gathered buffer have been published for this epoch
B200_DEVINL void ag_wait_chunks(const AgParams& ag, unsigned long long byte_lo, unsigned long long byte_hi) {
  if (byte_lo < ag.begin) byte_lo = ag.begin;
  if (byte_hi > ag.end) byte_hi = ag.end;
  if (byte_hi <= byte_lo) return;
  const unsigned c0 = (unsigned)(byte_lo / AG_CHUNK), c1 = (unsigned)((byte_hi - 1) / AG_CHUNK);
  for (unsigned c = c0; c <= c1; ++c) {
    uint64_t t0 = 0;
    uint32_t spins = 0;
    while (ld_acquire_gpu(ag.flags + c) != ag.epoch) {
      if ((++spins & 0x3ff) == 0) {
        uint64_t now = global_timer_ns();
        if (t0 == 0) t0 = now;
        else if (now - t0 > B200_WAIT_TIMEOUT_NS) __trap();
      }
    }
  }
  asm volatile("fence.proxy.async;" ::: "memory");  // generic-proxy writes of the comm warps -> TMA (async proxy) reads
}

struct GemmParams {
  int M, N, K;          // C is [M,N], reduction length K
  int ldc, ldr;         // row strides (elements) of C and residual
  void* C;
  const void* R;        // residual (bf16) or nullptr
  int m_tiles, n_tiles;
  // batched mode (BATCH = true): nb0 x nb1 independent problems; operands come through rank-4 tensor maps
  // {inner, outer, b0, b1}; C of problem (b0, b1) starts at b0 * sc0 + b1 * sc1 elements
  int nb0, nb1;
  long long sc0, sc1;
  // EPI_ROPE (QKV projection): rotate adjacent column pairs of the first rope_cols columns by the angle of
  // (row % rope_S, (col % rope_hd) / 2) before the bf16 store; table is [S][hd/2][cos, sin] fp32 (SURVEY.md K2)
  // Grouped launches never rotate, so they keep the expert tables in the same slots: grp_tile = the plan's tile table,
  // grp_rows = weight rows per expert.
  union { const float* rope; const int* grp_tile; };
  union { int rope_S; int grp_rows; };
  int rope_hd, rope_cols;
  // EPI_PUSH (fused wgrad GEMM -> reduce-scatter, SURVEY.md N8): the wgrad tile is not stored to C but pushed over
  // NVLink into the staging buffer of the rank that OWNS that slice of the unit's flat gradient:
  //   e = push_off + row * ldc + col ; owner = e / push_n ; dst = push_bases[owner] + push_rank * push_n + (e - owner * push_n)
  void* const* push_bases;
  long long push_n, push_off;
  int push_rank;
  int push_bulk;        // 1: stage rows in shared memory, 128-byte bulk stores; 0: 4-byte stores from registers
  // every CTA starts its sweep `tile_rot` tiles into the raster (wraps around).  The push epilogue sets it to
  // rank * tiles / world so that the ranks, which run the same wgrad GEMM at the same time, write into different owners.
  int tile_rot;
  // EPI_SWIGLU (gate/up projection, nt): B is the fused [2F, K] weight.  A tile covers 64 features: accumulator columns
  // [0,64) come from rows [f0, f0+64) of the FIRST half of the weight and [64,128) from the same features of the SECOND
  // half, so every thread holds gate and up of the same feature: it stores the bf16 projection to C [M, 2F] (needed by
  // the backward) AND silu(gate) * up to aux [M, F].  N of the launch = F.
  // EPI_SWIGLU_BWD (down-projection dgrad, nn): the accumulator is dS [M, F]; the epilogue reads gate / up from
  // aux = the saved projection [M, 2F] and stores d(gate) | d(up) to C [M, 2F] -- dS itself never reaches memory.
  void* aux;
  int ld_aux, swi_F, swi_gate_first;
  // EPI_SCALE (fp8 e4m3 operands, FP8 = true): C = acc * scale_a[row] * scale_b[col].  GRP_K: grp_seg = the plan's
  // [start | len] of every expert.
  union { const float* scale_a; const int* grp_seg; };
  const float* scale_b;
};

B200_DEVINL void bulk_store_s2g(void* gdst, const void* ssrc, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
               ::"l"(gdst), "r"(smem_u32(ssrc)), "r"(bytes) : "memory");
}

// destination of element e of the unit's flat gradient in its owner's staging slot for this rank
B200_DEVINL __nv_bfloat16* push_dst(const GemmParams& p, long long e) {
  const long long owner = e / p.push_n;
  return reinterpret_cast<__nv_bfloat16*>(p.push_bases[owner]) + ((long long)p.push_rank * p.push_n + (e - owner * p.push_n));
}

B200_DEVINL float sigmoidf_fast(float x) { return __frcp_rn(1.f + exp2f(-1.4426950408889634f * x)); }

template <typename OutT>
B200_DEVINL void store2(OutT* p, float a, float b) {
  if constexpr (sizeof(OutT) == 2) *reinterpret_cast<uint32_t*>(p) = pack_bf16x2(a, b);
  else *reinterpret_cast<float2*>(p) = make_float2(a, b);
}
template <typename OutT>
B200_DEVINL float2 load2(const OutT* p) {
  if constexpr (sizeof(OutT) == 2) return unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p));
  else return *reinterpret_cast<const float2*>(p);
}

// Epilogue of one column pair (col, col + 1) of one row; col is even and N is a multiple of 8.
template <int EPI, typename OutT>
B200_DEVINL void epi_pair(const GemmParams& p, OutT* crow, int row, int col, float f0, float f1) {
  if constexpr (EPI == EPI_PUSH) {
    // made visible by the flag round that follows
    *reinterpret_cast<uint32_t*>(push_dst(p, p.push_off + (long long)row * p.ldc + col)) = pack_bf16x2(f0, f1);
    return;
  }
  if constexpr (EPI == EPI_SCALE) {
    const float sa = p.scale_a[row];
    const float2 sb = *reinterpret_cast<const float2*>(p.scale_b + col);
    f0 *= sa * sb.x; f1 *= sa * sb.y;
  } else if constexpr (EPI == EPI_ROPE) {
    if (col < p.rope_cols) {
      const float2 cs = *reinterpret_cast<const float2*>(
          p.rope + ((size_t)(row % p.rope_S) * (p.rope_hd >> 1) + ((col % p.rope_hd) >> 1)) * 2);
      const float a0 = f0, a1 = f1;
      f0 = a0 * cs.x - a1 * cs.y;
      f1 = a0 * cs.y + a1 * cs.x;
    }
  } else if constexpr (EPI == EPI_RESIDUAL) {
    const float2 r = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(
        reinterpret_cast<const __nv_bfloat16*>(p.R) + (size_t)row * p.ldr + col));
    f0 += r.x; f1 += r.y;
  } else if constexpr (EPI == EPI_ACCUM) {
    const float2 r = load2(crow + col);
    f0 += r.x; f1 += r.y;
  }
  store2(crow + col, f0, f1);
}

// Register epilogue of one consumer warpgroup's 64-row slice of a tile that is 8 * NJ columns wide (NJ = 16: 128x128
// kernel, 32: 128x256 kernel) in tile column nt.  The thread holds rows rbase and rbase + 8, column pairs 8 j + cq for
// j < NJ.  EPI_SWIGLU: the tile holds gate and up of 4 * NJ features side by side.
template <int EPI, typename OutT, int NJ>
B200_DEVINL void epilogue_tile(const GemmParams& p, const float (&acc)[4 * NJ], size_t boff, int rbase, int nt, int cq) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = rbase + 8 * h;
    if (row >= p.M) continue;
    OutT* crow = reinterpret_cast<OutT*>(p.C) + boff + static_cast<size_t>(row) * p.ldc;
    if constexpr (EPI == EPI_SWIGLU) {
      __nv_bfloat16* arow = reinterpret_cast<__nv_bfloat16*>(p.aux) + static_cast<size_t>(row) * p.ld_aux;
#pragma unroll
      for (int j = 0; j < NJ / 2; ++j) {
        const int col = nt * (4 * NJ) + 8 * j + cq;
        const uint32_t w1 = pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        const uint32_t w2 = pack_bf16x2(acc[4 * (j + NJ / 2) + 2 * h], acc[4 * (j + NJ / 2) + 2 * h + 1]);
        // activation from the ROUNDED projection: forward and backward see the same gate / up values
        const float2 x1 = unpack_bf16x2(w1), x2 = unpack_bf16x2(w2);
        const float2 gt = p.swi_gate_first ? x1 : x2, up = p.swi_gate_first ? x2 : x1;
        *reinterpret_cast<uint32_t*>(crow + col) = w1;
        *reinterpret_cast<uint32_t*>(crow + p.swi_F + col) = w2;
        *reinterpret_cast<uint32_t*>(arow + col) =
            pack_bf16x2(gt.x * sigmoidf_fast(gt.x) * up.x, gt.y * sigmoidf_fast(gt.y) * up.y);
      }
    } else if constexpr (EPI == EPI_SWIGLU_BWD) {
      const __nv_bfloat16* grow = reinterpret_cast<const __nv_bfloat16*>(p.aux) + static_cast<size_t>(row) * p.ld_aux;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int col = nt * (8 * NJ) + 8 * j + cq;
        if (col >= p.N) break;
        const float2 x1 = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(grow + col));
        const float2 x2 = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(grow + p.swi_F + col));
        const float2 gt = p.swi_gate_first ? x1 : x2, up = p.swi_gate_first ? x2 : x1;
        const float ds0 = acc[4 * j + 2 * h], ds1 = acc[4 * j + 2 * h + 1];
        const float s0 = sigmoidf_fast(gt.x), s1 = sigmoidf_fast(gt.y);
        const float dg0 = ds0 * up.x * s0 * (1.f + gt.x * (1.f - s0)), dg1 = ds1 * up.y * s1 * (1.f + gt.y * (1.f - s1));
        const float du0 = ds0 * gt.x * s0, du1 = ds1 * gt.y * s1;
        const uint32_t pg = pack_bf16x2(dg0, dg1), pu = pack_bf16x2(du0, du1);
        *reinterpret_cast<uint32_t*>(crow + col) = p.swi_gate_first ? pg : pu;
        *reinterpret_cast<uint32_t*>(crow + p.swi_F + col) = p.swi_gate_first ? pu : pg;
      }
    } else {
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int col = nt * (8 * NJ) + 8 * j + cq;
        if (col >= p.N) break;
        epi_pair<EPI, OutT>(p, crow, row, col, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      }
    }
  }
}

template <bool A_MN, bool B_MN, int EPI, typename OutT, bool AG, bool FP8 = false, bool BATCH = false>
__global__ void __launch_bounds__(THREADS, 1)
gemm_bf16_wgmma(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, GemmParams p,
                AgParams ag) {
  static_assert(!FP8 || (!A_MN && !B_MN && !AG && !BATCH), "fp8 operands: K-major (nt) only");
  constexpr int EP = EPI & EPI_MASK;                            // the epilogue
  constexpr bool GM = (EPI & GRP_M) != 0, GK = (EPI & GRP_K) != 0;
  static_assert(!(GM || GK) || (!AG && !FP8 && !BATCH && EP != EPI_PUSH), "grouped: no comm, fp8, batch or push");
  static_assert(!GK || (A_MN && B_MN), "k-grouped: wgrad (tn) only");
  constexpr int NST = ring_stages<EP>();
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B atoms must sit on 1024 B boundaries
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + NST * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + NST;
  uint8_t* push_stage = smem + NST * STAGE_BYTES + 256;     // EPI_PUSH only

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // elements per k-block: one 128-byte swizzle atom per row = 64 bf16 or 128 e4m3
  constexpr int BKE = FP8 ? 2 * BK : BK;
  const int num_kb = (p.K + BKE - 1) / BKE;
  const int tiles_per_problem = p.m_tiles * p.n_tiles;
  const int num_tiles = (BATCH || GK) ? tiles_per_problem * p.nb0 * p.nb1 : tiles_per_problem;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < NST; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);   // one arrive per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  auto coords = [&](int t, int& mt, int& nt, int& b0, int& b1) {
    b0 = b1 = 0;
    if constexpr (BATCH || GK) {
      const int prob = t / tiles_per_problem;
      b0 = prob % p.nb0; b1 = prob / p.nb0;
      tile_coords(t - prob * tiles_per_problem, p.m_tiles, p.n_tiles, mt, nt);
    } else {
      tile_coords((t + p.tile_rot) % num_tiles, p.m_tiles, p.n_tiles, mt, nt);
    }
  };
  // grouped modes: the expert of an m-tile (GRP_M, -1 = skip the tile) and the k-blocks of a problem (GRP_K)
  auto group = [&](int mt, int b0, int& e, int& kb0, int& kb1) {
    e = 0; kb0 = 0; kb1 = num_kb;
    if constexpr (GM) e = p.grp_tile[mt];
    if constexpr (GK) {
      const int s = p.grp_seg[b0];
      kb0 = s / BKE;
      kb1 = (s + p.grp_seg[p.nb0 + b0] + BKE - 1) / BKE;
    }
  };

  if (warp < 4) {
    if (warp == 0 && lane == 0) {
      // ============================== TMA producer ==============================
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        int mt, nt, b0, b1, e, kb0, kb1;
        coords(t, mt, nt, b0, b1);
        group(mt, b0, e, kb0, kb1);
        if (e < 0) continue;
        const int m0 = mt * BM;
        // GRP_M: the expert's slab of the weight rows -- B's rows (K-major) or k-rows (MN-major)
        const int bn = (GM && !B_MN) ? e * p.grp_rows : 0, bk = (GM && B_MN) ? e * p.grp_rows : 0;
        // B rows of the two 64-row halves of the tile (SwiGLU: the same features of both halves of the fused weight)
        const int n0 = ((EP == EPI_SWIGLU) ? nt * 64 : nt * BN) + bn;
        const int n1 = (EP == EPI_SWIGLU) ? n0 + p.swi_F : n0 + 64;
        auto load = [&](void* dst, const CUtensorMap* tm, int c0, int c1) {
          if constexpr (BATCH) tma_load_4d(dst, tm, &full_bar[stage], c0, c1, b0, b1);
          else tma_load_2d(dst, tm, &full_bar[stage], c0, c1);
        };
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          uint8_t* sb = sa + A_BYTES;
          const int k0 = kb * BKE;
          if constexpr (AG) {
            if (ag.dependent) {
              // stored rows of B under this tile: K-major -> rows [n0, n0+128) (once per tile); MN-major -> rows
              // [k0, k0+64) (every k-block)
              if constexpr (!B_MN) {
                if (kb == 0) ag_wait_chunks(ag, ag.b_off + (unsigned long long)n0 * ag.b_row_bytes,
                                            ag.b_off + (unsigned long long)min(n0 + BN, p.N) * ag.b_row_bytes);
              } else {
                ag_wait_chunks(ag, ag.b_off + (unsigned long long)k0 * ag.b_row_bytes,
                               ag.b_off + (unsigned long long)min(k0 + BK, p.K) * ag.b_row_bytes);
              }
            }
          }
          mbar_arrive_expect_tx(&full_bar[stage], STAGE_BYTES);
          if constexpr (!A_MN) {
            load(sa, &tmA, k0, m0);                                    // box {64 k, 128 rows}
          } else {
            load(sa, &tmA, m0, k0);                                    // boxes {64 m, 64 k-rows}
            load(sa + 64 * BK * 2, &tmA, m0 + 64, k0);
          }
          if constexpr (!B_MN) {
            load(sb, &tmB, k0, n0);                                    // boxes {64 k, 64 rows}
            load(sb + 64 * BK * 2, &tmB, k0, n1);
          } else {
            load(sb, &tmB, n0, k0 + bk);                               // boxes {64 n, 64 k-rows}
            load(sb + 64 * BK * 2, &tmB, n0 + 64, k0 + bk);
          }
          if (++stage == NST) { stage = 0; phase ^= 1; }
        }
      }
    } else if (AG && warp >= 2) {
      // ===================== comm warps: pull peer shards into the local gathered buffer =====================
      if constexpr (AG) {
        const int ct = (warp - 2) * 32 + lane;              // 0 .. 63
        const unsigned long long total = ag.end - ag.begin;
        const unsigned n_chunks = (unsigned)((total + AG_CHUNK - 1) / AG_CHUNK);
        const unsigned first = (unsigned)(ag.begin / AG_CHUNK);
        // rotate the start so the ranks do not all hit the same peer first
        const unsigned rot = (unsigned)(((unsigned long long)ag.rank * n_chunks) / (unsigned)ag.world);
        for (unsigned i = blockIdx.x; i < n_chunks; i += gridDim.x) {
          const unsigned ci = ag.dependent ? i : (i + rot) % n_chunks;   // dependent mode keeps B-first order
          const unsigned long long lo = ag.begin + (unsigned long long)ci * AG_CHUNK;
          const unsigned long long hi = (lo + AG_CHUNK < ag.end) ? lo + AG_CHUNK : ag.end;
          const unsigned nvec = (unsigned)((hi - lo) / 16);
          const unsigned src_lo = (unsigned)(lo / ag.shard_bytes), src_hi = (unsigned)((hi - 1) / ag.shard_bytes);
          const uint8_t* base_lo = reinterpret_cast<const uint8_t*>(ag.peer_shards[src_lo]) - (unsigned long long)src_lo * ag.shard_bytes;
          const uint8_t* base_hi = reinterpret_cast<const uint8_t*>(ag.peer_shards[src_hi]) - (unsigned long long)src_hi * ag.shard_bytes;
          const unsigned long long split = (unsigned long long)src_hi * ag.shard_bytes;  // a chunk spans <= 2 shards
          for (unsigned v0 = ct; v0 < nvec; v0 += 64 * 8) {
            uint4 buf[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
              const unsigned v = v0 + u * 64;
              if (v < nvec) {
                const unsigned long long off = lo + (unsigned long long)v * 16;
                buf[u] = ld_peer_v4(((src_lo != src_hi && off >= split) ? base_hi : base_lo) + off);
              }
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
              const unsigned v = v0 + u * 64;
              if (v < nvec) *reinterpret_cast<uint4*>(ag.full + lo + (unsigned long long)v * 16) = buf[u];
            }
          }
          __threadfence();
          named_bar_sync(2, 64);      // both comm warps finished this chunk
          if (ct == 0) {
            asm volatile("fence.proxy.async;" ::: "memory");
            st_release_gpu(ag.flags + first + ci, ag.epoch);
          }
        }
      }
    }
  } else {
    // ============================== consumers: wgmma + epilogue ==============================
    const int cw = (warp >> 2) - 1;          // consumer warpgroup: rows [64 cw, 64 cw + 64) of the tile
    const int w4 = warp & 3;
    int stage = 0;
    uint32_t phase = 0;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      int mt, nt, b0, b1, e, kb0, kb1;
      coords(t, mt, nt, b0, b1);
      group(mt, b0, e, kb0, kb1);
      if (e < 0) continue;
      float acc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES) + cw * (64 * 128);   // this warpgroup's 64 rows / box
        const uint32_t sb = smem_u32(smem + stage * STAGE_BYTES) + A_BYTES;
        const uint64_t a0 = make_smem_desc(sa, 0, 1024);
        const uint64_t bd0 = make_smem_desc(sb, B_MN ? 64 * BK * 2 : 0, 1024);
        wgmma_fence();
        if constexpr (FP8) {
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_e4m3_ss_n128(acc, a0 + ((k * 32) >> 4), bd0 + ((k * 32) >> 4), (kb | k) != 0);
        } else {
#pragma unroll
          for (int k = 0; k < BK / 16; ++k) {
            const uint64_t adesc = a0 + ((A_MN ? k * 2048 : k * 32) >> 4);
            const uint64_t bdesc = bd0 + ((B_MN ? k * 2048 : k * 32) >> 4);
            wgmma_bf16_ss_n128<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, adesc, bdesc, (kb | k) != 0);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();                     // the previous k-block's MMAs have retired: release its stage
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == NST) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);

      // ---- epilogue: thread holds rows r and r + 8, column pairs 8 j + 2 (lane & 3) for j = 0..15
      size_t boff = 0;
      if constexpr (BATCH || GK) boff = (size_t)b0 * p.sc0 + (size_t)b1 * p.sc1;
      const int rbase = mt * BM + cw * 64 + w4 * 16 + (lane >> 2);
      const int cq = 2 * (lane & 3);
      if constexpr (EP == EPI_PUSH) {
        if (p.push_bulk) {
          uint8_t* stg = push_stage + cw * 64 * PUSH_PITCH;
          asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // own bulk stores of the last tile have read
          named_bar_sync(3 + cw, 128);                                         // ... and so have everyone else's
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = w4 * 16 + (lane >> 2) + 8 * h;
#pragma unroll
            for (int j = 0; j < 16; ++j)
              *reinterpret_cast<uint32_t*>(stg + r * PUSH_PITCH + (8 * j + cq) * 2) =
                  pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
          }
          fence_proxy_async_smem();          // generic smem writes -> async-proxy (bulk copy) reads
          named_bar_sync(3 + cw, 128);
          // thread t of the warpgroup sends row t / 2, columns [64 (t & 1), 64 (t & 1) + 64)
          const int t = threadIdx.x & 127;
          const int row = mt * BM + cw * 64 + (t >> 1), col = nt * BN + 64 * (t & 1);
          if (row < p.M && col < p.N) {
            const uint8_t* src = stg + (t >> 1) * PUSH_PITCH + 128 * (t & 1);
            const int ncols = min(64, p.N - col);              // multiple of 8
            const long long e = p.push_off + (long long)row * p.ldc + col;
            if (ncols == 64 && (e & 63) == 0 && (p.push_n & 63) == 0) {
              bulk_store_s2g(push_dst(p, e), src, 128);
            } else {   // a chunk that may straddle two owners / a ragged right edge: one 16-byte store per vector
              for (int g = 0; g * 8 < ncols; ++g) bulk_store_s2g(push_dst(p, e + 8 * g), src + 16 * g, 16);
            }
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
          }
          continue;
        }
      }
      epilogue_tile<EP, OutT, BN / 8>(p, acc, boff, rbase, nt, cq);
    }
    if constexpr (EP == EPI_PUSH) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // every pushed row is out
  }
}

template <bool A_MN, bool B_MN, int EPI, typename OutT, bool AG, bool FP8 = false, bool BATCH = false>
static int launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, const AgParams& ag,
                  cudaStream_t stream) {
  auto kern = gemm_bf16_wgmma<A_MN, B_MN, EPI, OutT, AG, FP8, BATCH>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes<EPI>());
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  long long tiles = (long long)p.m_tiles * p.n_tiles * ((BATCH || (EPI & GRP_K)) ? (long long)p.nb0 * p.nb1 : 1);
  // the comm warps of ALL SMs carry the fused gather, so that launch always covers the full machine
  int grid = (!AG && tiles < sm_count()) ? (int)tiles : sm_count();
  if (grid < 1) grid = 1;
  kern<<<grid, THREADS, smem_bytes<EPI>(), stream>>>(tmA, tmB, p, ag);
  return (int)cudaGetLastError();
}

// ---- 128 x 256 tile ("wide"), for the GEMMs without fused communication.  The same pipeline with twice the B tile per
// stage: a k-block moves 48 KiB for 4.2 MFLOP (85 FLOP per byte from L2, against 64 for 128 x 128), and each consumer
// warpgroup issues m64n256k16, which reads 10 KiB of shared-memory operands per 524k FLOP where two m64n128k16 read
// 12 KiB.  A 64 x 256 fp32 accumulator is 128 registers per consumer thread, more than 384 threads get by default:
// setmaxnreg hands the producer warpgroup's registers to the consumers (128 x 40 + 256 x 232 <= 64K).
// Epilogues: store, +residual, accumulate (bf16 or fp32 output), RoPE, SwiGLU forward (F % 128 == 0) and backward.
constexpr int WBN = 256;
constexpr int W_STAGES = 4;
constexpr int W_STAGE_BYTES = A_BYTES + WBN * BK * 2;   // 16 + 32 KiB
constexpr int W_SMEM_BYTES = W_STAGES * W_STAGE_BYTES + 1024 + 256;

template <int N>
B200_DEVINL void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
B200_DEVINL void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

template <bool A_MN, bool B_MN, int EPI, typename OutT>
__global__ void __launch_bounds__(THREADS, 1)
gemm_wide_bf16(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + W_STAGES * W_STAGE_BYTES);
  uint64_t* empty_bar = full_bar + W_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_kb = (p.K + BK - 1) / BK;
  const int num_tiles = p.m_tiles * p.n_tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < W_STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);   // one arrive per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      // ============================== TMA producer ==============================
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        int mt, nt;
        tile_coords(t, p.m_tiles, p.n_tiles, mt, nt);
        const int m0 = mt * BM;
        // first B row (K-major) or column (MN-major) of the tile; SwiGLU: 128 features of the first half of the fused
        // weight in B rows [f0, f0 + 128), the same features of the second half in [F + f0, F + f0 + 128)
        const int n0 = (EPI == EPI_SWIGLU) ? nt * 128 : nt * WBN;
        const int n2 = (EPI == EPI_SWIGLU) ? n0 + p.swi_F : n0 + 128;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * W_STAGE_BYTES;
          uint8_t* sb = sa + A_BYTES;
          const int k0 = kb * BK;
          mbar_arrive_expect_tx(&full_bar[stage], W_STAGE_BYTES);
          if constexpr (!A_MN) {
            tma_load_2d(sa, &tmA, &full_bar[stage], k0, m0);                     // box {64 k, 128 rows}
          } else {
            tma_load_2d(sa, &tmA, &full_bar[stage], m0, k0);                     // boxes {64 m, 64 k-rows}
            tma_load_2d(sa + 64 * BK * 2, &tmA, &full_bar[stage], m0 + 64, k0);
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) {                                            // four 64-wide quarters of B
            const int nq = (q < 2 ? n0 : n2) + 64 * (q & 1);
            if constexpr (!B_MN) tma_load_2d(sb + q * 64 * BK * 2, &tmB, &full_bar[stage], k0, nq);
            else                 tma_load_2d(sb + q * 64 * BK * 2, &tmB, &full_bar[stage], nq, k0);
          }
          if (++stage == W_STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // ============================== consumers: wgmma + epilogue ==============================
    const int cw = (warp >> 2) - 1;          // consumer warpgroup: rows [64 cw, 64 cw + 64) of the tile
    const int w4 = warp & 3;
    int stage = 0;
    uint32_t phase = 0;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      int mt, nt;
      tile_coords(t, p.m_tiles, p.n_tiles, mt, nt);
      float acc[128];
#pragma unroll
      for (int i = 0; i < 128; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * W_STAGE_BYTES) + cw * (64 * 128);
        const uint32_t sb = smem_u32(smem + stage * W_STAGE_BYTES) + A_BYTES;
        const uint64_t a0 = make_smem_desc(sa, 0, 1024);
        const uint64_t bd0 = make_smem_desc(sb, B_MN ? 64 * BK * 2 : 0, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint64_t adesc = a0 + ((A_MN ? k * 2048 : k * 32) >> 4);
          const uint64_t bdesc = bd0 + ((B_MN ? k * 2048 : k * 32) >> 4);
          wgmma_bf16_ss_n256<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, adesc, bdesc, (kb | k) != 0);
        }
        wgmma_commit();
        wgmma_wait<1>();                     // the previous k-block's MMAs have retired: release its stage
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == W_STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      const int rbase = mt * BM + cw * 64 + w4 * 16 + (lane >> 2);
      epilogue_tile<EPI, OutT, WBN / 8>(p, acc, 0, rbase, nt, 2 * (lane & 3));
    }
  }
}

template <bool A_MN, bool B_MN, int EPI, typename OutT>
static int launch_wide(const CUtensorMap& tmA, const CUtensorMap& tmB, GemmParams p, cudaStream_t stream) {
  auto kern = gemm_wide_bf16<A_MN, B_MN, EPI, OutT>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, W_SMEM_BYTES);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  p.n_tiles = (EPI == EPI_SWIGLU) ? p.swi_F / 128 : (p.N + WBN - 1) / WBN;
  const long long tiles = (long long)p.m_tiles * p.n_tiles;
  const int grid = tiles < sm_count() ? (int)tiles : sm_count();
  kern<<<grid, THREADS, W_SMEM_BYTES, stream>>>(tmA, tmB, p);
  return (int)cudaGetLastError();
}

// 0: the launcher picks the tile; 1: always 128 x 128; 2: 128 x 256 wherever the epilogue allows it.  Set only by the
// GEMM benchmark and the tests, which compare the two tiles on the same operands.
static int g_tile_override = 0;

// The wide tile moves less data per FLOP but halves the tile count, so it wins unless it leaves a worse last wave:
// a persistent sweep takes about ceil(tiles / SMs) tile times, and a wide tile takes WIDE_TILE_COST / 16 of two narrow
// ones.
constexpr int WIDE_TILE_COST = 15;
static bool use_wide(const GemmParams& p, int epi) {
  if (g_tile_override == 1 || (epi == EPI_SWIGLU && p.swi_F % 128)) return false;
  if (g_tile_override == 2) return true;
  const long long sm = sm_count();
  const long long n_wide = (epi == EPI_SWIGLU) ? p.swi_F / 128 : (p.N + WBN - 1) / WBN;
  const long long waves_narrow = ((long long)p.m_tiles * p.n_tiles + sm - 1) / sm;
  const long long waves_wide = ((long long)p.m_tiles * n_wide + sm - 1) / sm;
  return 2 * WIDE_TILE_COST * waves_wide <= 16 * waves_narrow;
}

// every GEMM of the single-GPU path (no fused all-gather, no push): one launch of the tile use_wide picks
template <bool A_MN, bool B_MN, int EPI, typename OutT>
static int launch_local(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, cudaStream_t stream) {
  if (use_wide(p, EPI)) return launch_wide<A_MN, B_MN, EPI, OutT>(tmA, tmB, p, stream);
  return launch<A_MN, B_MN, EPI, OutT, false>(tmA, tmB, p, AgParams{}, stream);
}

template <bool A_MN, bool B_MN>
static int dispatch_epi(const CUtensorMap& a, const CUtensorMap& b, const GemmParams& p, int epi, int out_fp32,
                        cudaStream_t s) {
  if (out_fp32) {
    if (epi == EPI_STORE) return launch_local<A_MN, B_MN, EPI_STORE, float>(a, b, p, s);
    if (epi == EPI_RESIDUAL) return launch_local<A_MN, B_MN, EPI_RESIDUAL, float>(a, b, p, s);
    return launch_local<A_MN, B_MN, EPI_ACCUM, float>(a, b, p, s);
  }
  if (epi == EPI_STORE) return launch_local<A_MN, B_MN, EPI_STORE, __nv_bfloat16>(a, b, p, s);
  if (epi == EPI_RESIDUAL) return launch_local<A_MN, B_MN, EPI_RESIDUAL, __nv_bfloat16>(a, b, p, s);
  return launch_local<A_MN, B_MN, EPI_ACCUM, __nv_bfloat16>(a, b, p, s);
}

// batched dispatch: store / accumulate epilogues, bf16 or fp32 output
template <bool A_MN, bool B_MN>
static int dispatch_batched(const CUtensorMap& a, const CUtensorMap& b, const GemmParams& p, int epi, int out_fp32,
                            cudaStream_t s) {
  const AgParams ag{};
  if (out_fp32) {
    if (epi == EPI_ACCUM) return launch<A_MN, B_MN, EPI_ACCUM, float, false, false, true>(a, b, p, ag, s);
    return launch<A_MN, B_MN, EPI_STORE, float, false, false, true>(a, b, p, ag, s);
  }
  if (epi == EPI_ACCUM) return launch<A_MN, B_MN, EPI_ACCUM, __nv_bfloat16, false, false, true>(a, b, p, ag, s);
  return launch<A_MN, B_MN, EPI_STORE, __nv_bfloat16, false, false, true>(a, b, p, ag, s);
}

inline int make_tmap_4d_bf16(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer, uint64_t nb0, uint64_t nb1,
                             uint64_t ld, uint64_t s0, uint64_t s1, uint32_t box_inner, uint32_t box_outer) {
  uint64_t dims[4] = {inner, outer, nb0, nb1};
  uint64_t strides[3] = {ld * 2, s0 * 2, s1 * 2};
  uint32_t box[4] = {box_inner, box_outer, 1, 1};
  return make_tmap(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, ptr, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

// operand maps of one (unbatched) GEMM: K-major A box {64 k, 128 rows}, K-major B box {64 k, 64 rows},
// MN-major boxes {64 m|n, 64 k}
static int make_maps(CUtensorMap* tmA, CUtensorMap* tmB, const void* A, const void* B, int M, int N, int K, int lda,
                     int ldb, int a_mn, int b_mn) {
  int rc;
  if (!a_mn) rc = make_tmap_2d_bf16(tmA, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, BK, BM);
  else       rc = make_tmap_2d_bf16(tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, 64, BK);
  if (rc) return 1000 - rc;
  if (!b_mn) rc = make_tmap_2d_bf16(tmB, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb, BK, 64);
  else       rc = make_tmap_2d_bf16(tmB, B, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, 64, BK);
  if (rc) return 2000 - rc;
  return 0;
}

// RoPE epilogue parameters of the NEXT epi == EPI_ROPE launch (set immediately before it by the single host thread
// that owns the stream; keeps the launcher signatures unchanged)
static const float* g_rope_table = nullptr;
static int g_rope_S = 1, g_rope_hd = 2, g_rope_cols = 0;
// same convention for the push epilogue
static void* const* g_push_bases = nullptr;
static long long g_push_n = 1, g_push_off = 0;
static int g_push_rank = 0, g_push_bulk = 1, g_push_world = 1;
// same convention for the SwiGLU epilogues: aux = activation output (forward) / saved projection (backward)
static void* g_swi_aux = nullptr;
static int g_swi_ld = 0, g_swi_F = 0, g_swi_gate_first = 1;

static GemmParams make_params(void* C, const void* R, int M, int N, int K, int ldc, int ldr, int epi) {
  GemmParams p{};
  p.M = M; p.N = N; p.K = K; p.ldc = ldc; p.ldr = ldr; p.C = C; p.R = R;
  p.m_tiles = (M + BM - 1) / BM;
  p.n_tiles = (N + BN - 1) / BN;
  p.nb0 = p.nb1 = 1;
  p.rope = g_rope_table; p.rope_S = g_rope_S; p.rope_hd = g_rope_hd; p.rope_cols = g_rope_cols;
  p.push_bases = g_push_bases; p.push_n = g_push_n; p.push_off = g_push_off; p.push_rank = g_push_rank;
  p.push_bulk = g_push_bulk;
  p.aux = g_swi_aux; p.ld_aux = g_swi_ld; p.swi_F = g_swi_F; p.swi_gate_first = g_swi_gate_first;
  if (epi == EPI_PUSH && g_push_world > 1) {
    const int per_band = GROUP_M * p.n_tiles, tiles = p.m_tiles * p.n_tiles;
    const int bands = (tiles + per_band - 1) / per_band;
    p.tile_rot = (int)(((long long)(g_push_rank % g_push_world) * bands / g_push_world) * per_band) % tiles;
  }
  return p;
}

}  // namespace b200

extern "C" void b200_gemm2_set_rope(const float* table, int S, int hd, int cols) {
  b200::g_rope_table = table; b200::g_rope_S = S; b200::g_rope_hd = hd; b200::g_rope_cols = cols;
}

// world > 1: rotate the tile raster by rank * tiles / world (0 / 1 = no rotation).  bulk = 1: tiles are staged in shared
// memory and leave as 128-byte cp.async.bulk stores; 0: 4-byte stores straight from the accumulator registers.
extern "C" void b200_gemm2_set_push(void* const* bases, long long n, long long off, int rank, int bulk, int world) {
  b200::g_push_bases = bases; b200::g_push_n = n; b200::g_push_off = off; b200::g_push_rank = rank;
  b200::g_push_bulk = bulk ? 1 : 0;
  b200::g_push_world = world < 1 ? 1 : world;
}

extern "C" void b200_gemm2_set_swiglu(void* aux, int ld_aux, int F, int gate_first) {
  b200::g_swi_aux = aux; b200::g_swi_ld = ld_aux; b200::g_swi_F = F; b200::g_swi_gate_first = gate_first;
}

// tile of the single-GPU GEMMs: 0 = chosen per launch, 1 = 128 x 128, 2 = 128 x 256 where the epilogue allows it
extern "C" void b200_gemm2_set_tile(int mode) { b200::g_tile_override = (mode == 1 || mode == 2) ? mode : 0; }

// C[M,N] = op(A) op(B) (+R | +C | fused epilogue).  a_mn: A is stored [K,M] (M contiguous) else [M,K];  b_mn: B is
// stored [K,N] (N contiguous) else [N,K].  lda/ldb/ldc/ldr are row strides in elements.  Returns 0 or an error code.
extern "C" int b200_gemm2_bf16(const void* A, const void* B, void* C, const void* R, int M, int N, int K, int lda,
                               int ldb, int ldc, int ldr, int a_mn, int b_mn, int epi, int out_fp32,
                               cudaStream_t stream) {
  using namespace b200;
  CUtensorMap tmA, tmB;
  if (int rc = make_maps(&tmA, &tmB, A, B, M, N, K, lda, ldb, a_mn, b_mn)) return rc;
  GemmParams p = make_params(C, R, M, N, K, ldc, ldr, epi);
  if (epi == EPI_SWIGLU) {   // nt; N = 2F rows of the fused weight, tiles of 64 features
    if (a_mn || b_mn || out_fp32 || !p.aux || p.swi_F <= 0 || N != 2 * p.swi_F || (p.swi_F % 64) || (p.ld_aux % 8)) return -11;
    p.N = p.swi_F;
    p.n_tiles = p.swi_F / 64;
    return launch_local<false, false, EPI_SWIGLU, __nv_bfloat16>(tmA, tmB, p, stream);
  }
  if (epi == EPI_SWIGLU_BWD) {   // nn; N = F columns of dS, output [M, 2F]
    if (a_mn || !b_mn || out_fp32 || !p.aux || p.swi_F != N || (N % 8) || (p.ld_aux % 8)) return -12;
    return launch_local<false, true, EPI_SWIGLU_BWD, __nv_bfloat16>(tmA, tmB, p, stream);
  }
  if (epi == EPI_ROPE) {
    if (a_mn || b_mn || out_fp32 || !p.rope || (p.rope_hd % 8) || (p.rope_cols % 8)) return -8;
    return launch_local<false, false, EPI_ROPE, __nv_bfloat16>(tmA, tmB, p, stream);
  }
  if (epi == EPI_PUSH) {   // wgrad (tn) only; every 8-element vector must stay inside one owner's slice
    if (!a_mn || !b_mn || out_fp32 || !p.push_bases || p.push_n <= 0 || (p.push_n % 8) || (p.push_off % 8) || (ldc % 8))
      return -9;
    return launch<true, true, EPI_PUSH, __nv_bfloat16, false>(tmA, tmB, p, AgParams{}, stream);
  }
  if (a_mn) {
    if (b_mn) return dispatch_epi<true, true>(tmA, tmB, p, epi, out_fp32, stream);
    return dispatch_epi<true, false>(tmA, tmB, p, epi, out_fp32, stream);
  }
  if (b_mn) return dispatch_epi<false, true>(tmA, tmB, p, epi, out_fp32, stream);
  return dispatch_epi<false, false>(tmA, tmB, p, epi, out_fp32, stream);
}

// store / residual / accumulate epilogues only (the small-M path of the bindings)
extern "C" int b200_gemm_bf16(const void* A, const void* B, void* C, const void* R, int M, int N, int K, int lda,
                              int ldb, int ldc, int ldr, int a_mn, int b_mn, int epi, int out_fp32,
                              cudaStream_t stream) {
  if (epi < 0 || epi > 2) return -10;
  return b200_gemm2_bf16(A, B, C, R, M, N, K, lda, ldb, ldc, ldr, a_mn, b_mn, epi, out_fp32, stream);
}

// Batched C[b0,b1] = op(A[b0,b1]) op(B[b0,b1]) (+C): nb0 x nb1 problems of identical shape; sa*/sb*/sc* are the element
// strides of the two batch indices (each a multiple of 8 elements; use any valid stride when the count is 1).
extern "C" int b200_bgemm_bf16(const void* A, const void* B, void* C, int M, int N, int K, int lda, int ldb, int ldc,
                               int nb0, int nb1, long long sa0, long long sa1, long long sb0, long long sb1,
                               long long sc0, long long sc1, int a_mn, int b_mn, int epi, int out_fp32,
                               cudaStream_t stream) {
  using namespace b200;
  if (epi != EPI_STORE && epi != EPI_ACCUM) return -1;
  CUtensorMap tmA, tmB;
  int rc;
  if (!a_mn) rc = make_tmap_4d_bf16(&tmA, A, K, M, nb0, nb1, lda, sa0, sa1, BK, BM);
  else       rc = make_tmap_4d_bf16(&tmA, A, M, K, nb0, nb1, lda, sa0, sa1, 64, BK);
  if (rc) return 1000 - rc;
  if (!b_mn) rc = make_tmap_4d_bf16(&tmB, B, K, N, nb0, nb1, ldb, sb0, sb1, BK, 64);
  else       rc = make_tmap_4d_bf16(&tmB, B, N, K, nb0, nb1, ldb, sb0, sb1, 64, BK);
  if (rc) return 2000 - rc;
  GemmParams p{};
  p.M = M; p.N = N; p.K = K; p.ldc = ldc; p.C = C;
  p.m_tiles = (M + BM - 1) / BM;
  p.n_tiles = (N + BN - 1) / BN;
  p.nb0 = nb0; p.nb1 = nb1; p.sc0 = sc0; p.sc1 = sc1;
  if (a_mn) {
    if (b_mn) return dispatch_batched<true, true>(tmA, tmB, p, epi, out_fp32, stream);
    return dispatch_batched<true, false>(tmA, tmB, p, epi, out_fp32, stream);
  }
  if (b_mn) return dispatch_batched<false, true>(tmA, tmB, p, epi, out_fp32, stream);
  return dispatch_batched<false, false>(tmA, tmB, p, epi, out_fp32, stream);
}

// Grouped GEMM over the expert-sorted rows of csrc/moe.cu, 128 x 128 tiles.  tile / seg: the plan's tile table and
// [start | len] of the E experts; Mpad: rows of the permuted buffer (a multiple of 128).  lda / ldb / ldc: row strides.
//   layout 0 (nt, GRP_M): C[Mpad, N] = A[Mpad, K] W_e[N, K]^T, B = W [E N, K].  epi store, or SwiGLU (N = 2F rows of
//                  the expert's fused [gate | up]; C = the projection [Mpad, 2F], aux = silu(gate) up [Mpad, F])
//   layout 1 (nn, GRP_M): C[Mpad, N] = A[Mpad, K] W_e[K, N], B = W [E K, N].  epi store, or SwiGLU backward (C = the
//                  projection's gradient [Mpad, 2N], aux = the projection)
//   layout 2 (tn, GRP_K): C[e] = A_e^T B_e [M, N] over the rows of expert e, A [Mpad, M], B [Mpad, N], C [E, M, N]
//                  contiguous.  epi store or accumulate, bf16 or fp32 output.
extern "C" int b200_gemm_grouped_bf16(const void* A, const void* B, void* C, const int* tile, const int* seg, int E,
                                      int Mpad, int M, int N, int K, int lda, int ldb, int ldc, int layout, int epi,
                                      int out_fp32, cudaStream_t stream) {
  using namespace b200;
  if (E < 1 || Mpad % BM || (N % 8) || (K % 8) || (M % 8)) return -14;
  CUtensorMap tmA, tmB;
  const AgParams ag{};
  if (layout == 2) {
    if (epi != EPI_STORE && epi != EPI_ACCUM) return -14;
    if (make_tmap_2d_bf16(&tmA, A, (uint64_t)M, (uint64_t)Mpad, (uint64_t)lda, 64, BK)) return 1001;
    if (make_tmap_2d_bf16(&tmB, B, (uint64_t)N, (uint64_t)Mpad, (uint64_t)ldb, 64, BK)) return 2001;
    GemmParams p = make_params(C, nullptr, M, N, Mpad, ldc, 0, epi);
    p.nb0 = E; p.nb1 = 1; p.sc0 = (long long)M * N; p.sc1 = 0;
    p.grp_seg = seg;
    constexpr int G = GRP_K;
    if (out_fp32) {
      if (epi == EPI_ACCUM) return launch<true, true, G | EPI_ACCUM, float, false>(tmA, tmB, p, ag, stream);
      return launch<true, true, G | EPI_STORE, float, false>(tmA, tmB, p, ag, stream);
    }
    if (epi == EPI_ACCUM) return launch<true, true, G | EPI_ACCUM, __nv_bfloat16, false>(tmA, tmB, p, ag, stream);
    return launch<true, true, G | EPI_STORE, __nv_bfloat16, false>(tmA, tmB, p, ag, stream);
  }
  if (out_fp32 || M != Mpad) return -14;
  if (make_tmap_2d_bf16(&tmA, A, (uint64_t)K, (uint64_t)Mpad, (uint64_t)lda, BK, BM)) return 1001;
  GemmParams p = make_params(C, nullptr, Mpad, N, K, ldc, 0, epi);
  p.grp_tile = tile;
  constexpr int G = GRP_M;
  if (layout == 0) {
    if (make_tmap_2d_bf16(&tmB, B, (uint64_t)K, (uint64_t)E * N, (uint64_t)ldb, BK, 64)) return 2001;
    p.grp_rows = N;
    if (epi == EPI_SWIGLU) {
      if (!p.aux || p.swi_F <= 0 || N != 2 * p.swi_F || (p.swi_F % 64) || (p.ld_aux % 8)) return -11;
      p.N = p.swi_F;
      p.n_tiles = p.swi_F / 64;
      return launch<false, false, G | EPI_SWIGLU, __nv_bfloat16, false>(tmA, tmB, p, ag, stream);
    }
    if (epi != EPI_STORE) return -14;
    return launch<false, false, G | EPI_STORE, __nv_bfloat16, false>(tmA, tmB, p, ag, stream);
  }
  if (layout != 1) return -14;
  if (make_tmap_2d_bf16(&tmB, B, (uint64_t)N, (uint64_t)E * K, (uint64_t)ldb, 64, BK)) return 2001;
  p.grp_rows = K;
  if (epi == EPI_SWIGLU_BWD) {
    if (!p.aux || p.swi_F != N || (p.ld_aux % 8)) return -12;
    return launch<false, true, G | EPI_SWIGLU_BWD, __nv_bfloat16, false>(tmA, tmB, p, ag, stream);
  }
  if (epi != EPI_STORE) return -14;
  return launch<false, true, G | EPI_STORE, __nv_bfloat16, false>(tmA, tmB, p, ag, stream);
}

// GEMM + fused all-gather.  Supported: bf16 output, EPI store|residual|rope|swiglu (nt), store|residual|swiglu_bwd (nn),
// store|accumulate|push (tn).
extern "C" int b200_gemm2_ag_bf16(const void* A, const void* B, void* C, const void* R, int M, int N, int K, int lda,
                                  int ldb, int ldc, int ldr, int a_mn, int b_mn, int epi,
                                  const void* const* peer_shards, void* full, unsigned long long shard_bytes,
                                  unsigned long long begin, unsigned long long end, int world, int rank,
                                  uint32_t* flags, uint32_t epoch, int dependent, cudaStream_t stream) {
  using namespace b200;
  if ((begin % 16) || (end % 16) || (begin % AG_CHUNK)) return -5;
  CUtensorMap tmA, tmB;
  if (int rc = make_maps(&tmA, &tmB, A, B, M, N, K, lda, ldb, a_mn, b_mn)) return rc;
  GemmParams p = make_params(C, R, M, N, K, ldc, ldr, epi);
  if (epi == EPI_SWIGLU) {
    if (a_mn || b_mn || !p.aux || p.swi_F <= 0 || N != 2 * p.swi_F || (p.swi_F % 64) || (p.ld_aux % 8) || dependent) return -11;
    p.N = p.swi_F;
    p.n_tiles = p.swi_F / 64;
  }
  if (epi == EPI_SWIGLU_BWD && (a_mn || !b_mn || !p.aux || p.swi_F != N || (N % 8) || (p.ld_aux % 8))) return -12;
  AgParams ag;
  ag.peer_shards = peer_shards; ag.full = (uint8_t*)full; ag.shard_bytes = shard_bytes; ag.begin = begin; ag.end = end;
  ag.world = world; ag.rank = rank; ag.flags = flags; ag.epoch = epoch; ag.dependent = dependent;
  ag.b_off = (unsigned long long)((const uint8_t*)B - (const uint8_t*)full);
  ag.b_row_bytes = (unsigned long long)ldb * 2;
  if (dependent && ((const uint8_t*)B < (const uint8_t*)full)) return -6;
#define AGL(AM, BM_, E) return launch<AM, BM_, E, __nv_bfloat16, true>(tmA, tmB, p, ag, stream)
  if (epi == EPI_ROPE) {
    if (a_mn || b_mn || !p.rope || (p.rope_hd % 8) || (p.rope_cols % 8)) return -8;
    AGL(false, false, EPI_ROPE);
  }
  if (!a_mn && !b_mn) {
    if (epi == EPI_SWIGLU) AGL(false, false, EPI_SWIGLU);
    if (epi == EPI_RESIDUAL) AGL(false, false, EPI_RESIDUAL);
    AGL(false, false, EPI_STORE);
  }
  if (!a_mn && b_mn) {
    if (epi == EPI_SWIGLU_BWD) AGL(false, true, EPI_SWIGLU_BWD);
    if (epi == EPI_RESIDUAL) AGL(false, true, EPI_RESIDUAL);
    AGL(false, true, EPI_STORE);
  }
  if (a_mn && b_mn) {
    if (epi == EPI_PUSH) {   // wgrad that pushes its tiles to the owners AND carries the next unit's all-gather
      if (!p.push_bases || p.push_n <= 0 || (p.push_n % 8) || (p.push_off % 8) || (ldc % 8)) return -9;
      AGL(true, true, EPI_PUSH);
    }
    if (epi == EPI_ACCUM) AGL(true, true, EPI_ACCUM);
    AGL(true, true, EPI_STORE);
  }
#undef AGL
  return -7;
}

// C[M, N] (bf16) = (A_q[M, K] x B_q[N, K]^T) * scale_a[M] * scale_b[N]  with e4m3 operands on the tensor cores
// (wgmma e4m3, fp32 accumulate).  K (bytes = elements) must be a multiple of 16; rows 16-byte aligned.
extern "C" int b200_gemm2_fp8(const void* A, const void* B, void* C, const float* scale_a, const float* scale_b, int M, int N,
                              int K, int lda, int ldb, int ldc, cudaStream_t stream) {
  using namespace b200;
  if ((K % 16) || (lda % 16) || (ldb % 16) || (N % 8) || (ldc % 8) || M < 1) return -13;
  CUtensorMap tmA, tmB;
  if (make_tmap_2d_u8(&tmA, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, 2 * BK, BM)) return 1001;
  if (make_tmap_2d_u8(&tmB, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb, 2 * BK, 64)) return 2001;
  GemmParams p{};
  p.M = M; p.N = N; p.K = K; p.ldc = ldc; p.C = C;
  p.m_tiles = (M + BM - 1) / BM;
  p.n_tiles = (N + BN - 1) / BN;
  p.nb0 = p.nb1 = 1;
  p.scale_a = scale_a; p.scale_b = scale_b;
  return launch<false, false, EPI_SCALE, __nv_bfloat16, false, true>(tmA, tmB, p, AgParams{}, stream);
}
