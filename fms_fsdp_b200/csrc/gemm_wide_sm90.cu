// The 128 x 256 GEMM tile: the pipeline of the 128 x 128 kernel in csrc/gemm_sm90.cu with twice the B tile per stage,
// and an epilogue staged in shared memory.  The launcher in gemm_sm90.cu calls b200_gemm_wide_staged for the 128 x 256
// GEMMs whose operands TMA can describe; the others run on the 128 x 128 tile.
//
// A k-block moves 48 KiB for 4.2 MFLOP (85 FLOP per byte from L2, against 64 for 128 x 128), and each consumer
// warpgroup issues m64n256k16, which reads 10 KiB of shared-memory operands per 524k FLOP where two m64n128k16 read
// 12 KiB.  A 64 x 256 fp32 accumulator is 128 registers per consumer thread, more than 384 threads get by default:
// setmaxnreg hands the producer warpgroup's registers to the consumers (128 x 40 + 256 x 232 <= 64K).
//
// Each consumer warpgroup walks its 64 x 256 slice in 32-column subtiles, writes each result block ("slab", 64 rows x
// 32 columns of one output) into a swizzled staging buffer and one thread sends it with a TMA tensor store, which clips
// at the M and N edges.  The epilogue operands (residual, the C that is accumulated into, the saved SwiGLU projection)
// arrive by TMA loads into the same slabs, the first ones while the main loop's last k-blocks run and the next ones
// while a subtile is computed; each result is written in place over its operand.  The arithmetic per element is that
// of epi_pair / epilogue_tile in gemm_sm90.cu, so both tiles give the same bits.
// Epilogues: store, +residual (bf16 output), accumulate (bf16 or fp32 output), RoPE (with or without bias), SwiGLU
// forward (F % 128 == 0) and backward.
#include "common.cuh"
#include "gemm_sm90.cuh"
#include "tensormap.h"
#include "wgmma.cuh"

namespace b200 {

constexpr int W_STAGES = 4;
constexpr int W_STAGE_BYTES = A_BYTES + WBN * BK * 2;   // 16 + 32 KiB
constexpr int W_SUB = 32;                               // columns per epilogue subtile
constexpr int W_STG_BYTES = 16384;                      // epilogue staging per consumer warpgroup
constexpr int W_SMEM_BYTES = W_STAGES * W_STAGE_BYTES + 2 * W_STG_BYTES + 1024 + 256;
constexpr int W_PREFETCH_KB = 4;                        // k-blocks before the end of the main loop: operand loads

// Staging plan of one epilogue.  A slab is one 64 x 32 block of one output (or operand) in shared memory: 64-byte
// rows with the 64-byte swizzle for bf16, 128-byte rows with the 128-byte swizzle for fp32, so the fragment writes of
// a warp (8 rows, 16 bytes each) hit 8 different bank groups.
template <int EPI, typename OutT>
struct WideEpi {
  static constexpr int SLAB = 64 * W_SUB * (int)sizeof(OutT);
  static constexpr int NSLAB = W_STG_BYTES / SLAB;
  // slabs per subtile: SwiGLU forward writes gate, up and the activation; backward reads and writes gate and up
  static constexpr int P = EPI == EPI_SWIGLU ? 3 : EPI == EPI_SWIGLU_BWD ? 2 : 1;
  static constexpr bool LOADS = EPI == EPI_RESIDUAL || EPI == EPI_ACCUM || EPI == EPI_SWIGLU_BWD;
  static constexpr int D = NSLAB / P;                                      // subtiles resident at once
  static constexpr int NSUB = (EPI == EPI_SWIGLU ? 128 : WBN) / W_SUB;     // SwiGLU: 128 features per tile
  static_assert(!(EPI == EPI_RESIDUAL && sizeof(OutT) == 4), "fp32 +residual runs on the 128 x 128 tile");
  static_assert(!LOADS || (D >= 2 && NSUB % D == 0), "operand slabs: double-buffered, fixed slot per subtile");
};

// Output / operand tensor maps of the wide epilogue, box {32 columns, 64 rows}:
//   c: C (SwiGLU forward and backward: its first F columns), c2: C's second F columns (SwiGLU),
//   x: the residual (+residual), the activation output aux (SwiGLU forward), the gate|up projection's first F columns
//   (SwiGLU backward), x2: its second F columns (SwiGLU backward).
struct WideEpiMaps {
  CUtensorMap c, c2, x, x2;
};

template <int N>
B200_DEVINL void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
B200_DEVINL void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// byte offset of element (r, c) in a slab
template <typename OutT>
B200_DEVINL uint32_t slab_off(int r, int c) {
  const uint32_t o = (uint32_t)(r * W_SUB + c) * (uint32_t)sizeof(OutT);
  return sizeof(OutT) == 4 ? o ^ ((o >> 3) & 0x70) : o ^ ((o >> 3) & 0x30);
}


template <bool A_MN, bool B_MN, int EPI, typename OutT>
__global__ void __launch_bounds__(THREADS, 1)
gemm_wide_staged_bf16(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ WideEpiMaps em, GemmParams p) {
  using E = WideEpi<EPI, OutT>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* stg = smem + W_STAGES * W_STAGE_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(stg + 2 * W_STG_BYTES);
  uint64_t* empty_bar = full_bar + W_STAGES;
  uint64_t* ld_bar = empty_bar + W_STAGES;   // [consumer warpgroup][subtile slot]: operand slabs landed

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_kb = (p.K + BK - 1) / BK;
  const int num_tiles = p.m_tiles * p.n_tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&em.c);
    for (int s = 0; s < W_STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);   // one arrive per consumer warp
    }
    for (int s = 0; s < 8; ++s) mbar_init(&ld_bar[s], 1);
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
    const bool leader = (threadIdx.x & 127) == 0;   // issues this warpgroup's epilogue loads and stores
    uint8_t* wstg = stg + cw * W_STG_BYTES;
    uint64_t* wbar = ld_bar + 4 * cw;
    uint32_t ld_par = 0;                     // bit k: parity of the next completion of wbar[k]
    int q = 0;                               // store-only epilogues: next slab of the staging ring
    const int r0 = w4 * 16 + (lane >> 2);    // this thread's rows r0 and r0 + 8 of the warpgroup's slice
    const int cq = 2 * (lane & 3);
    const int kb_pref = num_kb > W_PREFETCH_KB ? num_kb - W_PREFETCH_KB : 0;
    // output columns of the tile: SwiGLU forward counts features (its tile holds 128 of them)
    const int ncols = (EPI == EPI_SWIGLU) ? p.swi_F : p.N;
    int stage = 0;
    uint32_t phase = 0;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      int mt, nt;
      tile_coords(t, p.m_tiles, p.n_tiles, mt, nt);
      const int row0 = mt * BM + cw * 64;
      const int col0 = nt * ((EPI == EPI_SWIGLU) ? 128 : WBN);
      auto live = [&](int s) { return row0 < p.M && col0 + s * W_SUB < ncols; };
      // operand slabs of subtile s -> slot s % D
      auto load_sub = [&](int s) {
        uint8_t* dst = wstg + (s % E::D) * E::P * E::SLAB;
        uint64_t* bar = &wbar[s % E::D];
        const int c = col0 + s * W_SUB;
        mbar_arrive_expect_tx(bar, E::P * E::SLAB);
        if constexpr (EPI == EPI_RESIDUAL) tma_load_2d(dst, &em.x, bar, c, row0);
        if constexpr (EPI == EPI_ACCUM) tma_load_2d(dst, &em.c, bar, c, row0);
        if constexpr (EPI == EPI_SWIGLU_BWD) {
          tma_load_2d(dst, &em.x, bar, c, row0);
          tma_load_2d(dst + E::SLAB, &em.x2, bar, c, row0);
        }
      };
      float acc[128];
#pragma unroll
      for (int i = 0; i < 128; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        if constexpr (E::LOADS) {
          if (kb == kb_pref && leader) {
            tma_store_wait_read<0>();          // the last tile's stores have left the staging buffer
            for (int s = 0; s < E::D - 1; ++s)
              if (live(s)) load_sub(s);
          }
        }
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

      // RoPE: table row of each of the thread's two rows (one division per row), and the column's offset in its head,
      // advanced by 8 per column pair group in the order the table entries are fetched
      uint32_t trow[2] = {0, 0};
      int hcol = 0;
      float2 cs[2][4];
      auto fetch_rope = [&](float2 (&c)[2][4]) {
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          // hcol >> 1 < hd / 2 and the row is in the table for every column: the loads are in bounds
          c[0][jj] = reinterpret_cast<const float2*>(p.rope)[trow[0] + (hcol >> 1)];
          c[1][jj] = reinterpret_cast<const float2*>(p.rope)[trow[1] + (hcol >> 1)];
          hcol += 8;
          if (hcol >= p.rope_hd) hcol -= p.rope_hd;
        }
      };
      if constexpr (EPI == EPI_ROPE || EPI == EPI_ROPE_BIAS) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
          trow[h] = (uint32_t)((row0 + r0 + 8 * h) % p.rope_S) * (uint32_t)(p.rope_hd >> 1);
        hcol = (col0 + cq) % p.rope_hd;
        fetch_rope(cs);
      }

#pragma unroll
      for (int s = 0; s < E::NSUB; ++s) {
        const bool on = live(s);
        uint8_t* sl;                         // the subtile's first slab
        if constexpr (E::LOADS) {
          if (leader) {
            tma_store_wait_read<0>();        // the previous subtile's slabs have been read out
            if (s + E::D - 1 < E::NSUB && live(s + E::D - 1)) load_sub(s + E::D - 1);
          }
          sl = wstg + (s % E::D) * E::P * E::SLAB;
          if (on) {
            mbar_wait(&wbar[s % E::D], (ld_par >> (s % E::D)) & 1);
            ld_par ^= 1u << (s % E::D);
          }
        } else {
          if (leader) tma_store_wait_read<E::NSLAB - E::P>();   // the P slabs this subtile writes have been read out
          named_bar_sync(1 + cw, 128);
          sl = wstg + q * E::SLAB;
        }
        if (on) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = r0 + 8 * h;
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int j = 4 * s + jj;
              const uint32_t o = slab_off<OutT>(r, 8 * jj + cq);
              if constexpr (EPI == EPI_SWIGLU) {
                uint8_t* s1 = wstg + ((q + 1) % E::NSLAB) * E::SLAB;
                uint8_t* s2 = wstg + ((q + 2) % E::NSLAB) * E::SLAB;
                const uint32_t w1 = pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
                const uint32_t w2 = pack_bf16x2(acc[4 * (j + 16) + 2 * h], acc[4 * (j + 16) + 2 * h + 1]);
                // activation from the ROUNDED projection: forward and backward see the same gate / up values
                const float2 x1 = unpack_bf16x2(w1), x2 = unpack_bf16x2(w2);
                const float2 gt = p.swi_gate_first ? x1 : x2, up = p.swi_gate_first ? x2 : x1;
                *reinterpret_cast<uint32_t*>(sl + o) = w1;
                *reinterpret_cast<uint32_t*>(s1 + o) = w2;
                *reinterpret_cast<uint32_t*>(s2 + o) =
                    pack_bf16x2(gt.x * sigmoidf_fast(gt.x) * up.x, gt.y * sigmoidf_fast(gt.y) * up.y);
              } else if constexpr (EPI == EPI_SWIGLU_BWD) {
                uint32_t* lo = reinterpret_cast<uint32_t*>(sl + o);
                uint32_t* hi = reinterpret_cast<uint32_t*>(sl + E::SLAB + o);
                const float2 x1 = unpack_bf16x2(*lo), x2 = unpack_bf16x2(*hi);
                const float2 gt = p.swi_gate_first ? x1 : x2, up = p.swi_gate_first ? x2 : x1;
                const float ds0 = acc[4 * j + 2 * h], ds1 = acc[4 * j + 2 * h + 1];
                const float s0 = sigmoidf_fast(gt.x), s1 = sigmoidf_fast(gt.y);
                const float dg0 = ds0 * up.x * s0 * (1.f + gt.x * (1.f - s0)), dg1 = ds1 * up.y * s1 * (1.f + gt.y * (1.f - s1));
                const float du0 = ds0 * gt.x * s0, du1 = ds1 * gt.y * s1;
                const uint32_t pg = pack_bf16x2(dg0, dg1), pu = pack_bf16x2(du0, du1);
                *lo = p.swi_gate_first ? pg : pu;
                *hi = p.swi_gate_first ? pu : pg;
              } else {
                float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
                OutT* e = reinterpret_cast<OutT*>(sl + o);
                if constexpr (EPI == EPI_ROPE || EPI == EPI_ROPE_BIAS) {
                  if constexpr (EPI == EPI_ROPE_BIAS) {   // the bias is [N]: a few KiB that stay in L1
                    const int col = col0 + s * W_SUB + 8 * jj + cq;
                    const float2 b =
                        unpack_bf16x2(col < p.N ? *reinterpret_cast<const uint32_t*>(p.bias + col) : 0u);
                    f0 += b.x; f1 += b.y;
                  }
                  if (col0 + s * W_SUB + 8 * jj + cq < p.rope_cols) {
                    const float a0 = f0, a1 = f1;
                    f0 = a0 * cs[h][jj].x - a1 * cs[h][jj].y;
                    f1 = a0 * cs[h][jj].y + a1 * cs[h][jj].x;
                  }
                } else if constexpr (EPI == EPI_RESIDUAL) {
                  const float2 rr = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(e));
                  f0 += rr.x; f1 += rr.y;
                } else if constexpr (EPI == EPI_ACCUM) {
                  const float2 rr = load2(e);
                  f0 += rr.x; f1 += rr.y;
                }
                store2(e, f0, f1);
              }
            }
          }
        }
        // the next subtile's table entries travel while this one is fenced, synchronised and sent
        if constexpr (EPI == EPI_ROPE || EPI == EPI_ROPE_BIAS) {
          if (s + 1 < E::NSUB) fetch_rope(cs);
        }
        fence_proxy_async_smem();            // generic-proxy slab writes -> TMA store reads
        named_bar_sync(1 + cw, 128);
        // bulk groups: one per slab for the store-only epilogues (their waits count slabs), one per subtile for the
        // others (they wait for all); committed whether or not the subtile is inside C
        if (leader) {
          const int c = col0 + s * W_SUB;
          if constexpr (EPI == EPI_SWIGLU) {
            if (on) tma_store_2d(&em.c, sl, c, row0);
            tma_store_commit();
            if (on) tma_store_2d(&em.c2, wstg + ((q + 1) % E::NSLAB) * E::SLAB, c, row0);
            tma_store_commit();
            if (on) tma_store_2d(&em.x, wstg + ((q + 2) % E::NSLAB) * E::SLAB, c, row0);
            tma_store_commit();
          } else if constexpr (EPI == EPI_SWIGLU_BWD) {
            if (on) {
              tma_store_2d(&em.c, sl, c, row0);
              tma_store_2d(&em.c2, sl + E::SLAB, c, row0);
            }
            tma_store_commit();
          } else {
            if (on) tma_store_2d(&em.c, sl, c, row0);
            tma_store_commit();
          }
        }
        if constexpr (!E::LOADS) q = (q + E::P) % E::NSLAB;
      }
    }
    if (leader) tma_store_wait<0>();         // every store has completed before the CTA exits
  }
}

// map of a [rows, cols] block of a row-major matrix for the wide epilogue: box {32 columns, 64 rows}, the slab swizzle
static int make_epi_map(CUtensorMap* m, const void* ptr, int cols, int rows, int ld, bool fp32) {
  const uint64_t dims[2] = {(uint64_t)cols, (uint64_t)rows};
  const uint64_t strides[1] = {(uint64_t)ld * (fp32 ? 4 : 2)};
  const uint32_t box[2] = {W_SUB, 64};
  return make_tmap(m, fp32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, ptr, dims, strides,
                   box, fp32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B);
}

// TMA needs 16-byte aligned bases and row strides; a stride below the row length (a broadcast residual) cannot be
// described either.  Such GEMMs run on the 128 x 128 tile.
static bool staged_ok(const GemmParams& p, int epi, int out_bytes) {
  auto ok = [](const void* ptr, long long ld, int cols, int eb) {
    return reinterpret_cast<uintptr_t>(ptr) % 16 == 0 && (ld * eb) % 16 == 0 && ld >= cols;
  };
  if (epi == EPI_SWIGLU || epi == EPI_SWIGLU_BWD)
    return ok(p.C, p.ldc, 2 * p.swi_F, 2) && ok(p.aux, p.ld_aux, epi == EPI_SWIGLU ? p.swi_F : 2 * p.swi_F, 2) &&
           p.swi_F % 8 == 0;
  if (epi == EPI_RESIDUAL && !ok(p.R, p.ldr, p.N, 2)) return false;
  return ok(p.C, p.ldc, p.N, out_bytes);
}

template <int EPI, typename OutT>
static int make_wide_maps(WideEpiMaps* em, const GemmParams& p) {
  constexpr bool fp32 = sizeof(OutT) == 4;
  int rc = 0;
  if constexpr (EPI == EPI_SWIGLU || EPI == EPI_SWIGLU_BWD) {
    const int F = p.swi_F;
    const __nv_bfloat16* aux = static_cast<const __nv_bfloat16*>(p.aux);
    rc = make_epi_map(&em->c, p.C, F, p.M, p.ldc, false);
    if (!rc) rc = make_epi_map(&em->c2, static_cast<const __nv_bfloat16*>(p.C) + F, F, p.M, p.ldc, false);
    if (!rc) rc = make_epi_map(&em->x, aux, F, p.M, p.ld_aux, false);
    if (!rc && EPI == EPI_SWIGLU_BWD) rc = make_epi_map(&em->x2, aux + F, F, p.M, p.ld_aux, false);
  } else {
    rc = make_epi_map(&em->c, p.C, p.N, p.M, p.ldc, fp32);
    if (!rc && EPI == EPI_RESIDUAL) rc = make_epi_map(&em->x, p.R, p.N, p.M, p.ldr, false);
  }
  return rc ? 3000 - rc : 0;
}

template <bool A_MN, bool B_MN, int EPI, typename OutT>
static int launch_staged(const CUtensorMap& tmA, const CUtensorMap& tmB, GemmParams p, cudaStream_t stream) {
  auto kern = gemm_wide_staged_bf16<A_MN, B_MN, EPI, OutT>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, W_SMEM_BYTES);
    if (e != cudaSuccess) return (int)e;
    configured = true;
  }
  WideEpiMaps em;
  if (int rc = make_wide_maps<EPI, OutT>(&em, p)) return rc;
  p.n_tiles = (EPI == EPI_SWIGLU) ? p.swi_F / 128 : (p.N + WBN - 1) / WBN;
  const long long tiles = (long long)p.m_tiles * p.n_tiles;
  const int grid = tiles < sm_count() ? (int)tiles : sm_count();
  kern<<<grid, THREADS, W_SMEM_BYTES, stream>>>(tmA, tmB, em, p);
  return (int)cudaGetLastError();
}


template <bool A_MN, bool B_MN>
static int dispatch_staged(const CUtensorMap& a, const CUtensorMap& b, const GemmParams& p, int epi, int out_fp32,
                           cudaStream_t s) {
  if (out_fp32) {
    if (epi == EPI_STORE) return launch_staged<A_MN, B_MN, EPI_STORE, float>(a, b, p, s);
    if (epi == EPI_ACCUM) return launch_staged<A_MN, B_MN, EPI_ACCUM, float>(a, b, p, s);
    return -10;
  }
  if (epi == EPI_STORE) return launch_staged<A_MN, B_MN, EPI_STORE, __nv_bfloat16>(a, b, p, s);
  if (epi == EPI_RESIDUAL) return launch_staged<A_MN, B_MN, EPI_RESIDUAL, __nv_bfloat16>(a, b, p, s);
  if (epi == EPI_ACCUM) return launch_staged<A_MN, B_MN, EPI_ACCUM, __nv_bfloat16>(a, b, p, s);
  return -10;
}

}  // namespace b200

extern "C" int b200_gemm_wide_staged_ok(const b200::GemmParams* p, int epi, int out_fp32) {
  using namespace b200;
  if (out_fp32 && epi != EPI_STORE && epi != EPI_ACCUM) return 0;   // fp32 +residual: 128 x 128 tile
  return staged_ok(*p, epi, out_fp32 ? 4 : 2) ? 1 : 0;
}

extern "C" int b200_gemm_wide_staged(const CUtensorMap* tmA, const CUtensorMap* tmB, const b200::GemmParams* p,
                                     int a_mn, int b_mn, int epi, int out_fp32, cudaStream_t stream) {
  using namespace b200;
  if (epi == EPI_SWIGLU) return launch_staged<false, false, EPI_SWIGLU, __nv_bfloat16>(*tmA, *tmB, *p, stream);
  if (epi == EPI_SWIGLU_BWD) return launch_staged<false, true, EPI_SWIGLU_BWD, __nv_bfloat16>(*tmA, *tmB, *p, stream);
  if (epi == EPI_ROPE) return launch_staged<false, false, EPI_ROPE, __nv_bfloat16>(*tmA, *tmB, *p, stream);
  if (epi == EPI_ROPE_BIAS) return launch_staged<false, false, EPI_ROPE_BIAS, __nv_bfloat16>(*tmA, *tmB, *p, stream);
  if (a_mn) {
    if (b_mn) return dispatch_staged<true, true>(*tmA, *tmB, *p, epi, out_fp32, stream);
    return dispatch_staged<true, false>(*tmA, *tmB, *p, epi, out_fp32, stream);
  }
  if (b_mn) return dispatch_staged<false, true>(*tmA, *tmB, *p, epi, out_fp32, stream);
  return dispatch_staged<false, false>(*tmA, *tmB, *p, epi, out_fp32, stream);
}
