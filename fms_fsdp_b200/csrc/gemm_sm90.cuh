// Definitions shared by the 128 x 128 GEMM kernels of csrc/gemm_sm90.cu and the 128 x 256 GEMM of
// csrc/gemm_wide_sm90.cu: tile constants, epilogue codes, the launch parameters and the per-element helpers.
#pragma once
#include "common.cuh"

namespace b200 {

constexpr int BM = 128, BN = 128, BK = 64;   // BK in bf16 elements = one 128-byte swizzle atom per row
constexpr int STAGES = 6;
constexpr int A_BYTES = BM * BK * 2;          // 16 KiB
constexpr int B_BYTES = BN * BK * 2;          // 16 KiB
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int THREADS = 384;

enum { EPI_STORE = 0, EPI_RESIDUAL = 1, EPI_ACCUM = 2, EPI_ROPE = 3, EPI_PUSH = 4, EPI_SWIGLU = 5, EPI_SWIGLU_BWD = 6,
       EPI_SCALE = 7, EPI_ROPE_BIAS = 8 };
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
  // EPI_ROPE_BIAS (QKV projection with q / k / v biases): bias [N] bf16 is added to the accumulator, then the q / k
  // columns are rotated as in EPI_ROPE.  fp8 launches never rotate, so the bias shares scale_b's slot.
  union { const float* scale_a; const int* grp_seg; };
  union { const float* scale_b; const __nv_bfloat16* bias; };
};

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

constexpr int WBN = 256;                      // columns of the 128 x 256 tile

}  // namespace b200

// The 128 x 256 tile (csrc/gemm_wide_sm90.cu).  _ok: 1 when the tile has the epilogue (all but fp32 +residual) and TMA
// can describe its operands (16-byte aligned bases and row strides, no row stride below the row).
extern "C" int b200_gemm_wide_staged_ok(const b200::GemmParams* p, int epi, int out_fp32);
extern "C" int b200_gemm_wide_staged(const CUtensorMap* tmA, const CUtensorMap* tmB, const b200::GemmParams* p,
                                     int a_mn, int b_mn, int epi, int out_fp32, cudaStream_t stream);
