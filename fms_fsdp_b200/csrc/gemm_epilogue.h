// Operands of the fused GEMM epilogues (csrc/gemm_sm90.cu), passed with every launch.  Host-only: the launcher copies
// them into the kernel's GemmParams.  Each epilogue reads its own group; the others keep these defaults.
#pragma once

struct GemmEpilogueArgs {
  // EPI_ROPE / EPI_ROPE_BIAS: table [S][hd/2][cos, sin] fp32; the first rope_cols columns are rotated
  const float* rope_table = nullptr;
  int rope_S = 1, rope_hd = 2, rope_cols = 0;
  const void* bias = nullptr;        // EPI_ROPE_BIAS: [N] bf16, 4-byte aligned, added before the rotation
  // EPI_SWIGLU / EPI_SWIGLU_BWD: aux = activation output [M, F] (forward) / saved bf16 projection [M, 2F] (backward)
  void* aux = nullptr;
  int ld_aux = 0, swi_F = 0, gate_first = 1;
  // EPI_PUSH: device table of the ranks' staging-buffer bases; push_n elements per shard, the weight starts push_off
  // elements into the flat unit.  push_bulk = 1: tiles leave as 128-byte cp.async.bulk stores staged in shared memory;
  // 0: 4-byte stores from registers.  push_world > 1 rotates the tile raster by push_rank / push_world of a sweep.
  void* const* push_bases = nullptr;
  long long push_n = 1, push_off = 0;
  int push_rank = 0, push_bulk = 1, push_world = 1;
};
