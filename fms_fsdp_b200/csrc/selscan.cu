// Mamba1 selective scan, forward and backward (SURVEY.md M4; reference: mamba_ssm selective_scan_{fwd,bwd}_kernel.cuh).
//
//   h_t = exp(delta_t A) h_{t-1} + delta_t u_t B_t ;   y_t = C_t . h_t + D u_t ;   y_t *= silu(z_t)
//
// Not GEMM-shaped (d_state = 16): a bandwidth/latency kernel.  H100 mapping: CTA = 32 channels x the whole sequence of
// one batch element; WARP = one channel, LANE = one of 32 consecutive timesteps; the recurrence over a 32-step block is
// an affine inclusive scan done with 5 shuffle rounds per state, blocks are chained through a per-warp carry.  Tiles of
// [32 t x 32 d] go through shared memory so every global access is a coalesced 64-byte row segment, and B_t / C_t
// (shared by all channels) are staged once per block.  Backward walks the blocks in reverse, recomputes the in-block
// forward scan from the carries the forward pass checkpointed, and runs the adjoint recurrence as a suffix scan.
#include "common.cuh"

namespace b200 {

constexpr int SS_N = 16;   // d_state
constexpr int SS_T = 32;   // timesteps per block (= warp width)
constexpr int SS_D = 32;   // channels per CTA (= warps per CTA)

B200_DEVINL float ss_softplus(float x) { return x > 20.f ? x : log1pf(__expf(x)); }

struct SelScanParams {
  const __nv_bfloat16 *u, *delta, *z, *Bm, *Cm;   // [M, Dm], [M, Dm], [M, Dm] or null, [M, N], [M, N]
  const float *A, *D, *dbias;                     // [Dm, N], [Dm] or null, [Dm] or null
  float* hcarry;                                  // [B, L/32, Dm, N] state entering each block (fwd writes, bwd reads)
  int L, Dm, softplus;
};

// cooperative tile load: element (t = warp, d = lane) of a [32 x 32] bf16 tile -> smem[t][d]
B200_DEVINL void load_tile(float (*s)[SS_D + 1], const __nv_bfloat16* g, size_t row0, int Dm, int d0, int w, int lane) {
  s[w][lane] = __bfloat162float(g[(row0 + w) * Dm + d0 + lane]);
}

__global__ void __launch_bounds__(1024, 1) selscan_fwd_kernel(SelScanParams p, __nv_bfloat16* __restrict__ y) {
  __shared__ float s_u[SS_T][SS_D + 1], s_dl[SS_T][SS_D + 1], s_z[SS_T][SS_D + 1], s_y[SS_T][SS_D + 1];
  __shared__ float s_B[SS_T][SS_N], s_C[SS_T][SS_N];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int d0 = blockIdx.x * SS_D, d = d0 + w, b = blockIdx.y;
  // per-channel vectors over the 16 states live one-per-lane (lane n <-> state n) and are broadcast with shuffles
  const float A_l = (lane < SS_N) ? p.A[(size_t)d * SS_N + lane] : 0.f;
  float h_l = 0.f;
  const float Dd = p.D ? p.D[d] : 0.f, bias = p.dbias ? p.dbias[d] : 0.f;
  const int nblk = p.L / SS_T;
  for (int tb = 0; tb < nblk; ++tb) {
    const size_t row0 = (size_t)b * p.L + (size_t)tb * SS_T;
    __syncthreads();
    load_tile(s_u, p.u, row0, p.Dm, d0, w, lane);
    load_tile(s_dl, p.delta, row0, p.Dm, d0, w, lane);
    if (p.z) load_tile(s_z, p.z, row0, p.Dm, d0, w, lane);
    if (threadIdx.x < SS_T * SS_N) {
      const int t = threadIdx.x / SS_N, n = threadIdx.x % SS_N;
      s_B[t][n] = __bfloat162float(p.Bm[(row0 + t) * SS_N + n]);
      s_C[t][n] = __bfloat162float(p.Cm[(row0 + t) * SS_N + n]);
    }
    __syncthreads();
    if (p.hcarry && lane < SS_N) p.hcarry[(((size_t)b * nblk + tb) * p.Dm + d) * SS_N + lane] = h_l;
    const float ut = s_u[lane][w];
    float dt = s_dl[lane][w] + bias;
    if (p.softplus) dt = ss_softplus(dt);
    float yt = Dd * ut;
#pragma unroll
    for (int n = 0; n < SS_N; ++n) {
      const float An = __shfl_sync(0xffffffffu, A_l, n), h_in = __shfl_sync(0xffffffffu, h_l, n);
      float a = __expf(dt * An);
      float bb = dt * ut * s_B[lane][n];
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {       // inclusive scan of the affine maps h -> a h + b
        const float a2 = __shfl_up_sync(0xffffffffu, a, off), b2 = __shfl_up_sync(0xffffffffu, bb, off);
        if (lane >= off) { bb = fmaf(a, b2, bb); a *= a2; }
      }
      const float ht = fmaf(a, h_in, bb);
      yt = fmaf(s_C[lane][n], ht, yt);
      const float hl = __shfl_sync(0xffffffffu, ht, 31);
      if (lane == n) h_l = hl;
    }
    if (p.z) { const float zt = s_z[lane][w]; yt *= zt / (1.f + __expf(-zt)); }
    s_y[lane][w] = yt;
    __syncthreads();
    y[(row0 + w) * p.Dm + d0 + lane] = __float2bfloat16(s_y[w][lane]);
  }
}

struct SelScanGrads {
  __nv_bfloat16 *du, *ddelta, *dz;    // [M, Dm]
  float *dA, *dB, *dC, *dD, *ddbias;  // [Dm, N], [M, N], [M, N], [Dm], [Dm]  (zero-initialised, accumulated atomically)
};

__global__ void __launch_bounds__(1024, 1) selscan_bwd_kernel(SelScanParams p, const __nv_bfloat16* __restrict__ dy,
                                                              SelScanGrads g) {
  __shared__ float s_u[SS_T][SS_D + 1], s_dl[SS_T][SS_D + 1], s_z[SS_T][SS_D + 1], s_dy[SS_T][SS_D + 1];
  __shared__ float s_o1[SS_T][SS_D + 1], s_o2[SS_T][SS_D + 1], s_o3[SS_T][SS_D + 1];
  __shared__ float s_B[SS_T][SS_N], s_C[SS_T][SS_N], s_dB[SS_T][SS_N], s_dC[SS_T][SS_N];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int d0 = blockIdx.x * SS_D, d = d0 + w, b = blockIdx.y;
  // lane n <-> state n for A, the adjoint carry and the next block's first decay; dA partials stay per lane (timestep)
  const float A_l = (lane < SS_N) ? p.A[(size_t)d * SS_N + lane] : 0.f;
  float dhc_l = 0.f, anext_l = 0.f, dA_acc[SS_N];
#pragma unroll
  for (int n = 0; n < SS_N; ++n) dA_acc[n] = 0.f;
  const float Dd = p.D ? p.D[d] : 0.f, bias = p.dbias ? p.dbias[d] : 0.f;
  float dD_acc = 0.f, db_acc = 0.f;
  const int nblk = p.L / SS_T;
  for (int tb = nblk - 1; tb >= 0; --tb) {
    const size_t row0 = (size_t)b * p.L + (size_t)tb * SS_T;
    __syncthreads();
    load_tile(s_u, p.u, row0, p.Dm, d0, w, lane);
    load_tile(s_dl, p.delta, row0, p.Dm, d0, w, lane);
    load_tile(s_dy, dy, row0, p.Dm, d0, w, lane);
    if (p.z) load_tile(s_z, p.z, row0, p.Dm, d0, w, lane);
    if (threadIdx.x < SS_T * SS_N) {
      const int t = threadIdx.x / SS_N, n = threadIdx.x % SS_N;
      s_B[t][n] = __bfloat162float(p.Bm[(row0 + t) * SS_N + n]);
      s_C[t][n] = __bfloat162float(p.Cm[(row0 + t) * SS_N + n]);
      s_dB[t][n] = 0.f;
      s_dC[t][n] = 0.f;
    }
    __syncthreads();
    const float ut = s_u[lane][w];
    const float raw = s_dl[lane][w] + bias;
    const float dt = p.softplus ? ss_softplus(raw) : raw;
    float gy = s_dy[lane][w];                         // gradient w.r.t. the pre-gate output
    float zt = 0.f, sg = 0.f;
    if (p.z) { zt = s_z[lane][w]; sg = 1.f / (1.f + __expf(-zt)); }
    const float gy_out = gy;
    if (p.z) gy *= zt * sg;
    // carry entering this block (checkpointed by the forward pass): lane n holds state n
    const float hin_l = (lane < SS_N) ? p.hcarry[(((size_t)b * nblk + tb) * p.Dm + d) * SS_N + lane] : 0.f;
    float ypre = Dd * ut, ddt = 0.f, dut = Dd * gy;
#pragma unroll
    for (int n = 0; n < SS_N; ++n) {
      const float h_in = __shfl_sync(0xffffffffu, hin_l, n), An = __shfl_sync(0xffffffffu, A_l, n);
      const float dh_in = __shfl_sync(0xffffffffu, dhc_l, n), a_nx = __shfl_sync(0xffffffffu, anext_l, n);
      const float a_t = __expf(dt * An);
      const float Bt = s_B[lane][n], Ct = s_C[lane][n];
      // forward in-block scan
      float a = a_t, bb = dt * ut * Bt;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const float a2 = __shfl_up_sync(0xffffffffu, a, off), b2 = __shfl_up_sync(0xffffffffu, bb, off);
        if (lane >= off) { bb = fmaf(a, b2, bb); a *= a2; }
      }
      const float ht = fmaf(a, h_in, bb);
      float hprev = __shfl_up_sync(0xffffffffu, ht, 1);
      if (lane == 0) hprev = h_in;
      ypre = fmaf(Ct, ht, ypre);
      // adjoint recurrence dh_t = C_t gy_t + a_{t+1} dh_{t+1}: suffix scan with alpha_t = a_{t+1}
      float al = __shfl_down_sync(0xffffffffu, a_t, 1);
      if (lane == 31) al = a_nx;
      float gg = Ct * gy;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const float al2 = __shfl_down_sync(0xffffffffu, al, off), g2 = __shfl_down_sync(0xffffffffu, gg, off);
        if (lane + off < 32) { gg = fmaf(al, g2, gg); al *= al2; }
      }
      const float dh = fmaf(al, dh_in, gg);
      const float dh0 = __shfl_sync(0xffffffffu, dh, 0), a0 = __shfl_sync(0xffffffffu, a_t, 0);
      if (lane == n) { dhc_l = dh0; anext_l = a0; }
      const float da = dh * hprev * a_t;              // d / d(delta_t A_n)
      ddt = fmaf(da, An, ddt);
      ddt = fmaf(dh * ut, Bt, ddt);
      dA_acc[n] = fmaf(da, dt, dA_acc[n]);
      dut = fmaf(dh * dt, Bt, dut);
      atomicAdd(&s_dB[lane][n], dh * dt * ut);        // summed over the CTA's 32 channels
      atomicAdd(&s_dC[lane][n], gy * ht);
    }
    dD_acc = fmaf(gy, ut, dD_acc);
    float draw = ddt;
    if (p.softplus && raw <= 20.f) draw = ddt / (1.f + __expf(-raw));
    db_acc += draw;
    s_o1[lane][w] = dut;
    s_o2[lane][w] = draw;
    if (p.z) s_o3[lane][w] = gy_out * ypre * sg * (1.f + zt * (1.f - sg));   // d silu(z) = sg (1 + z (1 - sg))
    __syncthreads();
    g.du[(row0 + w) * p.Dm + d0 + lane] = __float2bfloat16(s_o1[w][lane]);
    g.ddelta[(row0 + w) * p.Dm + d0 + lane] = __float2bfloat16(s_o2[w][lane]);
    if (p.z) g.dz[(row0 + w) * p.Dm + d0 + lane] = __float2bfloat16(s_o3[w][lane]);
    if (threadIdx.x < SS_T * SS_N) {
      const int t = threadIdx.x / SS_N, n = threadIdx.x % SS_N;
      atomicAdd(&g.dB[(row0 + t) * SS_N + n], s_dB[t][n]);
      atomicAdd(&g.dC[(row0 + t) * SS_N + n], s_dC[t][n]);
    }
  }
#pragma unroll
  for (int n = 0; n < SS_N; ++n) {
    const float v = warp_sum(dA_acc[n]);
    if (lane == 0) atomicAdd(&g.dA[(size_t)d * SS_N + n], v);
  }
  dD_acc = warp_sum(dD_acc);
  db_acc = warp_sum(db_acc);
  if (lane == 0) {
    if (g.dD) atomicAdd(&g.dD[d], dD_acc);
    if (g.ddbias) atomicAdd(&g.ddbias[d], db_acc);
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_selscan_fwd(const void* u, const void* delta, const float* A, const void* Bm, const void* Cm,
                                const float* D, const void* z, const float* dbias, float* hcarry, void* y, int batch, int L,
                                int Dm, int N, int softplus, cudaStream_t s) {
  if (N != SS_N || L % SS_T || Dm % SS_D) return -1;
  SelScanParams p{(const __nv_bfloat16*)u, (const __nv_bfloat16*)delta, (const __nv_bfloat16*)z, (const __nv_bfloat16*)Bm,
                  (const __nv_bfloat16*)Cm, A, D, dbias, hcarry, L, Dm, softplus};
  selscan_fwd_kernel<<<dim3(Dm / SS_D, batch), 1024, 0, s>>>(p, (__nv_bfloat16*)y);
  return (int)cudaGetLastError();
}
extern "C" int b200_selscan_bwd(const void* dy, const void* u, const void* delta, const float* A, const void* Bm,
                                const void* Cm, const float* D, const void* z, const float* dbias, float* hcarry, void* du,
                                void* ddelta, void* dz, float* dA, float* dB, float* dC, float* dD, float* ddbias, int batch,
                                int L, int Dm, int N, int softplus, cudaStream_t s) {
  if (N != SS_N || L % SS_T || Dm % SS_D) return -1;
  SelScanParams p{(const __nv_bfloat16*)u, (const __nv_bfloat16*)delta, (const __nv_bfloat16*)z, (const __nv_bfloat16*)Bm,
                  (const __nv_bfloat16*)Cm, A, D, dbias, hcarry, L, Dm, softplus};
  SelScanGrads g{(__nv_bfloat16*)du, (__nv_bfloat16*)ddelta, (__nv_bfloat16*)dz, dA, dB, dC, dD, ddbias};
  selscan_bwd_kernel<<<dim3(Dm / SS_D, batch), 1024, 0, s>>>(p, (const __nv_bfloat16*)dy, g);
  return (int)cudaGetLastError();
}
