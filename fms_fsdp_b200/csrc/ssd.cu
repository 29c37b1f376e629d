// Mamba2 state-space-dual (SSD) chunk scan, forward and backward (SURVEY.md M3; reference: mamba_ssm's Triton
// ssd_chunk_state / ssd_state_passing / ssd_bmm / ssd_chunk_scan / ssd_combined).
//
// All GEMM-shaped work runs on the wgmma GEMM in batched mode (gemm_sm90.cu, BATCH=true): per 128-token chunk
//   CB = C_c B_c^T,  Y_diag = (CB o decay-mask_h) X_h,  S_c = B_c^T (X o dt o decay),  Y_off = C_c prev_c
// with the per-head products folded into the N (or K) dimension wherever the other operand is shared by the heads.
// This file holds the glue between those GEMMs: dt softplus + in-chunk cumsum, the per-head decay mask, the
// sequential inter-chunk state recurrence (fp32), the output combine, and their backward counterparts.
//
// Shapes: x [M, H, P]; dt [M, H]; A, D, dt_bias [H]; B, C [M, G, N]; M = batch * S, chunks of L = 128 tokens.
// acs[row, h] = inclusive in-chunk cumsum of dt*A (<= 0);  aL[bc, h] = acs of the chunk's last row.
#include "common.cuh"

namespace b200 {

constexpr int SSD_L = 128;

B200_DEVINL float softplus_f(float x) { return x > 20.f ? x : log1pf(__expf(x)); }
B200_DEVINL float sigmoid_f(float x) { return 1.f / (1.f + __expf(-x)); }

// ------------------------------------------------------------------ forward glue
// one thread per (chunk, head): dtv = softplus(dt + bias), acs = cumsum(dtv * A)
__global__ void ssd_prep_kernel(const __nv_bfloat16* __restrict__ dt, const float* __restrict__ A,
                                const float* __restrict__ dt_bias, float* __restrict__ dtv, float* __restrict__ acs,
                                float* __restrict__ aL, int n_chunks, int H, int softplus) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_chunks * H) return;
  const int h = idx % H, bc = idx / H;
  const float a_h = A[h], bias = dt_bias ? dt_bias[h] : 0.f;
  float run = 0.f;
  for (int l = 0; l < SSD_L; ++l) {
    const size_t o = ((size_t)bc * SSD_L + l) * H + h;
    float v = __bfloat162float(dt[o]) + bias;
    if (softplus) v = softplus_f(v);
    run += v * a_h;
    dtv[o] = v;
    acs[o] = run;
  }
  aL[idx] = run;
}

// CTA per (chunk, head): Mh[l, s] = CB[l, s] * exp(acs_l - acs_s) * dtv_s  (s <= l), 0 above the diagonal
__global__ void __launch_bounds__(256) ssd_mask_kernel(const __nv_bfloat16* __restrict__ CB, const float* __restrict__ acs,
                                                       const float* __restrict__ dtv, __nv_bfloat16* __restrict__ Mh,
                                                       int H, int G) {
  __shared__ float s_a[SSD_L], s_d[SSD_L];
  const int h = blockIdx.x, bc = blockIdx.y, g = h / (H / G);
  if (threadIdx.x < SSD_L) {
    const size_t o = ((size_t)bc * SSD_L + threadIdx.x) * H + h;
    s_a[threadIdx.x] = acs[o];
    s_d[threadIdx.x] = dtv[o];
  }
  __syncthreads();
  const __nv_bfloat16* cb = CB + ((size_t)bc * G + g) * SSD_L * SSD_L;
  __nv_bfloat16* out = Mh + ((size_t)bc * H + h) * SSD_L * SSD_L;
  for (int v = threadIdx.x; v < SSD_L * SSD_L / 8; v += 256) {
    const int l = v / (SSD_L / 8), s0 = (v % (SSD_L / 8)) * 8;
    uint4 o = make_uint4(0, 0, 0, 0);
    if (s0 <= l) {
      const uint4 c = *reinterpret_cast<const uint4*>(cb + l * SSD_L + s0);
      const uint32_t cw[4] = {c.x, c.y, c.z, c.w};
      uint32_t ow[4];
      const float al = s_a[l];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 cf = unpack_bf16x2(cw[j]);
        const int s = s0 + 2 * j;
        const float m0 = (s <= l) ? cf.x * __expf(al - s_a[s]) * s_d[s] : 0.f;
        const float m1 = (s + 1 <= l) ? cf.y * __expf(al - s_a[s + 1]) * s_d[s + 1] : 0.f;
        ow[j] = pack_bf16x2(m0, m1);
      }
      o = make_uint4(ow[0], ow[1], ow[2], ow[3]);
    }
    *reinterpret_cast<uint4*>(out + l * SSD_L + s0) = o;
  }
}

// Xs = x * dtv * exp(aL - acs)   (thread per 8 channels of one (row, head))
__global__ void ssd_xs_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ dtv,
                              const float* __restrict__ acs, const float* __restrict__ aL,
                              __nv_bfloat16* __restrict__ xs, size_t M, int H, int P) {
  const int vph = P / 8;
  const size_t total = M * H * vph;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t rh = i / vph;                      // row * H + h
    const size_t row = rh / H;
    const int h = (int)(rh % H);
    const float sc = dtv[rh] * __expf(aL[(row / SSD_L) * H + h] - acs[rh]);
    const uint4 u = *reinterpret_cast<const uint4*>(x + i * 8);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      o[j] = pack_bf16x2(f.x * sc, f.y * sc);
    }
    *reinterpret_cast<uint4*>(xs + i * 8) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// Inter-chunk recurrence, thread per state element (n, h, p) of one sequence:
//   prev[c] = R_c ;  R_{c+1} = exp(aL_c) R_c + S_c          (R_0 = 0, fp32 running value)
__global__ void ssd_state_pass_kernel(const float* __restrict__ states, const float* __restrict__ aL,
                                      __nv_bfloat16* __restrict__ prev, int nc, int Nd, int H, int P) {
  const size_t per_seq = (size_t)Nd * H * P;
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (e >= per_seq) return;
  const int h = (int)((e % ((size_t)H * P)) / P);
  float run = 0.f;
  for (int c = 0; c < nc; ++c) {
    const size_t o = ((size_t)b * nc + c) * per_seq + e;
    prev[o] = __float2bfloat16(run);
    run = run * __expf(aL[((size_t)b * nc + c) * H + h]) + states[o];
  }
}

// y = Y_diag + exp(acs) * Y_off + D * x
__global__ void ssd_combine_kernel(const __nv_bfloat16* __restrict__ yd, const __nv_bfloat16* __restrict__ yoff,
                                   const __nv_bfloat16* __restrict__ x, const float* __restrict__ acs,
                                   const float* __restrict__ D, __nv_bfloat16* __restrict__ y, size_t M, int H, int P) {
  const int vph = P / 8;
  const size_t total = M * H * vph;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t rh = i / vph;
    const int h = (int)(rh % H);
    const float ea = __expf(acs[rh]), dh = D ? D[h] : 0.f;
    const uint4 a = *reinterpret_cast<const uint4*>(yd + i * 8);
    const uint4 b = *reinterpret_cast<const uint4*>(yoff + i * 8);
    const uint4 c = *reinterpret_cast<const uint4*>(x + i * 8);
    const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w}, cw[4] = {c.x, c.y, c.z, c.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 fa = unpack_bf16x2(aw[j]), fb = unpack_bf16x2(bw[j]), fc = unpack_bf16x2(cw[j]);
      o[j] = pack_bf16x2(fa.x + ea * fb.x + dh * fc.x, fa.y + ea * fb.y + dh * fc.y);
    }
    *reinterpret_cast<uint4*>(y + i * 8) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// ------------------------------------------------------------------ backward glue
// warp per (row, head): dYs = dy * exp(acs) ; dacs = sum_p dYs * Yoff ; dDrow = sum_p dy * x
__global__ void ssd_dyoff_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ yoff,
                                 const __nv_bfloat16* __restrict__ x, const float* __restrict__ acs,
                                 __nv_bfloat16* __restrict__ dys, float* __restrict__ dacs, float* __restrict__ dDrow,
                                 size_t MH, int P) {
  const size_t w = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= MH) return;
  const float ea = __expf(acs[w]);
  float s1 = 0.f, s2 = 0.f;
  for (int p = lane * 2; p < P; p += 64) {
    const size_t o = w * P + p;
    const float2 g = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dy + o));
    const float2 yo = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(yoff + o));
    const float2 xv = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(x + o));
    const float d0 = g.x * ea, d1 = g.y * ea;
    *reinterpret_cast<uint32_t*>(dys + o) = pack_bf16x2(d0, d1);
    s1 += d0 * yo.x + d1 * yo.y;
    s2 += g.x * xv.x + g.y * xv.y;
  }
  s1 = warp_sum(s1);
  s2 = warp_sum(s2);
  if (lane == 0) { dacs[w] = s1; dDrow[w] = s2; }
}

// CTA per (32-row band, group, chunk), looping over the group's heads.  With W = exp(acs_l - acs_s) dtv_s (s <= l):
//   dCB[l,s]  = sum_h dMh W          T = dMh CB W
//   dacs[l] += sum_s T ;  dacs[s] -= sum_l T ;  ddtv[s] += sum_l T / dtv_s
__global__ void __launch_bounds__(256) ssd_mask_bwd_kernel(const __nv_bfloat16* __restrict__ dMh,
                                                           const __nv_bfloat16* __restrict__ CB,
                                                           const float* __restrict__ acs, const float* __restrict__ dtv,
                                                           __nv_bfloat16* __restrict__ dCB, float* __restrict__ dacs,
                                                           float* __restrict__ ddtv, int H, int G) {
  __shared__ float s_a[SSD_L], s_d[SSD_L], s_col[SSD_L], s_row[32];
  const int band = blockIdx.x, g = blockIdx.y, bc = blockIdx.z, Hg = H / G;
  // thread -> (row within band, 16 consecutive columns): 32 rows x 8 column groups = 256 threads
  const int lr = threadIdx.x >> 3, cg = threadIdx.x & 7;
  const int l = band * 32 + lr, s0 = cg * 16;
  float cbv[16], acc[16];
  {
    const __nv_bfloat16* cb = CB + (((size_t)bc * G + g) * SSD_L + l) * SSD_L + s0;
#pragma unroll
    for (int j = 0; j < 16; j += 2) {
      const float2 f = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(cb + j));
      cbv[j] = f.x; cbv[j + 1] = f.y;
      acc[j] = acc[j + 1] = 0.f;
    }
  }
  for (int hh = 0; hh < Hg; ++hh) {
    const int h = g * Hg + hh;
    __syncthreads();
    if (threadIdx.x < SSD_L) {
      const size_t o = ((size_t)bc * SSD_L + threadIdx.x) * H + h;
      s_a[threadIdx.x] = acs[o];
      s_d[threadIdx.x] = dtv[o];
      s_col[threadIdx.x] = 0.f;
    }
    if (threadIdx.x < 32) s_row[threadIdx.x] = 0.f;
    __syncthreads();
    const __nv_bfloat16* dm = dMh + (((size_t)bc * H + h) * SSD_L + l) * SSD_L + s0;
    const float al = s_a[l];
    float rsum = 0.f;
    // a warp holds 4 rows x 8 column groups: column sums are first reduced over its 4 rows with shuffles
#pragma unroll
    for (int j = 0; j < 16; j += 2) {
      float2 gm = make_float2(0.f, 0.f);
      if (s0 + j <= l) gm = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dm + j));
      const float gg[2] = {gm.x, gm.y};
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int s = s0 + j + e;
        float t = 0.f;
        if (s <= l) {
          const float w = __expf(al - s_a[s]) * s_d[s];
          acc[j + e] += gg[e] * w;
          t = gg[e] * cbv[j + e] * w;
        }
        rsum += t;
        t += __shfl_xor_sync(0xffffffffu, t, 8);
        t += __shfl_xor_sync(0xffffffffu, t, 16);
        if ((threadIdx.x & 31) < 8 && t != 0.f) atomicAdd(&s_col[s], t);
      }
    }
    // row sum: the 8 column groups of a row are 8 consecutive lanes
    rsum += __shfl_xor_sync(0xffffffffu, rsum, 1);
    rsum += __shfl_xor_sync(0xffffffffu, rsum, 2);
    rsum += __shfl_xor_sync(0xffffffffu, rsum, 4);
    if (cg == 0) s_row[lr] = rsum;
    __syncthreads();
    if (threadIdx.x < SSD_L) {
      const int s = threadIdx.x;
      const size_t o = ((size_t)bc * SSD_L + s) * H + h;
      const float cs = s_col[s];
      if (cs != 0.f) {
        atomicAdd(&dacs[o], -cs);
        atomicAdd(&ddtv[o], cs / s_d[s]);
      }
    }
    if (threadIdx.x < 32) {
      const size_t o = ((size_t)bc * SSD_L + band * 32 + threadIdx.x) * H + h;
      atomicAdd(&dacs[o], s_row[threadIdx.x]);
    }
  }
  __nv_bfloat16* out = dCB + (((size_t)bc * G + g) * SSD_L + l) * SSD_L + s0;
#pragma unroll
  for (int j = 0; j < 16; j += 2) *reinterpret_cast<uint32_t*>(out + j) = pack_bf16x2(acc[j], acc[j + 1]);
}

// reverse inter-chunk recurrence, thread per state element:  g_c = total dR_{c+1}
//   dS_c = g_c ;  daL_c += sum g_c * exp(aL_c) * R_c ;  g_{c-1} = dprev_c + exp(aL_c) * g_c
__global__ void ssd_state_pass_bwd_kernel(const float* __restrict__ dprev, const __nv_bfloat16* __restrict__ prev,
                                          const float* __restrict__ aL, __nv_bfloat16* __restrict__ dstates,
                                          float* __restrict__ daL, int nc, int Nd, int H, int P) {
  const size_t per_seq = (size_t)Nd * H * P;
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  const bool ok = e < per_seq;
  const int h = ok ? (int)((e % ((size_t)H * P)) / P) : 0;
  const int lane = threadIdx.x & 31;
  float g = 0.f;
  for (int c = nc - 1; c >= 0; --c) {
    const size_t o = ((size_t)b * nc + c) * per_seq + e;
    const float ea = __expf(aL[((size_t)b * nc + c) * H + h]);
    float contrib = 0.f;
    if (ok) {
      dstates[o] = __float2bfloat16(g);
      contrib = g * ea * __bfloat162float(prev[o]);
      g = dprev[o] + ea * g;
    }
    // lanes of a warp share the head when P is a multiple of 32 (asserted by the launcher)
    contrib = warp_sum(contrib);
    if (lane == 0 && contrib != 0.f) atomicAdd(&daL[((size_t)b * nc + c) * H + h], contrib);
  }
}

// warp per (row, head):  e2 = exp(aL - acs)
//   dx = dx_diag + dXs * dtv * e2 + D * dy ;  ddtv += sum_p dXs x e2 ;  t = dtv * that ;  dacs -= t ;  daL += t
__global__ void ssd_dx_kernel(const __nv_bfloat16* __restrict__ dxd, const __nv_bfloat16* __restrict__ dxs,
                              const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                              const float* __restrict__ dtv, const float* __restrict__ acs, const float* __restrict__ aL,
                              const float* __restrict__ D, __nv_bfloat16* __restrict__ dx, float* __restrict__ ddtv,
                              float* __restrict__ dacs, float* __restrict__ daL, size_t MH, int H, int P) {
  const size_t w = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= MH) return;
  const size_t row = w / H;
  const int h = (int)(w % H);
  const size_t ci = (row / SSD_L) * H + h;
  const float dv = dtv[w], e2 = __expf(aL[ci] - acs[w]), dh = D ? D[h] : 0.f;
  float s = 0.f;
  for (int p = lane * 2; p < P; p += 64) {
    const size_t o = w * P + p;
    const float2 a = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dxd + o));
    const float2 b = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dxs + o));
    const float2 g = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(dy + o));
    const float2 xv = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(x + o));
    *reinterpret_cast<uint32_t*>(dx + o) = pack_bf16x2(a.x + b.x * dv * e2 + dh * g.x, a.y + b.y * dv * e2 + dh * g.y);
    s += b.x * xv.x + b.y * xv.y;
  }
  s = warp_sum(s) * e2;
  if (lane == 0) {
    ddtv[w] += s;
    const float t = s * dv;
    dacs[w] -= t;
    atomicAdd(&daL[ci], t);
  }
}

// thread per (chunk, head): fold daL into the last row, reverse-cumsum dacs, chain through dt*A and softplus
__global__ void ssd_dt_bwd_kernel(const __nv_bfloat16* __restrict__ dt, const float* __restrict__ A,
                                  const float* __restrict__ dt_bias, const float* __restrict__ dtv,
                                  const float* __restrict__ dacs, const float* __restrict__ ddtv,
                                  const float* __restrict__ daL, __nv_bfloat16* __restrict__ ddt, float* __restrict__ dA,
                                  float* __restrict__ dbias, int n_chunks, int H, int softplus) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_chunks * H) return;
  const int h = idx % H, bc = idx / H;
  const float a_h = A[h], bias = dt_bias ? dt_bias[h] : 0.f;
  float rcs = daL[idx], dA_acc = 0.f, db_acc = 0.f;
  for (int l = SSD_L - 1; l >= 0; --l) {
    const size_t o = ((size_t)bc * SSD_L + l) * H + h;
    rcs += dacs[o];
    const float g = ddtv[o] + a_h * rcs;
    dA_acc += dtv[o] * rcs;
    float draw = g;
    if (softplus) {
      const float raw = __bfloat162float(dt[o]) + bias;
      if (raw <= 20.f) draw = g * sigmoid_f(raw);
    }
    ddt[o] = __float2bfloat16(draw);
    db_acc += draw;
  }
  atomicAdd(&dA[h], dA_acc);
  if (dbias) atomicAdd(&dbias[h], db_acc);
}

static inline int ew_grid(size_t work, int threads) {
  size_t b = (work + threads - 1) / threads;
  return (int)(b > 132 * 16 ? 132 * 16 : (b < 1 ? 1 : b));
}

}  // namespace b200

using namespace b200;
#define CKE() return (int)cudaGetLastError()

extern "C" int b200_ssd_prep(const void* dt, const float* A, const float* bias, float* dtv, float* acs, float* aL,
                             int n_chunks, int H, int softplus, cudaStream_t s) {
  const int n = n_chunks * H;
  ssd_prep_kernel<<<(n + 127) / 128, 128, 0, s>>>((const __nv_bfloat16*)dt, A, bias, dtv, acs, aL, n_chunks, H, softplus);
  CKE();
}
extern "C" int b200_ssd_mask(const void* CB, const float* acs, const float* dtv, void* Mh, int n_chunks, int H, int G,
                             cudaStream_t s) {
  ssd_mask_kernel<<<dim3(H, n_chunks), 256, 0, s>>>((const __nv_bfloat16*)CB, acs, dtv, (__nv_bfloat16*)Mh, H, G);
  CKE();
}
extern "C" int b200_ssd_xs(const void* x, const float* dtv, const float* acs, const float* aL, void* xs, long long M, int H,
                           int P, cudaStream_t s) {
  if (P % 8) return -1;
  ssd_xs_kernel<<<ew_grid((size_t)M * H * (P / 8), 256), 256, 0, s>>>((const __nv_bfloat16*)x, dtv, acs, aL,
                                                                     (__nv_bfloat16*)xs, (size_t)M, H, P);
  CKE();
}
extern "C" int b200_ssd_state_pass(const float* states, const float* aL, void* prev, int batch, int nc, int Nd, int H, int P,
                                   cudaStream_t s) {
  const size_t per_seq = (size_t)Nd * H * P;
  ssd_state_pass_kernel<<<dim3((unsigned)((per_seq + 255) / 256), batch), 256, 0, s>>>(states, aL, (__nv_bfloat16*)prev, nc,
                                                                                     Nd, H, P);
  CKE();
}
extern "C" int b200_ssd_combine(const void* yd, const void* yoff, const void* x, const float* acs, const float* D, void* y,
                                long long M, int H, int P, cudaStream_t s) {
  if (P % 8) return -1;
  ssd_combine_kernel<<<ew_grid((size_t)M * H * (P / 8), 256), 256, 0, s>>>(
      (const __nv_bfloat16*)yd, (const __nv_bfloat16*)yoff, (const __nv_bfloat16*)x, acs, D, (__nv_bfloat16*)y, (size_t)M, H, P);
  CKE();
}
extern "C" int b200_ssd_dyoff(const void* dy, const void* yoff, const void* x, const float* acs, void* dys, float* dacs,
                              float* dDrow, long long MH, int P, cudaStream_t s) {
  if (P % 2) return -1;
  const size_t threads = (size_t)MH * 32;
  ssd_dyoff_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)yoff,
                                                                    (const __nv_bfloat16*)x, acs, (__nv_bfloat16*)dys, dacs,
                                                                    dDrow, (size_t)MH, P);
  CKE();
}
extern "C" int b200_ssd_mask_bwd(const void* dMh, const void* CB, const float* acs, const float* dtv, void* dCB, float* dacs,
                                 float* ddtv, int n_chunks, int H, int G, cudaStream_t s) {
  ssd_mask_bwd_kernel<<<dim3(SSD_L / 32, G, n_chunks), 256, 0, s>>>((const __nv_bfloat16*)dMh, (const __nv_bfloat16*)CB, acs,
                                                                   dtv, (__nv_bfloat16*)dCB, dacs, ddtv, H, G);
  CKE();
}
extern "C" int b200_ssd_state_pass_bwd(const float* dprev, const void* prev, const float* aL, void* dstates, float* daL,
                                       int batch, int nc, int Nd, int H, int P, cudaStream_t s) {
  if (P % 32) return -1;
  const size_t per_seq = (size_t)Nd * H * P;
  ssd_state_pass_bwd_kernel<<<dim3((unsigned)((per_seq + 255) / 256), batch), 256, 0, s>>>(
      dprev, (const __nv_bfloat16*)prev, aL, (__nv_bfloat16*)dstates, daL, nc, Nd, H, P);
  CKE();
}
extern "C" int b200_ssd_dx(const void* dxd, const void* dxs, const void* dy, const void* x, const float* dtv,
                           const float* acs, const float* aL, const float* D, void* dx, float* ddtv, float* dacs,
                           float* daL, long long MH, int H, int P, cudaStream_t s) {
  if (P % 2) return -1;
  const size_t threads = (size_t)MH * 32;
  ssd_dx_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(
      (const __nv_bfloat16*)dxd, (const __nv_bfloat16*)dxs, (const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, dtv, acs, aL, D,
      (__nv_bfloat16*)dx, ddtv, dacs, daL, (size_t)MH, H, P);
  CKE();
}
extern "C" int b200_ssd_dt_bwd(const void* dt, const float* A, const float* bias, const float* dtv, const float* dacs,
                               const float* ddtv, const float* daL, void* ddt, float* dA, float* dbias, int n_chunks, int H,
                               int softplus, cudaStream_t s) {
  const int n = n_chunks * H;
  ssd_dt_bwd_kernel<<<(n + 127) / 128, 128, 0, s>>>((const __nv_bfloat16*)dt, A, bias, dtv, dacs, ddtv, daL,
                                                   (__nv_bfloat16*)ddt, dA, dbias, n_chunks, H, softplus);
  CKE();
}
