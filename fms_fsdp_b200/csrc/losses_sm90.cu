// Auxiliary stability losses fused into the kernels that already hold the softmax normaliser (sm_90a):
//   * output z-loss  c * mean_t lse_t^2 inside the softmax cross-entropy gradient of a logits chunk;
//   * router z-loss  c_r * mean_t (logsumexp_e router_logits_te)^2 of the mixture-of-experts routing.
// Every statistic goes to per-row or per-CTA fp32 partials that one CTA sums in a fixed order: no float atomics, so
// gradients and statistics are the same bits on every run.
#include "common.cuh"

namespace b200 {
namespace {

constexpr int LNT = 256;          // threads per CTA of the row kernels
constexpr int RZ_TOK = 8;         // router tokens per CTA (one warp each)
constexpr int RZ_MAX_E = 256;     // 8 experts per lane
constexpr int RED_NT = 1024;      // threads of the partials reduction

// The same reductions and 16-byte accesses as the cross-entropy kernel of csrc/elementwise.cu, so that with c = 0 the
// z-loss kernel reproduces its gradient bit for bit.
B200_DEVINL float lz_block_sum(float v, float* sh) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  float r = (l < (blockDim.x >> 5)) ? sh[l] : 0.f;
  return warp_sum(r);
}
B200_DEVINL float lz_block_max(float v, float* sh) {
  v = warp_max(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  float r = (l < (blockDim.x >> 5)) ? sh[l] : -INFINITY;
  return warp_max(r);
}
B200_DEVINL void lz_load8(const __nv_bfloat16* p, float (&f)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
B200_DEVINL void lz_store8(__nv_bfloat16* p, const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

}  // namespace

// One CTA per row of a bf16 logits chunk [rows, V] (row stride ld), grid-stride over rows.  In place:
//   logits -> [(1 + 2c lse) softmax - onehot] / n_valid   (zero on ignored rows)
// and part[row] = (lse - logit[label], lse^2), both 0 on ignored rows.
__global__ void __launch_bounds__(LNT) ce_zloss_grad_inplace_kernel(__nv_bfloat16* __restrict__ logits,
                                                                    const long long* __restrict__ labels,
                                                                    const float* __restrict__ n_valid,
                                                                    float2* __restrict__ part, int rows, int V, int ld,
                                                                    long long ignore, float two_c) {
  __shared__ float sh[32];
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    __nv_bfloat16* lr = logits + (size_t)row * ld;
    const long long lab = labels[row];
    const bool valid = lab != ignore;
    // pass 1: row max
    float mx = -INFINITY;
    for (int c = threadIdx.x * 8; c < V; c += LNT * 8) {
      float f[8];
      lz_load8(lr + c, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) mx = fmaxf(mx, f[i]);
    }
    mx = lz_block_max(mx, sh);
    // pass 2: sum of exp (the row is L2 / L1 resident: 2 V bytes)
    float se = 0.f;
    for (int c = threadIdx.x * 8; c < V; c += LNT * 8) {
      float f[8];
      lz_load8(lr + c, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) se += __expf(f[i] - mx);
    }
    se = lz_block_sum(se, sh);
    const float lse = mx + __logf(se);
    const float inv_n = valid ? 1.f / fmaxf(*n_valid, 1.f) : 0.f;
    const float g = 1.f + two_c * lse;                           // d(CE + c lse^2) / d lse
    if (threadIdx.x == 0)
      part[row] = valid ? make_float2(lse - __bfloat162float(lr[lab]), lse * lse) : make_float2(0.f, 0.f);
    __syncthreads();  // the label logit must be read before it is overwritten
    // pass 3: gradient in place
    for (int c = threadIdx.x * 8; c < V; c += LNT * 8) {
      float f[8], o[8];
      lz_load8(lr + c, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float p = __expf(f[i] - lse) * g;
        if (c + i == lab) p -= 1.f;
        o[i] = p * inv_n;
      }
      lz_store8(lr + c, o);
    }
  }
}

// One CTA: out[j] = scale * (sum_i part[i nstat + j]) / max(*denom, 1) (denom null: 1) for j < nstat.  Thread t sums
// rows t, t + RED_NT, ... in order, then a fixed tree: the same bits on every run.
__global__ void __launch_bounds__(RED_NT) loss_partials_reduce_kernel(const float* __restrict__ part, int n, int nstat,
                                                                      const float* __restrict__ denom, float scale,
                                                                      float* __restrict__ out) {
  __shared__ float sh[32];
  const float d = denom ? fmaxf(*denom, 1.f) : 1.f;
  for (int j = 0; j < nstat; ++j) {
    float s = 0.f;
    for (int i = threadIdx.x; i < n; i += RED_NT) s += part[(size_t)i * nstat + j];
    s = lz_block_sum(s, sh);
    if (threadIdx.x == 0) out[j] = s / d * scale;
  }
}

// Router z-loss forward: warp per token.  lse[t] = logsumexp_e logits[t, e] (fp32), and part[CTA] = sum of lse^2 of
// the CTA's tokens in token order.
__global__ void __launch_bounds__(RZ_TOK * 32) router_z_fwd_kernel(const float* __restrict__ logits, int T, int E,
                                                                   float* __restrict__ lse, float* __restrict__ part) {
  __shared__ float sq[RZ_TOK];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, t = blockIdx.x * RZ_TOK + w;
  float v = 0.f;
  if (t < T) {
    const float* lr = logits + (size_t)t * E;
    float l[8], mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int e = lane + 32 * j;
      l[j] = e < E ? lr[e] : -INFINITY;
      mx = fmaxf(mx, l[j]);
    }
    mx = warp_max(mx);
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) s += (lane + 32 * j < E) ? expf(l[j] - mx) : 0.f;
    v = mx + logf(warp_sum(s));
    if (lane == 0) lse[t] = v;
  }
  if (lane == 0) sq[w] = v * v;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < RZ_TOK; ++i) s += sq[i];
    part[blockIdx.x] = s;
  }
}

// Router z-loss backward, in place on the bf16 router-logit gradient [T, E]:  dl += scale * lse_t * p_te, in fp32.
// Pairs of experts per thread (E is even), grid-stride.
__global__ void __launch_bounds__(256) router_z_bwd_kernel(__nv_bfloat16* __restrict__ dl,
                                                           const float* __restrict__ probs,
                                                           const float* __restrict__ lse, int T, int E, float scale) {
  const size_t n2 = (size_t)T * E / 2;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += (size_t)gridDim.x * blockDim.x) {
    const int t = (int)(2 * i / E);
    const float a = scale * lse[t];
    uint32_t* q = reinterpret_cast<uint32_t*>(dl) + i;
    const float2 g = unpack_bf16x2(*q);
    const float2 p = reinterpret_cast<const float2*>(probs)[i];
    *q = pack_bf16x2(fmaf(a, p.x, g.x), fmaf(a, p.y, g.y));
  }
}

}  // namespace b200

#define CK() return (int)cudaGetLastError()
using namespace b200;

extern "C" int b200_ce_zloss_grad_inplace(void* logits, const long long* labels, const float* n_valid, float* part,
                                          int rows, int V, int ld, long long ignore, float z_coef, cudaStream_t s) {
  if (V % 8 || ld % 8) return -1;
  if (rows < 1) return 0;
  ce_zloss_grad_inplace_kernel<<<rows < 132 * 8 ? rows : 132 * 8, LNT, 0, s>>>(
      (__nv_bfloat16*)logits, labels, n_valid, reinterpret_cast<float2*>(part), rows, V, ld, ignore, 2.f * z_coef);
  CK();
}

extern "C" int b200_loss_partials_reduce(const float* part, int n, int nstat, const float* denom, float scale, float* out,
                                         cudaStream_t s) {
  if (n < 0 || nstat < 1) return -1;
  loss_partials_reduce_kernel<<<1, RED_NT, 0, s>>>(part, n, nstat, denom, scale, out);
  CK();
}

extern "C" int b200_router_z_parts(int T) { return (T + RZ_TOK - 1) / RZ_TOK; }

extern "C" int b200_router_z_fwd(const float* logits, int T, int E, float* lse, float* part, cudaStream_t s) {
  if (E < 1 || E > RZ_MAX_E) return -1;
  if (T < 1) return 0;
  router_z_fwd_kernel<<<b200_router_z_parts(T), RZ_TOK * 32, 0, s>>>(logits, T, E, lse, part);
  CK();
}

extern "C" int b200_router_z_bwd(void* dl, const float* probs, const float* lse, int T, int E, float scale,
                                 cudaStream_t s) {
  if (E < 2 || E % 2) return -1;
  const size_t n2 = (size_t)T * E / 2;
  if (n2 == 0) return 0;
  const size_t want = (n2 + 255) / 256;
  router_z_bwd_kernel<<<(int)(want < 132 * 16 ? want : 132 * 16), 256, 0, s>>>((__nv_bfloat16*)dl, probs, lse, T, E,
                                                                                scale);
  CK();
}
