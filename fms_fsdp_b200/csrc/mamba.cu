// Mamba-path kernels (sm_90a): depthwise causal conv1d (+SiLU) forward / backward on channels-last
// activations [B*S, C] (SURVEY.md M2).  The SSD / selective scans live in ssd.cu.
#include "common.cuh"

namespace b200 {

constexpr int CONV_MAXK = 4;
constexpr int TCH = 64;  // time steps per CTA row

B200_DEVINL void ld8(const __nv_bfloat16* p, float (&f)[8]) {
  uint4 u = *reinterpret_cast<const uint4*>(p);
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
B200_DEVINL void st8(__nv_bfloat16* p, const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

// thread = 8 channels, walks TCH consecutive time steps of one sequence with a sliding register window
__global__ void causal_conv1d_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                                         const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ y, int C,
                                         int K, int S, int act) {
  const int cv = blockIdx.x * blockDim.x + threadIdx.x;
  if (cv * 8 >= C) return;
  const int c0 = cv * 8;
  const int chunks = (S + TCH - 1) / TCH;
  const int b = blockIdx.y / chunks, t0 = (blockIdx.y % chunks) * TCH;
  float wk[CONV_MAXK][8], bv[8];
#pragma unroll
  for (int k = 0; k < CONV_MAXK; ++k)
#pragma unroll
    for (int i = 0; i < 8; ++i) wk[k][i] = (k < K) ? __bfloat162float(w[(size_t)(c0 + i) * K + k]) : 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) bv[i] = bias ? __bfloat162float(bias[c0 + i]) : 0.f;
  float win[CONV_MAXK][8];  // win[j] = x[t-(K-1)+j]
#pragma unroll
  for (int j = 0; j < CONV_MAXK; ++j)
#pragma unroll
    for (int i = 0; i < 8; ++i) win[j][i] = 0.f;
  const size_t base = (size_t)b * S;
  for (int j = 0; j < K - 1; ++j) {
    const int t = t0 - (K - 1) + j;
    if (t >= 0) ld8(x + (base + t) * C + c0, win[j + 1]);  // pre-shifted: first loop iteration shifts down by one
  }
  const int t1 = min(S, t0 + TCH);
  for (int t = t0; t < t1; ++t) {
#pragma unroll
    for (int j = 0; j < CONV_MAXK - 1; ++j)
#pragma unroll
      for (int i = 0; i < 8; ++i) win[j][i] = win[j + 1][i];
    ld8(x + (base + t) * C + c0, win[K - 1]);
    float o[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float a = bv[i];
#pragma unroll
      for (int k = 0; k < CONV_MAXK; ++k)
        if (k < K) a += wk[k][i] * win[k][i];
      o[i] = act ? a / (1.f + __expf(-a)) : a;
    }
    st8(y + (base + t) * C + c0, o);
  }
}

// dpre[t] = dy[t] * silu'(pre[t]);  dx[t] = sum_k w[k] dpre[t+K-1-k];  dw[k] += x[t-(K-1)+k] dpre[t];  db += dpre[t]
__global__ void causal_conv1d_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                                         const __nv_bfloat16* __restrict__ w, const __nv_bfloat16* __restrict__ bias,
                                         __nv_bfloat16* __restrict__ dx, float* __restrict__ dw, float* __restrict__ db,
                                         int C, int K, int S, int act) {
  const int cv = blockIdx.x * blockDim.x + threadIdx.x;
  if (cv * 8 >= C) return;
  const int c0 = cv * 8;
  const int chunks = (S + TCH - 1) / TCH;
  const int b = blockIdx.y / chunks, t0 = (blockIdx.y % chunks) * TCH;
  const size_t base = (size_t)b * S;
  float wk[CONV_MAXK][8], bv[8], dwacc[CONV_MAXK][8], dbacc[8];
#pragma unroll
  for (int k = 0; k < CONV_MAXK; ++k)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      wk[k][i] = (k < K) ? __bfloat162float(w[(size_t)(c0 + i) * K + k]) : 0.f;
      dwacc[k][i] = 0.f;
    }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    bv[i] = bias ? __bfloat162float(bias[c0 + i]) : 0.f;
    dbacc[i] = 0.f;
  }
  float xw[CONV_MAXK][8];   // x window ending at t
  float dp[CONV_MAXK][8];   // dp[j] = dpre[t-(K-1)+j]
#pragma unroll
  for (int j = 0; j < CONV_MAXK; ++j)
#pragma unroll
    for (int i = 0; i < 8; ++i) { xw[j][i] = 0.f; dp[j][i] = 0.f; }
  for (int j = 0; j < K - 1; ++j) {
    const int t = t0 - (K - 1) + j;
    if (t >= 0) ld8(x + (base + t) * C + c0, xw[j + 1]);
  }
  const int t1 = min(S, t0 + TCH);
  const int t_end = min(S, t1 + K - 1);  // halo: dx[t] needs dpre up to t+K-1
  for (int t = t0; t < t_end; ++t) {
#pragma unroll
    for (int j = 0; j < CONV_MAXK - 1; ++j)
#pragma unroll
      for (int i = 0; i < 8; ++i) { xw[j][i] = xw[j + 1][i]; dp[j][i] = dp[j + 1][i]; }
    ld8(x + (base + t) * C + c0, xw[K - 1]);
    float g[8];
    ld8(dy + (base + t) * C + c0, g);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float a = bv[i];
#pragma unroll
      for (int k = 0; k < CONV_MAXK; ++k)
        if (k < K) a += wk[k][i] * xw[k][i];
      float d = g[i];
      if (act) {
        const float sg = 1.f / (1.f + __expf(-a));
        d *= sg * (1.f + a * (1.f - sg));
      }
      dp[K - 1][i] = d;
      if (t < t1) {  // parameter gradients only for this CTA's own steps (halo steps belong to the next chunk)
        dbacc[i] += d;
#pragma unroll
        for (int k = 0; k < CONV_MAXK; ++k)
          if (k < K) dwacc[k][i] += xw[k][i] * d;
      }
    }
    // dx for step td = t-(K-1): sum_k w[k] * dpre[td+K-1-k] = sum_k w[k] * dp[K-1-k]
    const int td = t - (K - 1);
    if (td >= t0 && td < t1) {
      float o[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float a = 0.f;
#pragma unroll
        for (int k = 0; k < CONV_MAXK; ++k)
          if (k < K) a += wk[k][i] * dp[K - 1 - k][i];
        o[i] = a;
      }
      st8(dx + (base + td) * C + c0, o);
    }
  }
  // tail: steps whose future dpre lies beyond the sequence end (zero contribution from the missing steps)
  for (int td = max(t0, t_end - (K - 1)); td < t1; ++td) {
    // dp window currently ends at t_end-1; dpre[u] = dp[K-1-(t_end-1-u)] for u <= t_end-1, zero beyond
    float o[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = 0.f;
    for (int k = 0; k < K; ++k) {
      const int u = td + K - 1 - k;
      if (u <= t_end - 1) {
        const int j = K - 1 - (t_end - 1 - u);
        if (j >= 0) {
#pragma unroll
          for (int i = 0; i < 8; ++i) o[i] += wk[k][i] * dp[j][i];
        }
      }
    }
    st8(dx + (base + td) * C + c0, o);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    atomicAdd(db + c0 + i, dbacc[i]);
    for (int k = 0; k < K; ++k) atomicAdd(dw + (size_t)(c0 + i) * K + k, dwacc[k][i]);
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_causal_conv1d_fwd(const void* x, const void* w, const void* b, void* y, int M, int C, int K,
                                      int seq_len, int act, cudaStream_t s) {
  if (C % 8 || K > CONV_MAXK || K < 1 || M % seq_len) return -1;
  const int B = M / seq_len, chunks = (seq_len + TCH - 1) / TCH;
  dim3 grid((C / 8 + 127) / 128, B * chunks);
  causal_conv1d_fwd_kernel<<<grid, 128, 0, s>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)w,
                                                (const __nv_bfloat16*)b, (__nv_bfloat16*)y, C, K, seq_len, act);
  return (int)cudaGetLastError();
}
extern "C" int b200_causal_conv1d_bwd(const void* dy, const void* x, const void* w, const void* b, void* dx, float* dw,
                                      float* db, int M, int C, int K, int seq_len, int act, cudaStream_t s) {
  if (C % 8 || K > CONV_MAXK || K < 1 || M % seq_len) return -1;
  const int B = M / seq_len, chunks = (seq_len + TCH - 1) / TCH;
  dim3 grid((C / 8 + 127) / 128, B * chunks);
  causal_conv1d_bwd_kernel<<<grid, 128, 0, s>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x,
                                                (const __nv_bfloat16*)w, (const __nv_bfloat16*)b, (__nv_bfloat16*)dx, dw,
                                                db, C, K, seq_len, act);
  return (int)cudaGetLastError();
}
