// Mixture-of-experts routing and data movement (sm_90a).  Dropless: every (token, slot) gets a row of the expert-sorted
// ("permuted") buffer and nothing is ever synchronised to the host -- the buffer is sized for the worst case
// (T k + E 127 rows, rounded up to 128) and the real segment sizes stay on the device.
//
// The plan (int32, one buffer; see ops/torch_kernels.py MoEPlan for the Python view):
//   tile[NT]     expert of each 128-row tile of the permuted buffer, -1 past the last segment
//   start[E]     first row of each expert's segment (a multiple of 128)
//   len[E]       routed rows of each expert; rows [start + len, start + round_up(len, 128)) are padding
//   row[T k]     permuted row of entry i = t k + s
//   src[Mpad]    entry of each routed row (padding rows: unspecified)
// Inside a segment the rows follow the (token, slot) order, so the wgrad GEMMs, which sum over rows, see the same order
// on every run.  Every padding row of every permuted operand is zero: the grouped wgrad reads whole 64-row k-blocks.
#include "common.cuh"

namespace b200 {

constexpr int MOE_MAX_E = 256, MOE_MAX_K = 8;
constexpr int MOE_TOK_CHUNK = 256;   // tokens per block of the counting and scatter passes

// ---- route: fp32 softmax over E logits, top-k by logit (ties -> lower expert), optional renormalisation. Warp / token.
__global__ void __launch_bounds__(256) moe_route_kernel(const float* __restrict__ logits, int T, int E, int k,
                                                        int norm, float* __restrict__ probs, int* __restrict__ ids,
                                                        float* __restrict__ wts) {
  const int t = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (t >= T) return;
  const float* lr = logits + (size_t)t * E;
  // raw logits feed the softmax (a NaN reaches the probabilities, the weights and the output); the selection sees NaN
  // as -inf, so every token always gets k distinct experts in [0, E) whatever its logits hold
  float l[8];
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int e = lane + 32 * j;
    l[j] = e < E ? lr[e] : -INFINITY;
    mx = fmaxf(mx, l[j]);
  }
  mx = warp_max(mx);
  float p[8], sum = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    p[j] = (lane + 32 * j < E) ? expf(l[j] - mx) : 0.f;
    sum += p[j];
    if ((__float_as_uint(l[j]) & 0x7fffffffu) > 0x7f800000u) l[j] = -INFINITY;   // NaN (bit test: fast-math safe)
  }
  const float inv = 1.f / warp_sum(sum);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    p[j] *= inv;
    if (lane + 32 * j < E) probs[(size_t)t * E + lane + 32 * j] = p[j];
  }
  int my_e = 0;        // lane s keeps slot s
  float my_w = 0.f, wsum = 0.f;
  unsigned used = 0;   // bit j: expert lane + 32 j already selected
  for (int s = 0; s < k; ++s) {
    // the largest unused logit, ties (-inf included) to the lower expert: a lane's first unused expert is always a
    // candidate, so the winner is a valid index as long as k <= E
    float bv = -INFINITY;
    int be = 0x7fffffff;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (lane + 32 * j < E && !(used >> j & 1u) && (l[j] > bv || be == 0x7fffffff)) { bv = l[j]; be = lane + 32 * j; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oe = __shfl_xor_sync(0xffffffffu, be, o);
      if (ov > bv || (ov == bv && oe < be)) { bv = ov; be = oe; }
    }
    // the owner lane reads the probability and retires the expert
    float pv = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (lane + 32 * j == be) { pv = p[j]; used |= 1u << j; }
    pv = __shfl_sync(0xffffffffu, pv, be & 31);
    wsum += pv;
    if (lane == s) { my_e = be; my_w = pv; }
  }
  if (lane < k) {
    ids[(size_t)t * k + lane] = my_e;
    wts[(size_t)t * k + lane] = norm ? my_w / wsum : my_w;
  }
}

// ---- plan, pass 1: per block of MOE_TOK_CHUNK tokens, the expert histogram and the column sums of the probabilities
__global__ void __launch_bounds__(256) moe_count_kernel(const int* __restrict__ ids, const float* __restrict__ probs,
                                                        int T, int E, int k, int* __restrict__ cnt,
                                                        float* __restrict__ psum) {
  __shared__ int hist[MOE_MAX_E];
  const int c = blockIdx.x, t0 = c * MOE_TOK_CHUNK, t1 = min(T, t0 + MOE_TOK_CHUNK);
  for (int e = threadIdx.x; e < E; e += blockDim.x) hist[e] = 0;
  __syncthreads();
  for (int i = t0 * k + threadIdx.x; i < t1 * k; i += blockDim.x) atomicAdd(&hist[ids[i]], 1);   // integer: exact
  __syncthreads();
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    float s = 0.f;
    for (int t = t0; t < t1; ++t) s += probs[(size_t)t * E + e];
    cnt[(size_t)c * E + e] = hist[e];
    psum[(size_t)c * E + e] = s;
  }
}

// ---- plan, pass 2 (one block): segment sizes and starts, the tile table, per-block scatter bases (in place of cnt) and
// the load-balancing statistic aux = E * sum_e (count_e / T) * mean_t p_te
__global__ void __launch_bounds__(256) moe_scan_kernel(int* __restrict__ cnt, const float* __restrict__ psum, int C,
                                                       int T, int E, int NT, int* __restrict__ tile,
                                                       int* __restrict__ start, int* __restrict__ len,
                                                       float* __restrict__ aux) {
  __shared__ int s_start[MOE_MAX_E + 1];
  __shared__ float s_aux[MOE_MAX_E];
  const int e = threadIdx.x;
  int total = 0;
  if (e < E) {
    float ps = 0.f;
    for (int c = 0; c < C; ++c) {
      const int n = cnt[(size_t)c * E + e];
      cnt[(size_t)c * E + e] = total;   // offset of block c inside the segment (start added below)
      total += n;
      ps += psum[(size_t)c * E + e];
    }
    len[e] = total;
    s_start[e] = (total + 127) & ~127;
    s_aux[e] = (float)total * ps;
  }
  __syncthreads();
  if (e == 0) {
    int run = 0;
    float a = 0.f;
    for (int i = 0; i < E; ++i) {
      const int padded = s_start[i];
      s_start[i] = run;
      run += padded;
      a += s_aux[i];
    }
    s_start[E] = run;
    aux[0] = a * (float)E / ((float)T * (float)T);
  }
  __syncthreads();
  if (e < E) {
    start[e] = s_start[e];
    for (int c = 0; c < C; ++c) cnt[(size_t)c * E + e] += s_start[e];
  }
  for (int i = threadIdx.x; i < NT; i += blockDim.x) {
    const int r = i * 128;
    int lo = 0, hi = E;                // last expert whose segment starts at or before r (empty segments share a start
    while (hi - lo > 1) {              // with the next one, which is the one that owns the row)
      const int mid = (lo + hi) >> 1;
      if (s_start[mid] <= r) lo = mid; else hi = mid;
    }
    tile[i] = r < s_start[E] ? lo : -1;
  }
}

// ---- plan, pass 3: rows in (token, slot) order inside each segment.  A block walks its entries 256 at a time; a warp
// ranks equal experts with match.any, and the warps' counts are combined in warp order.
__global__ void __launch_bounds__(256) moe_scatter_kernel(const int* __restrict__ ids, const int* __restrict__ base_in,
                                                          int T, int E, int k, int* __restrict__ row,
                                                          int* __restrict__ src) {
  __shared__ int base[MOE_MAX_E];
  __shared__ int wcnt[8][MOE_MAX_E];
  const int c = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i0 = c * MOE_TOK_CHUNK * k, i1 = min(T, (c + 1) * MOE_TOK_CHUNK) * k;
  for (int e = threadIdx.x; e < E; e += blockDim.x) base[e] = base_in[(size_t)c * E + e];
  for (int b = i0; b < i1; b += 256) {
    for (int j = threadIdx.x; j < 8 * MOE_MAX_E; j += 256) (&wcnt[0][0])[j] = 0;
    __syncthreads();
    const int i = b + threadIdx.x;
    const int e = i < i1 ? ids[i] : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, e);
    const int rank = __popc(peers & ((1u << lane) - 1));
    if (e >= 0 && rank == 0) wcnt[warp][e] = __popc(peers);
    __syncthreads();
    if (e >= 0) {
      int off = base[e] + rank;
      for (int w = 0; w < warp; ++w) off += wcnt[w][e];
      row[i] = off;
      src[off] = i;
    }
    __syncthreads();
    for (int x = threadIdx.x; x < E; x += blockDim.x) {
      int n = 0;
#pragma unroll
      for (int w = 0; w < 8; ++w) n += wcnt[w][x];
      base[x] += n;
    }
    __syncthreads();
  }
}

// padding row of a segment (zero it), routed row (returns its entry), or a row past the last segment (-2)
B200_DEVINL int moe_row_kind(const int* tile, const int* start, const int* len, const int* src, int r) {
  const int e = tile[r >> 7];
  if (e < 0) return -2;
  return (r - start[e] < len[e]) ? src[r] : -1;
}

// ---- permute: X_perm[row(t, s)] = x[t], padding rows zero.  One warp per permuted row, 16-byte vectors.
__global__ void __launch_bounds__(256) moe_permute_kernel(const __nv_bfloat16* __restrict__ x, const int* __restrict__ tile,
                                                          const int* __restrict__ start, const int* __restrict__ len,
                                                          const int* __restrict__ src, int Mpad, int k, int D,
                                                          __nv_bfloat16* __restrict__ xp) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= Mpad) return;
  const int i = moe_row_kind(tile, start, len, src, r);
  if (i == -2) return;
  uint4* dst = reinterpret_cast<uint4*>(xp + (size_t)r * D);
  const uint4* s = reinterpret_cast<const uint4*>(x + (size_t)(i / k) * D);
  for (int v = lane; v < D / 8; v += 32) dst[v] = i >= 0 ? s[v] : make_uint4(0, 0, 0, 0);
}

// ---- permute backward: dx[t] = sum_s dX_perm[row(t, s)] in slot order, fp32.  One warp per token.
__global__ void __launch_bounds__(256) moe_permute_bwd_kernel(const __nv_bfloat16* __restrict__ dxp,
                                                              const int* __restrict__ row, int T, int k, int D,
                                                              __nv_bfloat16* __restrict__ dx) {
  const int t = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (t >= T) return;
  for (int v = lane; v < D / 8; v += 32) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int s = 0; s < k; ++s) {
      const uint4 u = reinterpret_cast<const uint4*>(dxp + (size_t)row[(size_t)t * k + s] * D)[v];
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 f = unpack_bf16x2(w[q]);
        acc[2 * q] += f.x; acc[2 * q + 1] += f.y;
      }
    }
    reinterpret_cast<uint4*>(dx + (size_t)t * D)[v] =
        make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]), pack_bf16x2(acc[4], acc[5]),
                   pack_bf16x2(acc[6], acc[7]));
  }
}

// ---- combine: y[t] = residual[t] + sum_s w[t, s] Y_perm[row(t, s)], fp32 in slot order.  One warp per token.
__global__ void __launch_bounds__(256) moe_combine_kernel(const __nv_bfloat16* __restrict__ yp, const int* __restrict__ row,
                                                          const float* __restrict__ wts,
                                                          const __nv_bfloat16* __restrict__ res, int T, int k, int D,
                                                          __nv_bfloat16* __restrict__ y) {
  const int t = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (t >= T) return;
  for (int v = lane; v < D / 8; v += 32) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (res) {
      const uint4 u = reinterpret_cast<const uint4*>(res + (size_t)t * D)[v];
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 f = unpack_bf16x2(w[q]);
        acc[2 * q] = f.x; acc[2 * q + 1] = f.y;
      }
    }
    for (int s = 0; s < k; ++s) {
      const float g = wts[(size_t)t * k + s];
      const uint4 u = reinterpret_cast<const uint4*>(yp + (size_t)row[(size_t)t * k + s] * D)[v];
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 f = unpack_bf16x2(w[q]);
        acc[2 * q] += g * f.x; acc[2 * q + 1] += g * f.y;
      }
    }
    reinterpret_cast<uint4*>(y + (size_t)t * D)[v] =
        make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]), pack_bf16x2(acc[4], acc[5]),
                   pack_bf16x2(acc[6], acc[7]));
  }
}

// ---- combine backward: dY_perm[row] = w dy[t] (padding rows zero) and dw[t, s] = <dy[t], Y_perm[row]>.  Warp per row.
__global__ void __launch_bounds__(256) moe_combine_bwd_kernel(const __nv_bfloat16* __restrict__ dy,
                                                              const __nv_bfloat16* __restrict__ yp,
                                                              const float* __restrict__ wts, const int* __restrict__ tile,
                                                              const int* __restrict__ start, const int* __restrict__ len,
                                                              const int* __restrict__ src, int Mpad, int k, int D,
                                                              __nv_bfloat16* __restrict__ dyp, float* __restrict__ dw) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= Mpad) return;
  const int i = moe_row_kind(tile, start, len, src, r);
  if (i == -2) return;
  uint4* dst = reinterpret_cast<uint4*>(dyp + (size_t)r * D);
  if (i < 0) {
    for (int v = lane; v < D / 8; v += 32) dst[v] = make_uint4(0, 0, 0, 0);
    return;
  }
  const float g = wts[i];
  const uint4* gy = reinterpret_cast<const uint4*>(dy + (size_t)(i / k) * D);
  const uint4* yr = reinterpret_cast<const uint4*>(yp + (size_t)r * D);
  float dot = 0.f;
  for (int v = lane; v < D / 8; v += 32) {
    const uint4 a = gy[v], b = yr[v];
    const uint32_t wa[4] = {a.x, a.y, a.z, a.w}, wb[4] = {b.x, b.y, b.z, b.w};
    uint32_t o[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float2 fa = unpack_bf16x2(wa[q]), fb = unpack_bf16x2(wb[q]);
      dot += fa.x * fb.x + fa.y * fb.y;
      o[q] = pack_bf16x2(g * fa.x, g * fa.y);
    }
    dst[v] = make_uint4(o[0], o[1], o[2], o[3]);
  }
  dot = warp_sum(dot);
  if (lane == 0) dw[i] = dot;
}

// ---- route backward: through the renormalisation and the softmax to dlogits (bf16, the operand of the router's dgrad
// and wgrad GEMMs), plus the load-balancing gradient aux_scale * count_e on every probability.  Warp per token.
__global__ void __launch_bounds__(256) moe_route_bwd_kernel(const float* __restrict__ probs, const int* __restrict__ ids,
                                                            const float* __restrict__ wts, const float* __restrict__ dw,
                                                            const int* __restrict__ count, int T, int E, int k,
                                                            int norm, float aux_scale,
                                                            __nv_bfloat16* __restrict__ dlogits) {
  const int t = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (t >= T) return;
  const float* pr = probs + (size_t)t * E;
  const int* it = ids + (size_t)t * k;
  const float* wt = wts + (size_t)t * k;
  const float* gt = dw + (size_t)t * k;
  // gradient of each selected probability
  float z = 0.f, gw = 0.f;
  if (norm) {
    for (int s = 0; s < k; ++s) { z += pr[it[s]]; gw += gt[s] * wt[s]; }
  }
  float dp[8], p[8], dot = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int e = lane + 32 * j;
    p[j] = e < E ? pr[e] : 0.f;
    float d = e < E ? aux_scale * (float)count[e] : 0.f;
    for (int s = 0; s < k; ++s)
      if (it[s] == e) d += norm ? (gt[s] - gw) / z : gt[s];
    dp[j] = d;
    dot += p[j] * d;
  }
  dot = warp_sum(dot);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int e = lane + 32 * j;
    if (e < E) dlogits[(size_t)t * E + e] = __float2bfloat16_rn(p[j] * (dp[j] - dot));
  }
}

static inline int blocks_of(long long n, int per) { return (int)((n + per - 1) / per); }

}  // namespace b200

#define CK() return (int)cudaGetLastError()
using namespace b200;

extern "C" int b200_moe_route(const float* logits, int T, int E, int k, int norm, float* probs, int* ids, float* wts,
                              cudaStream_t s) {
  if (E < 1 || E > MOE_MAX_E || k < 1 || k > MOE_MAX_K || k > E) return -1;
  if (T < 1) return 0;
  moe_route_kernel<<<blocks_of(T, 8), 256, 0, s>>>(logits, T, E, k, norm, probs, ids, wts);
  CK();
}

// ws: int [C, E] then float [C, E] with C = ceil(T / MOE_TOK_CHUNK) (b200_moe_plan_ws_chunks)
extern "C" int b200_moe_plan_ws_chunks(int T) { return (T + MOE_TOK_CHUNK - 1) / MOE_TOK_CHUNK; }

extern "C" int b200_moe_plan(const int* ids, const float* probs, int T, int E, int k, int NT, int* ws_cnt, float* ws_psum,
                             int* tile, int* start, int* len, int* row, int* src, float* aux, cudaStream_t s) {
  if (E < 1 || E > MOE_MAX_E || k < 1 || k > MOE_MAX_K || T < 1) return -1;
  const int C = b200_moe_plan_ws_chunks(T);
  moe_count_kernel<<<C, 256, 0, s>>>(ids, probs, T, E, k, ws_cnt, ws_psum);
  moe_scan_kernel<<<1, 256, 0, s>>>(ws_cnt, ws_psum, C, T, E, NT, tile, start, len, aux);
  moe_scatter_kernel<<<C, 256, 0, s>>>(ids, ws_cnt, T, E, k, row, src);
  CK();
}

extern "C" int b200_moe_permute(const void* x, const int* tile, const int* start, const int* len, const int* src,
                                int Mpad, int k, int D, void* xp, cudaStream_t s) {
  if (D % 8) return -1;
  moe_permute_kernel<<<blocks_of(Mpad, 8), 256, 0, s>>>((const __nv_bfloat16*)x, tile, start, len, src, Mpad, k, D,
                                                        (__nv_bfloat16*)xp);
  CK();
}

extern "C" int b200_moe_permute_bwd(const void* dxp, const int* row, int T, int k, int D, void* dx, cudaStream_t s) {
  if (D % 8) return -1;
  moe_permute_bwd_kernel<<<blocks_of(T, 8), 256, 0, s>>>((const __nv_bfloat16*)dxp, row, T, k, D, (__nv_bfloat16*)dx);
  CK();
}

extern "C" int b200_moe_combine(const void* yp, const int* row, const float* wts, const void* res, int T, int k, int D,
                                void* y, cudaStream_t s) {
  if (D % 8) return -1;
  moe_combine_kernel<<<blocks_of(T, 8), 256, 0, s>>>((const __nv_bfloat16*)yp, row, wts, (const __nv_bfloat16*)res, T,
                                                     k, D, (__nv_bfloat16*)y);
  CK();
}

extern "C" int b200_moe_combine_bwd(const void* dy, const void* yp, const float* wts, const int* tile, const int* start,
                                    const int* len, const int* src, int Mpad, int k, int D, void* dyp, float* dw,
                                    cudaStream_t s) {
  if (D % 8) return -1;
  moe_combine_bwd_kernel<<<blocks_of(Mpad, 8), 256, 0, s>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)yp, wts,
                                                            tile, start, len, src, Mpad, k, D, (__nv_bfloat16*)dyp, dw);
  CK();
}

extern "C" int b200_moe_route_bwd(const float* probs, const int* ids, const float* wts, const float* dw, const int* count,
                                  int T, int E, int k, int norm, float aux_scale, void* dlogits, cudaStream_t s) {
  if (E < 1 || E > MOE_MAX_E || k < 1 || k > MOE_MAX_K) return -1;
  if (T < 1) return 0;
  moe_route_bwd_kernel<<<blocks_of(T, 8), 256, 0, s>>>(probs, ids, wts, dw, count, T, E, k, norm, aux_scale,
                                                       (__nv_bfloat16*)dlogits);
  CK();
}
