// NVLink / NVSwitch peer-memory collectives (no NCCL on the hot path).
//
// Every rank registers its buffers in a symmetric heap (torch symmetric memory rendezvous); kernels get
// a device table of the W peer addresses of the same buffer and move data with plain 16-byte
// ld.global / st.global on peer-mapped pointers (SASS: LDG.E.128 on the peer aperture), i.e. the
// "P2P loads over NVSwitch" path of SURVEY.md §5.8.  Cross-GPU ordering uses a signal pad per rank and
// st.release.sys / ld.acquire.sys flags.
//
//   signal_barrier     all ranks of the group have reached this point of their stream
//   p2p_allgather      full[r*n:(r+1)*n] = shard of rank r          (pull; parameter path, N7)
//   reduce_scatter     out32 = scale * sum_r full_r[my slice] (+ sum of squares)   (gradient path, N8 + K11);
//                      accumulate mode: out32 += scale * sum_r ... (gradient accumulation over micro-steps)
//   allreduce_inplace  phase 1 of a two-phase all-reduce: reduce my slice in place (N9/N10)
#include "common.cuh"

namespace b200 {

B200_DEVINL void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
B200_DEVINL uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
B200_DEVINL uint4 ld_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
B200_DEVINL uint4 ld_relaxed_v4(const void* p) {
  // peer data written by another GPU before a barrier: must not be served from a stale non-coherent path
  uint4 r;
  asm volatile("ld.global.relaxed.sys.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}

// pads[r] -> uint32 signal pad on rank r, organised as channels of 32 slots.  Rank `rank` posts `epoch` into slot
// [slot_base + rank] of every peer's pad, then waits until slots [slot_base, slot_base + W) of its own pad have reached
// `epoch`.  Channels keep barriers that are enqueued on different streams from observing each other's epochs.
B200_DEVINL void spin_until(const uint32_t* flag, uint32_t epoch) {
  uint64_t t0 = 0;
  uint32_t spins = 0;
  while ((int32_t)(ld_acquire_sys(flag) - epoch) < 0) {
    if ((++spins & 0x3ff) == 0) {
      uint64_t now = global_timer_ns();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 20000000000ull) __trap();  // 20 s: a peer died
    }
  }
}

__global__ void signal_barrier_kernel(uint32_t* const* pads, int world, int rank, uint32_t epoch, int slot_base) {
  const int p = threadIdx.x;
  if (p < world) {
    __threadfence_system();
    st_release_sys(pads[p] + slot_base + rank, epoch);
    spin_until(pads[rank] + slot_base + p, epoch);
  }
}

// One-sided halves of the barrier: "my work up to here is visible" / "wait until every rank has posted".  Used for the
// per-unit optimizer flags: rank r posts (unit u, step t) after its AdamW of unit u; whoever gathers unit u waits.
__global__ void signal_post_kernel(uint32_t* const* pads, int world, int rank, uint32_t epoch, int slot_base) {
  const int p = threadIdx.x;
  if (p < world) {
    __threadfence_system();
    st_release_sys(pads[p] + slot_base + rank, epoch);
  }
}
__global__ void signal_wait_kernel(uint32_t* const* pads, int world, int rank, uint32_t epoch, int slot_base) {
  const int p = threadIdx.x;
  if (p < world) spin_until(pads[rank] + slot_base + p, epoch);
}

// One-shot all-reduce (sum) of a few fp32 scalars over the signal pads (grad-norm: SURVEY.md N11 / section 5.8 item 5).
// bufs[r] -> on rank r: float vals[2][32][MAXV] followed by uint32 flags[2][32]; parity = epoch & 1 double-buffers
// the slots (a rank can only be one call ahead of the slowest peer).  Every rank sums in rank order, so all ranks
// get bit-identical results.
constexpr int SAR_MAXV = 8;
__global__ void scalar_allreduce_kernel(uint8_t* const* bufs, int world, int rank, uint32_t epoch, float* inout, int nvals) {
  const int p = threadIdx.x;
  const int par = epoch & 1;
  const size_t flags_off = (size_t)2 * 32 * SAR_MAXV * sizeof(float);
  if (p < world) {
    float* vals = reinterpret_cast<float*>(bufs[p]) + ((size_t)par * 32 + rank) * SAR_MAXV;
    for (int i = 0; i < nvals; ++i) vals[i] = inout[i];
    __threadfence_system();
    st_release_sys(reinterpret_cast<uint32_t*>(bufs[p] + flags_off) + par * 32 + rank, epoch);
    spin_until(reinterpret_cast<const uint32_t*>(bufs[rank] + flags_off) + par * 32 + p, epoch);
  }
  __syncthreads();
  if (p < nvals) {
    const float* mine = reinterpret_cast<const float*>(bufs[rank]) + (size_t)par * 32 * SAR_MAXV;
    float acc = 0.f;
    for (int r = 0; r < world; ++r) acc += *reinterpret_cast<const volatile float*>(mine + r * SAR_MAXV + p);
    inout[p] = acc;
  }
}

// Pull all-gather.  One "row" of CTAs per source rank (rotated so that rank r starts on peer r+1 and the
// 7 inbound NVLink flows of the switch are all busy from the first instruction).
__global__ void __launch_bounds__(512) p2p_allgather_kernel(const void* const* shard_ptrs, uint8_t* full,
                                                            size_t shard_bytes, int world, int rank) {
  const int ctas_per_peer = gridDim.x / world;
  const int slot = blockIdx.x / ctas_per_peer;                 // 0..W-1
  const int src = (rank + 1 + slot) % world;                   // local copy is done last
  const int c = blockIdx.x % ctas_per_peer;
  const uint8_t* s = reinterpret_cast<const uint8_t*>(shard_ptrs[src]);
  uint8_t* d = full + (size_t)src * shard_bytes;
  const size_t nvec = shard_bytes / 16;
  const size_t stride = (size_t)ctas_per_peer * blockDim.x;
  size_t i = (size_t)c * blockDim.x + threadIdx.x;
  // 4 independent 16-byte loads in flight per thread before the first store
  for (; i + 3 * stride < nvec; i += 4 * stride) {
    uint4 a = ld_relaxed_v4(s + i * 16);
    uint4 b = ld_relaxed_v4(s + (i + stride) * 16);
    uint4 e = ld_relaxed_v4(s + (i + 2 * stride) * 16);
    uint4 f = ld_relaxed_v4(s + (i + 3 * stride) * 16);
    *reinterpret_cast<uint4*>(d + i * 16) = a;
    *reinterpret_cast<uint4*>(d + (i + stride) * 16) = b;
    *reinterpret_cast<uint4*>(d + (i + 2 * stride) * 16) = e;
    *reinterpret_cast<uint4*>(d + (i + 3 * stride) * 16) = f;
  }
  for (; i < nvec; i += stride) *reinterpret_cast<uint4*>(d + i * 16) = ld_relaxed_v4(s + i * 16);
}

// Gather an arbitrary byte range [begin, end) of the unit (flat = concatenation of the W shards) from the owners.
__global__ void __launch_bounds__(512) p2p_gather_range_kernel(const void* const* shard_ptrs, uint8_t* full,
                                                               size_t shard_bytes, size_t begin, size_t end) {
  const size_t nvec = (end - begin) / 16;
  for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += (size_t)gridDim.x * blockDim.x) {
    const size_t off = begin + v * 16;
    const size_t src = off / shard_bytes;
    *reinterpret_cast<uint4*>(full + off) =
        ld_relaxed_v4(reinterpret_cast<const uint8_t*>(shard_ptrs[src]) + (off - src * shard_bytes));
  }
}

// EXPERIMENTAL (docs/next_steps.md 2): the inverse of gather_range for gradients -- element range [off, off + len) of this
// rank's contribution to a unit's flat gradient is written into the OWNERS' staging slots
//   owner = e / n ;  dst = bases[owner] + rank * n + (e - owner * n)        (bf16 elements, 16-byte vectors)
__global__ void __launch_bounds__(256) p2p_push_range_kernel(const __nv_bfloat16* __restrict__ src, void* const* bases,
                                                             size_t n, size_t off, size_t len, int rank) {
  const size_t nvec = len / 8;
  for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += (size_t)gridDim.x * blockDim.x) {
    const size_t e = off + v * 8;
    const size_t owner = e / n;
    __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(bases[owner]) + ((size_t)rank * n + (e - owner * n));
    *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src + v * 8);
  }
}

B200_DEVINL float block_sum256(float v, float* sh) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) sh[w] = v;
  __syncthreads();
  float r = (l < (blockDim.x >> 5)) ? sh[l] : 0.f;
  return warp_sum(r);
}

// out[i] = scale * sum_r src_r[off + i]   (src bf16 or fp32, out fp32) ; sumsq += sum out^2
// ACC: out[i] += scale * sum_r src_r[off + i] ; sumsq += sum of the squared RESULT (the accumulated gradient)
template <bool SRC_BF16, int W, bool ACC = false>
__global__ void __launch_bounds__(256) reduce_scatter_kernel(const void* const* srcs, float* out, size_t n, size_t off,
                                                             int rank, float scale, float* sumsq) {
  __shared__ float sh[32];
  constexpr int VEC = SRC_BF16 ? 8 : 4;
  const uint8_t* base[W];
#pragma unroll
  for (int r = 0; r < W; ++r) {
    const int src = (rank + r) % W;
    base[r] = reinterpret_cast<const uint8_t*>(srcs[src]) + off * (SRC_BF16 ? 2 : 4);
  }
  float ss = 0.f;
  const size_t nvec = n / VEC;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    uint4 v[W];
#pragma unroll
    for (int r = 0; r < W; ++r) v[r] = ld_relaxed_v4(base[r] + i * 16);
    float acc[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) acc[k] = 0.f;
#pragma unroll
    for (int r = 0; r < W; ++r) {
      if constexpr (SRC_BF16) {
        float2 a = unpack_bf16x2(v[r].x), b = unpack_bf16x2(v[r].y), c = unpack_bf16x2(v[r].z), d = unpack_bf16x2(v[r].w);
        acc[0] += a.x; acc[1] += a.y; acc[2] += b.x; acc[3] += b.y;
        acc[4] += c.x; acc[5] += c.y; acc[6] += d.x; acc[7] += d.y;
      } else {
        acc[0] += __uint_as_float(v[r].x); acc[1] += __uint_as_float(v[r].y);
        acc[2] += __uint_as_float(v[r].z); acc[3] += __uint_as_float(v[r].w);
      }
    }
    float4* o = reinterpret_cast<float4*>(out + i * VEC);
    float prev[VEC];
    if constexpr (ACC) {
      const float4 p0 = o[0];
      prev[0] = p0.x; prev[1] = p0.y; prev[2] = p0.z; prev[3] = p0.w;
      if constexpr (SRC_BF16) {
        const float4 p1 = o[1];
        prev[4] = p1.x; prev[5] = p1.y; prev[6] = p1.z; prev[7] = p1.w;
      }
    }
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
      acc[k] *= scale;
      if constexpr (ACC) acc[k] += prev[k];
      ss += acc[k] * acc[k];
    }
    o[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    if constexpr (SRC_BF16) o[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
  }
  if (sumsq) {
    ss = block_sum256(ss, sh);
    if (threadIdx.x == 0) atomicAdd(sumsq, ss);
  }
}

// Any group size (HSDP 2x3, 6-GPU jobs ...): peer table read per iteration instead of W unrolled base registers.
template <bool SRC_BF16, bool ACC = false>
__global__ void __launch_bounds__(256) reduce_scatter_dyn_kernel(const void* const* srcs, float* out, size_t n, size_t off,
                                                                 int world, int rank, float scale, float* sumsq) {
  __shared__ float sh[32];
  constexpr int VEC = SRC_BF16 ? 8 : 4;
  float ss = 0.f;
  const size_t nvec = n / VEC;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    float acc[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) acc[k] = 0.f;
    for (int r = 0; r < world; ++r) {
      const uint8_t* b = reinterpret_cast<const uint8_t*>(srcs[(rank + r) % world]) + off * (SRC_BF16 ? 2 : 4);
      const uint4 v = ld_relaxed_v4(b + i * 16);
      if constexpr (SRC_BF16) {
        float2 a = unpack_bf16x2(v.x), bb = unpack_bf16x2(v.y), c = unpack_bf16x2(v.z), d = unpack_bf16x2(v.w);
        acc[0] += a.x; acc[1] += a.y; acc[2] += bb.x; acc[3] += bb.y;
        acc[4] += c.x; acc[5] += c.y; acc[6] += d.x; acc[7] += d.y;
      } else {
        acc[0] += __uint_as_float(v.x); acc[1] += __uint_as_float(v.y);
        acc[2] += __uint_as_float(v.z); acc[3] += __uint_as_float(v.w);
      }
    }
    float4* o = reinterpret_cast<float4*>(out + i * VEC);
    float prev[VEC];
    if constexpr (ACC) {
      const float4 p0 = o[0];
      prev[0] = p0.x; prev[1] = p0.y; prev[2] = p0.z; prev[3] = p0.w;
      if constexpr (SRC_BF16) {
        const float4 p1 = o[1];
        prev[4] = p1.x; prev[5] = p1.y; prev[6] = p1.z; prev[7] = p1.w;
      }
    }
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
      acc[k] *= scale;
      if constexpr (ACC) acc[k] += prev[k];
      ss += acc[k] * acc[k];
    }
    o[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    if constexpr (SRC_BF16) o[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
  }
  if (sumsq) {
    ss = block_sum256(ss, sh);
    if (threadIdx.x == 0) atomicAdd(sumsq, ss);
  }
}

// In-place reduction of this rank's slice [rank*n_slice, (rank+1)*n_slice) of a symmetric buffer (phase 1 of
// a two-phase all-reduce; phase 2 is p2p_allgather on the same buffers after a barrier).
template <bool IS_BF16, int W>
__global__ void __launch_bounds__(256) reduce_slice_inplace_kernel(void* const* bufs, size_t n_slice, int rank,
                                                                  float scale, float* sumsq) {
  __shared__ float sh[32];
  constexpr int VEC = IS_BF16 ? 8 : 4;
  constexpr int ES = IS_BF16 ? 2 : 4;
  const uint8_t* base[W];
#pragma unroll
  for (int r = 0; r < W; ++r)
    base[r] = reinterpret_cast<const uint8_t*>(bufs[(rank + r) % W]) + (size_t)rank * n_slice * ES;
  uint8_t* mine = reinterpret_cast<uint8_t*>(bufs[rank]) + (size_t)rank * n_slice * ES;
  float ss = 0.f;
  const size_t nvec = n_slice / VEC;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    uint4 v[W];
#pragma unroll
    for (int r = 0; r < W; ++r) v[r] = ld_relaxed_v4(base[r] + i * 16);
    float acc[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) acc[k] = 0.f;
#pragma unroll
    for (int r = 0; r < W; ++r) {
      if constexpr (IS_BF16) {
        float2 a = unpack_bf16x2(v[r].x), b = unpack_bf16x2(v[r].y), c = unpack_bf16x2(v[r].z), d = unpack_bf16x2(v[r].w);
        acc[0] += a.x; acc[1] += a.y; acc[2] += b.x; acc[3] += b.y;
        acc[4] += c.x; acc[5] += c.y; acc[6] += d.x; acc[7] += d.y;
      } else {
        acc[0] += __uint_as_float(v[r].x); acc[1] += __uint_as_float(v[r].y);
        acc[2] += __uint_as_float(v[r].z); acc[3] += __uint_as_float(v[r].w);
      }
    }
    uint4 o;
    if constexpr (IS_BF16) {
#pragma unroll
      for (int k = 0; k < VEC; ++k) acc[k] *= scale;
      o.x = pack_bf16x2(acc[0], acc[1]); o.y = pack_bf16x2(acc[2], acc[3]);
      o.z = pack_bf16x2(acc[4], acc[5]); o.w = pack_bf16x2(acc[6], acc[7]);
      // the norm must be that of the values the optimizer will read back (post-rounding)
      float2 a = unpack_bf16x2(o.x), b = unpack_bf16x2(o.y), c = unpack_bf16x2(o.z), d = unpack_bf16x2(o.w);
      ss += a.x * a.x + a.y * a.y + b.x * b.x + b.y * b.y + c.x * c.x + c.y * c.y + d.x * d.x + d.y * d.y;
    } else {
#pragma unroll
      for (int k = 0; k < VEC; ++k) {
        acc[k] *= scale;
        ss += acc[k] * acc[k];
      }
      o.x = __float_as_uint(acc[0]); o.y = __float_as_uint(acc[1]);
      o.z = __float_as_uint(acc[2]); o.w = __float_as_uint(acc[3]);
    }
    *reinterpret_cast<uint4*>(mine + i * 16) = o;
  }
  if (sumsq) {
    ss = block_sum256(ss, sh);
    if (threadIdx.x == 0) atomicAdd(sumsq, ss);
  }
}

template <bool IS_BF16>
__global__ void __launch_bounds__(256) reduce_slice_inplace_dyn_kernel(void* const* bufs, size_t n_slice, int world, int rank,
                                                                      float scale, float* sumsq) {
  __shared__ float sh[32];
  constexpr int VEC = IS_BF16 ? 8 : 4;
  constexpr int ES = IS_BF16 ? 2 : 4;
  uint8_t* mine = reinterpret_cast<uint8_t*>(bufs[rank]) + (size_t)rank * n_slice * ES;
  float ss = 0.f;
  const size_t nvec = n_slice / VEC;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    float acc[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) acc[k] = 0.f;
    for (int r = 0; r < world; ++r) {
      const uint8_t* b = reinterpret_cast<const uint8_t*>(bufs[(rank + r) % world]) + (size_t)rank * n_slice * ES;
      const uint4 v = ld_relaxed_v4(b + i * 16);
      if constexpr (IS_BF16) {
        float2 a = unpack_bf16x2(v.x), bb = unpack_bf16x2(v.y), c = unpack_bf16x2(v.z), d = unpack_bf16x2(v.w);
        acc[0] += a.x; acc[1] += a.y; acc[2] += bb.x; acc[3] += bb.y;
        acc[4] += c.x; acc[5] += c.y; acc[6] += d.x; acc[7] += d.y;
      } else {
        acc[0] += __uint_as_float(v.x); acc[1] += __uint_as_float(v.y);
        acc[2] += __uint_as_float(v.z); acc[3] += __uint_as_float(v.w);
      }
    }
    uint4 o;
    if constexpr (IS_BF16) {
#pragma unroll
      for (int k = 0; k < VEC; ++k) acc[k] *= scale;
      o.x = pack_bf16x2(acc[0], acc[1]); o.y = pack_bf16x2(acc[2], acc[3]);
      o.z = pack_bf16x2(acc[4], acc[5]); o.w = pack_bf16x2(acc[6], acc[7]);
      float2 a = unpack_bf16x2(o.x), bb = unpack_bf16x2(o.y), c = unpack_bf16x2(o.z), d = unpack_bf16x2(o.w);
      ss += a.x * a.x + a.y * a.y + bb.x * bb.x + bb.y * bb.y + c.x * c.x + c.y * c.y + d.x * d.x + d.y * d.y;
    } else {
#pragma unroll
      for (int k = 0; k < VEC; ++k) {
        acc[k] *= scale;
        ss += acc[k] * acc[k];
      }
      o.x = __float_as_uint(acc[0]); o.y = __float_as_uint(acc[1]);
      o.z = __float_as_uint(acc[2]); o.w = __float_as_uint(acc[3]);
    }
    *reinterpret_cast<uint4*>(mine + i * 16) = o;
  }
  if (sumsq) {
    ss = block_sum256(ss, sh);
    if (threadIdx.x == 0) atomicAdd(sumsq, ss);
  }
}

}  // namespace b200

using namespace b200;

// mode: 0 = barrier (post + wait), 1 = post only, 2 = wait only
extern "C" int b200_signal_barrier(uint32_t* const* pads, int world, int rank, uint32_t epoch, int slot_base, int mode,
                                   cudaStream_t s) {
  if (world > 32 || slot_base < 0) return -1;
  if (mode == 0) signal_barrier_kernel<<<1, 32, 0, s>>>(pads, world, rank, epoch, slot_base);
  else if (mode == 1) signal_post_kernel<<<1, 32, 0, s>>>(pads, world, rank, epoch, slot_base);
  else signal_wait_kernel<<<1, 32, 0, s>>>(pads, world, rank, epoch, slot_base);
  return (int)cudaGetLastError();
}

extern "C" int b200_scalar_allreduce_bytes() { return 2 * 32 * SAR_MAXV * (int)sizeof(float) + 2 * 32 * (int)sizeof(uint32_t); }
extern "C" int b200_scalar_allreduce(uint8_t* const* bufs, int world, int rank, uint32_t epoch, float* inout, int nvals,
                                     cudaStream_t s) {
  if (world > 32 || nvals < 1 || nvals > SAR_MAXV) return -1;
  scalar_allreduce_kernel<<<1, 32, 0, s>>>(bufs, world, rank, epoch, inout, nvals);
  return (int)cudaGetLastError();
}

extern "C" int b200_p2p_allgather(const void* const* shard_ptrs, void* full, long long shard_bytes, int world, int rank,
                                  cudaStream_t s) {
  if (shard_bytes % 16) return -1;
  // ~64 CTAs total: enough 16-byte loads in flight to cover NVLink latency x bandwidth, few enough to share
  // the SMs with a concurrently running persistent GEMM
  int per_peer = 64 / world;
  if (per_peer < 1) per_peer = 1;
  p2p_allgather_kernel<<<per_peer * world, 512, 0, s>>>(shard_ptrs, (uint8_t*)full, (size_t)shard_bytes, world, rank);
  return (int)cudaGetLastError();
}

extern "C" int b200_p2p_gather_range(const void* const* shard_ptrs, void* full, long long shard_bytes, long long begin,
                                     long long end, cudaStream_t s) {
  if ((begin % 16) || (end % 16) || end < begin) return -1;
  if (end == begin) return 0;
  long long nvec = (end - begin) / 16;
  int grid = (int)((nvec + 511) / 512);
  if (grid > 64) grid = 64;
  p2p_gather_range_kernel<<<grid, 512, 0, s>>>(shard_ptrs, (uint8_t*)full, (size_t)shard_bytes, (size_t)begin, (size_t)end);
  return (int)cudaGetLastError();
}

extern "C" int b200_p2p_push_range(const void* src, void* const* bases, long long n, long long off, long long len, int rank,
                                   cudaStream_t s) {
  if ((n % 8) || (off % 8) || (len % 8) || len < 0) return -1;
  if (len == 0) return 0;
  int grid = (int)((len / 8 + 255) / 256);
  if (grid > 64) grid = 64;
  p2p_push_range_kernel<<<grid, 256, 0, s>>>((const __nv_bfloat16*)src, bases, (size_t)n, (size_t)off, (size_t)len, rank);
  return (int)cudaGetLastError();
}

// Upper bound on the CTAs of the overlapped reduce kernels.  They run on a side stream UNDER the backward GEMMs (which
// also carry the next unit's all-gather in their comm warps): a full-chip burst steals SM issue slots and NVLink
// ingress exactly when those comm warps need it (measured at 8 GPUs: ag-GEMMs 760 -> 1080 us).  A unit's reduce only
// has to finish within one block's backward (~5 ms), so a few dozen CTAs are enough.
static int g_reduce_max_ctas = 132 * 2;
extern "C" void b200_comm_set_reduce_ctas(int n) { g_reduce_max_ctas = n < 1 ? 1 : n; }

#define RS_CASE(BF, WW) \
  case WW: reduce_scatter_kernel<BF, WW, ACC><<<grid, 256, 0, s>>>(srcs, out, (size_t)n, (size_t)off, rank, scale, sumsq); break;

template <bool ACC>
static void launch_reduce_scatter(const void* const* srcs, float* out, long long n, long long off, int world, int rank,
                                  int src_bf16, float scale, float* sumsq, int grid, cudaStream_t s) {
  if (src_bf16) {
    switch (world) { RS_CASE(true, 1) RS_CASE(true, 2) RS_CASE(true, 4) RS_CASE(true, 8)
      default: reduce_scatter_dyn_kernel<true, ACC><<<grid, 256, 0, s>>>(srcs, out, (size_t)n, (size_t)off, world, rank, scale,
                                                                        sumsq); }
  } else {
    switch (world) { RS_CASE(false, 1) RS_CASE(false, 2) RS_CASE(false, 4) RS_CASE(false, 8)
      default: reduce_scatter_dyn_kernel<false, ACC><<<grid, 256, 0, s>>>(srcs, out, (size_t)n, (size_t)off, world, rank, scale,
                                                                         sumsq); }
  }
}

// accumulate != 0: out += scale * sum (micro-steps 2..k of gradient accumulation)
extern "C" int b200_reduce_scatter(const void* const* srcs, float* out, long long n, long long off, int world, int rank,
                                   int src_bf16, float scale, float* sumsq, int accumulate, cudaStream_t s) {
  const int vec = src_bf16 ? 8 : 4;
  if (n % vec || off % vec) return -1;
  long long nvec = n / vec;
  int grid = (int)((nvec + 255) / 256);
  if (grid > g_reduce_max_ctas) grid = g_reduce_max_ctas;
  if (grid < 1) grid = 1;
  if (accumulate) launch_reduce_scatter<true>(srcs, out, n, off, world, rank, src_bf16, scale, sumsq, grid, s);
  else launch_reduce_scatter<false>(srcs, out, n, off, world, rank, src_bf16, scale, sumsq, grid, s);
  return (int)cudaGetLastError();
}

#define AR_CASE(BF, WW) \
  case WW: reduce_slice_inplace_kernel<BF, WW><<<grid, 256, 0, s>>>(bufs, (size_t)n_slice, rank, scale, sumsq); break;

extern "C" int b200_allreduce_inplace(void* const* bufs, long long numel, int world, int rank, int is_bf16, float scale,
                                      float* sumsq, cudaStream_t s) {
  const int vec = is_bf16 ? 8 : 4;
  if (numel % ((long long)world * vec)) return -1;
  long long n_slice = numel / world;
  long long nvec = n_slice / vec;
  int grid = (int)((nvec + 255) / 256);
  if (grid > 132 * 2) grid = 132 * 2;
  if (grid < 1) grid = 1;
  if (is_bf16) {
    switch (world) { AR_CASE(true, 1) AR_CASE(true, 2) AR_CASE(true, 4) AR_CASE(true, 8)
      default: reduce_slice_inplace_dyn_kernel<true><<<grid, 256, 0, s>>>(bufs, (size_t)n_slice, world, rank, scale, sumsq); }
  } else {
    switch (world) { AR_CASE(false, 1) AR_CASE(false, 2) AR_CASE(false, 4) AR_CASE(false, 8)
      default: reduce_slice_inplace_dyn_kernel<false><<<grid, 256, 0, s>>>(bufs, (size_t)n_slice, world, rank, scale, sumsq); }
  }
  return (int)cudaGetLastError();
}
