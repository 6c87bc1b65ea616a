// Common device/host helpers for the b200vlm kernels (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/b200vlm.h"

namespace b200 {

// ---- error plumbing (C-ABI: int status + b200_last_error()) ---------------
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define B200_CUDA(call)                                                     \
  do {                                                                      \
    cudaError_t _e = (call);                                                \
    if (_e != cudaSuccess) return ::b200::cuda_fail(_e, #call, __FILE__, __LINE__); \
  } while (0)

#define B200_CHECK_LAUNCH()                                                 \
  do {                                                                      \
    cudaError_t _e = cudaGetLastError();                                    \
    if (_e != cudaSuccess) return ::b200::cuda_fail(_e, "kernel launch", __FILE__, __LINE__); \
  } while (0)

#define B200_REQUIRE(cond, ...)                                             \
  do {                                                                      \
    if (!(cond)) { ::b200::set_error(__VA_ARGS__); return B200_ERR_INVALID; } \
  } while (0)

typedef __nv_bfloat16 bf16;

// ---- bf16 rounding points (the oracle's Rounder.r) ------------------------
__device__ __forceinline__ float rbf(float x) {
  return __bfloat162float(__float2bfloat16_rn(x));
}
__device__ __forceinline__ float bf2f(bf16 x) { return __bfloat162float(x); }
__device__ __forceinline__ bf16 f2bf(float x) { return __float2bfloat16_rn(x); }

// unpack 8 bf16 (one 16-byte vector) to 8 floats
__device__ __forceinline__ void unpack8(const uint4& v, float* f) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    f[2 * i] = __uint_as_float(w[i] << 16);
    f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
  }
}
__device__ __forceinline__ void unpack4(const uint2& v, float* f) {
  f[0] = __uint_as_float(v.x << 16);
  f[1] = __uint_as_float(v.x & 0xffff0000u);
  f[2] = __uint_as_float(v.y << 16);
  f[3] = __uint_as_float(v.y & 0xffff0000u);
}
__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
  __nv_bfloat162 p = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&p);
}

// streaming 16-byte load that does not allocate in L1 (weights are read once)
__device__ __forceinline__ uint4 ldg_stream(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- Qwen3-VL q/k norm (qwen3_vl/language.py:59-60,84-89) ------------------
// One attention head of hd = 32 * NU elements held by a warp, lane l owning elements l + 32 u.  mx.fast.rms_norm
// (oracle/mlx_semantics.py): bf16(x * rsqrt(mean(x^2) + eps)) then * w, two roundings.  Every kernel that writes a
// normalised K row (prefill, per-phase decode, lock-step batch) calls this helper, so their rows agree bit for bit.
template <int NU>
__device__ __forceinline__ void warp_head_rms(float (&x)[NU], const bf16* __restrict__ w, float eps) {
  const int lane = threadIdx.x & 31;
  float s = 0.f;
#pragma unroll
  for (int u = 0; u < NU; ++u) s = fmaf(x[u], x[u], s);
  s = warp_sum(s);
  const float rs = 1.0f / sqrtf(s / (float)(32 * NU) + eps);
#pragma unroll
  for (int u = 0; u < NU; ++u) x[u] = rbf(rbf(x[u] * rs) * bf2f(w[lane + 32 * u]));
}
// The rotate_half rotary of the same warp-held head at one position (decode: the three M-RoPE axes agree), three
// roundings like the M-RoPE kernels; element j pairs with j + hd/2, which the same lane holds (hd % 64 == 0).
template <int NU>
__device__ __forceinline__ void warp_head_rope(float (&x)[NU], int pos, const float* __restrict__ inv_freq) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int u = 0; u < NU / 2; ++u) {
    const float ang = (float)pos * inv_freq[lane + 32 * u];
    const float c = rbf(cosf(ang)), sn = rbf(sinf(ang));
    const float y1 = x[u], y2 = x[u + NU / 2];
    x[u] = rbf(rbf(y1 * c) + rbf((-y2) * sn));
    x[u + NU / 2] = rbf(rbf(y2 * c) + rbf(y1 * sn));
  }
}

// ---- activation restatements (oracle/mlx_semantics.py) --------------------
// 1 / (1 + e^-x) with the SFU exponential and reciprocal (branch-free, ~3 ulp): far below the bf16 rounding every
// bf16 caller applies next and below the 2^-17 of the split-operand GEMMs on the fp32 paths (the libm expf + IEEE
// division version has a slow-path branch per element and cost ~9 us per GEMM epilogue)
__device__ __forceinline__ float sigmoid_f(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
// nn.silu(g) * u : three roundings
__device__ __forceinline__ float swiglu_bf(float g, float u) {
  float s = rbf(g * rbf(sigmoid_f(g)));
  return rbf(s * u);
}
// nn.GELU(approx="fast"): x * sigmoid(1.702 x); 1.702 weak-typed to bf16 = 1.703125
__device__ __forceinline__ float gelu_fast_bf(float x) {
  return rbf(x * rbf(sigmoid_f(rbf(1.703125f * x))));
}
// nn.GELU(): x * (1 + erf(x / sqrt2)) / 2; sqrt2 weak-typed to bf16 = 1.4140625
__device__ __forceinline__ float gelu_exact_bf(float x) {
  float a = rbf(x / 1.4140625f);
  float b = rbf(erff(a));
  float c = rbf(1.0f + b);
  float d = rbf(x * c);
  return rbf(d * 0.5f);
}

// sum over a block of NWARPS warps through red[NWARPS]; every thread gets the total
template <int NWARPS>
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < NWARPS; ++w) t += red[w];
  return t;
}
// the same for a warp count known at run time only
__device__ __forceinline__ float block_sum(float v, float* red, int nwarps) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < nwarps; ++w) t += red[w];
  return t;
}

// float -> u32 whose unsigned order is the float order (the high half of a packed argmax key)
__device__ __forceinline__ uint32_t orderable(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// ---- Hopper asynchronous copies: mbarrier, 1-D bulk copy, proxy fence ------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t addr, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(addr), "r"(parity)
      : "memory");
  return done;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done;
  do {
    done = mbar_try_wait(addr, parity);
  } while (!done);
}
// bounded wait (k_mega): a scheduling bug must not hang the GPU (sets *err = 2 and falls through)
__device__ __forceinline__ void mbar_wait_bounded(uint64_t* bar, uint32_t parity, int* err) {
  uint32_t done;
  const uint32_t addr = smem_u32(bar);
  unsigned spins = 0;
  do {
    done = mbar_try_wait(addr, parity);
    if (!done && ++spins > (1u << 20)) {
      *err = 2;
      break;
    }
  } while (!done);
}
// 1-D bulk copy global -> shared through the TMA engine, completing on `bar`, with an L2 cache policy
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar,
                                         uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
// shared-memory writes of the generic proxy (ordinary stores, mbarrier init) become visible to the async proxy
// (TMA, wgmma operands)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

inline int cdiv(long a, long b) { return (int)((a + b - 1) / b); }

// 1-D grid for `work` items of `block` threads each, capped at 16 CTAs per SM of the H100 (grid-stride kernels)
inline int grid_for(long work, int block) {
  long g = (work + block - 1) / block;
  if (g > 132L * 16) g = 132L * 16;
  if (g < 1) g = 1;
  return (int)g;
}

// Function attributes are per (kernel, device).  Raises the kernel's dynamic shared-memory limit to max_dyn_smem
// (when > 0) and asks for the maximum shared-memory carve-out (when max_carveout) on the current device; a value
// already set for this kernel on this device is not set again, so callers may ask before every launch.
int kernel_opt_in(const void* kern, int max_dyn_smem, bool max_carveout);

// ---- programmatic dependent launch -------------------------------------------------
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// Every kernel of the prefill / vision / batched-decode sequences starts with pdl_prologue():
// it lets the NEXT kernel of the stream begin (its barrier set-up and the prefetch of its
// weights overlap this kernel) and then waits until everything the PREVIOUS kernels wrote is visible.
__device__ __forceinline__ void pdl_prologue() {
  pdl_launch_dependents();
  pdl_wait();
}

// ---- launches with attributes ----------------------------------------------------------------
struct LaunchOpts {
  bool pdl;          // programmatic stream serialization: the kernel may start before the previous one ends
  int cluster_x;     // > 0: thread-block clusters of cluster_x x 1 x 1 CTAs
  bool cooperative;  // every CTA resident at once (or the launch fails)
};
constexpr LaunchOpts PDL_LAUNCH = {true, 0, false};

#ifdef __CUDACC__
template <typename... KArgs, typename... Args>
inline cudaError_t launch(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                          LaunchOpts opts, Args... args) {
  cudaLaunchAttribute at[3];
  unsigned n = 0;
  if (opts.pdl) {
    at[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[n++].val.programmaticStreamSerializationAllowed = 1;
  }
  if (opts.cluster_x > 0) {
    at[n].id = cudaLaunchAttributeClusterDimension;
    at[n++].val.clusterDim = {(unsigned)opts.cluster_x, 1, 1};
  }
  if (opts.cooperative) {
    at[n].id = cudaLaunchAttributeCooperative;
    at[n++].val.cooperative = 1;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cfg.attrs = at;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}
#endif

}  // namespace b200
