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

inline int cdiv(long a, long b) { return (int)((a + b - 1) / b); }

// per-DEVICE one-time setup (cudaFuncSetAttribute is per device): true the first time the current device asks
inline bool first_use_on_device(unsigned long long* mask) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return true;
  const unsigned long long bit = 1ull << (dev & 63);
  if (*mask & bit) return false;
  *mask |= bit;
  return true;
}

// ---- programmatic dependent launch -------------------------------------------------
// Every kernel of the prefill / vision / batched-decode sequences starts with pdl_prologue():
// it lets the NEXT kernel of the stream begin (its barrier set-up and the prefetch of its
// weights overlap this kernel) and then waits until everything the PREVIOUS kernels wrote is visible.
__device__ __forceinline__ void pdl_prologue() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
}
#ifdef __CUDACC__
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                              Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}
#endif

}  // namespace b200
