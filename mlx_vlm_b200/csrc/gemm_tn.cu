// C[M,N] = epi(bf16(A[M,K] . W[N,K]^T + bias)) (+ residual) on the Hopper tensor cores:
// TMA (cp.async.bulk.tensor, 128B swizzle) -> shared-memory ring -> wgmma.mma_async (fp32
// accumulators in registers) -> epilogue straight from the registers.  Warp-specialised:
// warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = consumers, 64 rows of the
// 128-row tile each.
//
// Replaces nn.Linear / Conv3d(kernel==stride) / Embedding.as_linear of the
// reference (models/qwen2_vl/vision.py:83-102,108-119,132-133,168-169;
// language.py:52-55; mlp.py:9-15).  Rounding points follow
// oracle/mlx_semantics.py::linear (+ activations, residual add).
#include <mutex>
#include <unordered_map>

#include "common.cuh"
#include "wgmma.cuh"

namespace b200 {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = 128 B = one swizzle row
constexpr int GEMM_THREADS = 384;

struct GemmParams {
  const bf16* bias;
  const bf16* residual;
  bf16* C;
  long ldc, ldr;
  int M, N, K;
  int epilogue;
};

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
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  const uint32_t addr = smem_u32(bar);
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!done);
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%2, %3}], [%4];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}

template <int BN>
struct GemmSmem {
  static constexpr int STAGES = (BN == 128) ? 6 : 8;
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int RING = STAGES * (A_BYTES + B_BYTES);
  static constexpr int TOTAL = RING + 1024 /*align slack*/ + 256 /*barriers*/;
};

template <int BN>
__device__ __forceinline__ void gemm_mma(float (&acc)[BN / 2], uint64_t da, uint64_t db) {
  if constexpr (BN == 128) wgmma_n128_ss(acc, da, db, 1u);
  else wgmma_n64_ss(acc, da, db, 1u);
}

template <int BN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tn_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const GemmParams p) {
  using L = GemmSmem<BN>;
  constexpr int STAGES = L::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * L::A_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::RING);
  uint64_t* empty_bar = full_bar + STAGES;

  const int wg = threadIdx.x >> 7;
  const int n_blk = blockIdx.x, m_blk = blockIdx.y;
  const int num_k = (p.K + BK - 1) / BK;

  // The producer thread initialises the barriers itself and puts the first STAGES loads in
  // flight before the CTA-wide setup barrier.
  const int pre_k = num_k < STAGES ? num_k : STAGES;
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmB)) : "memory");
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);  // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    for (int k = 0; k < pre_k; ++k) {
      mbar_expect_tx(&full_bar[k], L::A_BYTES + L::B_BYTES);
      tma_load_2d(sA + k * L::A_BYTES, &tmA, &full_bar[k], k * BK, m_blk * BM);
      tma_load_2d(sB + k * L::B_BYTES, &tmB, &full_bar[k], k * BK, n_blk * BN);
    }
  }
  __syncthreads();

  if (wg == 0) {
    if (threadIdx.x == 0) {  // ===== TMA producer (the first pre_k stages are already in flight) =====
      for (int k = pre_k; k < num_k; ++k) {
        const int s = k % STAGES;
        const uint32_t ph = (k / STAGES) & 1;
        mbar_wait(&empty_bar[s], ph ^ 1);
        mbar_expect_tx(&full_bar[s], L::A_BYTES + L::B_BYTES);
        tma_load_2d(sA + s * L::A_BYTES, &tmA, &full_bar[s], k * BK, m_blk * BM);
        tma_load_2d(sB + s * L::B_BYTES, &tmB, &full_bar[s], k * BK, n_blk * BN);
      }
    }
    return;
  }

  // ===== consumers: warpgroup c = wg - 1 owns rows [64 c, 64 c + 64) of the tile =====
  const int c = wg - 1;
  const int t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  for (int k = 0; k < num_k; ++k) {
    const int s = k % STAGES;
    mbar_wait(&full_bar[s], (k / STAGES) & 1);
    const uint32_t a0 = wg_smem(sA + s * L::A_BYTES + c * 64 * 128);
    const uint32_t b0 = wg_smem(sB + s * L::B_BYTES);
    wg_fence_acc(acc);
    wg_arrive();
#pragma unroll
    for (int kk = 0; kk < BK / 16; ++kk) gemm_mma<BN>(acc, wg_desc(a0 + kk * 32), wg_desc(b0 + kk * 32));
    wg_commit();
    wg_wait<0>();
    wg_fence_acc(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s]);  // this warp's MMAs have read the slot
  }

  // ===== epilogue: registers -> bias/activation/residual -> global (pairs of columns) =====
  const bool vec_ok = ((p.ldc & 1) == 0) && (!p.residual || (p.ldr & 1) == 0) &&
                      ((reinterpret_cast<uintptr_t>(p.C) & 3) == 0) &&
                      (!p.residual || (reinterpret_cast<uintptr_t>(p.residual) & 3) == 0);
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int row = m_blk * BM + c * 64 + warp * 16 + (lane >> 2) + 8 * hr;
    if (row >= p.M) continue;
    bf16* crow = p.C + (long)row * p.ldc;
    const bf16* rrow = p.residual ? p.residual + (long)row * p.ldr : nullptr;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int n = n_blk * BN + j * 8 + 2 * (lane & 3);
      if (n >= p.N) continue;
      float v[2] = {acc[j * 4 + hr * 2], acc[j * 4 + hr * 2 + 1]};
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        if (p.bias && n + e < p.N) v[e] += bf2f(p.bias[n + e]);
        v[e] = rbf(v[e]);
        if (p.epilogue == B200_EPI_GELU_FAST) v[e] = gelu_fast_bf(v[e]);
        else if (p.epilogue == B200_EPI_GELU_EXACT) v[e] = gelu_exact_bf(v[e]);
      }
      if (n + 2 <= p.N && vec_ok) {
        if (rrow) {
          float rf[2];
          const uint32_t rw = *reinterpret_cast<const uint32_t*>(rrow + n);
          rf[0] = __uint_as_float(rw << 16);
          rf[1] = __uint_as_float(rw & 0xffff0000u);
          v[0] = rbf(rf[0] + v[0]);
          v[1] = rbf(rf[1] + v[1]);
        }
        *reinterpret_cast<uint32_t*>(crow + n) = pack2(v[0], v[1]);
      } else {
        for (int e = 0; e < 2 && n + e < p.N; ++e) {
          float o = v[e];
          if (rrow) o = rbf(bf2f(rrow[n + e]) + o);
          crow[n + e] = f2bf(o);
        }
      }
    }
  }
}

// ---- host: tensor maps ------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) ==
            cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

struct TmapKey {
  const void* ptr;
  long ld;
  int rows, k, box_rows;
  bool operator==(const TmapKey& o) const {
    return ptr == o.ptr && ld == o.ld && rows == o.rows && k == o.k && box_rows == o.box_rows;
  }
};
struct TmapHash {
  size_t operator()(const TmapKey& k) const {
    size_t h = std::hash<const void*>()(k.ptr);
    h = h * 1000003u ^ std::hash<long>()(k.ld);
    h = h * 1000003u ^ (size_t)k.rows;
    h = h * 1000003u ^ (size_t)k.k;
    h = h * 1000003u ^ (size_t)k.box_rows;
    return h;
  }
};

// 2-D K-major bf16 operand (rows x K, row pitch ld elements), box = box_rows x 64.
static int get_tmap(const void* ptr, long ld, int rows, int k, int box_rows, CUtensorMap* out) {
  static std::unordered_map<TmapKey, CUtensorMap, TmapHash> cache;
  static std::mutex mu;
  TmapKey key{ptr, ld, rows, k, box_rows};
  {
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(key);
    if (it != cache.end()) {
      *out = it->second;
      return B200_OK;
    }
  }
  EncodeTiledFn enc = get_encode();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return B200_ERR_CUDA;
  }
  cuuint64_t gdim[2] = {(cuuint64_t)k, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUtensorMap tm;
  CUresult r = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim, gstr,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d) ptr=%p ld=%ld rows=%d k=%d", (int)r, ptr, ld,
              rows, k);
    return B200_ERR_CUDA;
  }
  {
    std::lock_guard<std::mutex> g(mu);
    if (cache.size() > 8192) cache.clear();
    cache[key] = tm;
  }
  *out = tm;
  return B200_OK;
}

template <int BN>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p,
                       cudaStream_t st) {
  static unsigned long long attr_mask = 0ull;
  if (first_use_on_device(&attr_mask)) {
    B200_CUDA(cudaFuncSetAttribute(gemm_tn_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   GemmSmem<BN>::TOTAL));
  }
  dim3 grid(cdiv(p.N, BN), cdiv(p.M, BM));
  gemm_tn_kernel<BN><<<grid, GEMM_THREADS, GemmSmem<BN>::TOTAL, st>>>(ta, tb, p);
  B200_CHECK_LAUNCH();
  return B200_OK;
}

int gemm_bf16_tn(const void* A, long lda, const void* W, const void* bias, const void* residual,
                 long ldr, void* C, long ldc, int M, int N, int K, int epilogue,
                 cudaStream_t st) {
  B200_REQUIRE(M > 0 && N > 0 && K > 0, "gemm: empty problem M=%d N=%d K=%d", M, N, K);
  B200_REQUIRE((lda % 8) == 0 && (K % 8) == 0, "gemm: lda (%ld) and K (%d) must be multiples of 8",
               lda, K);
  B200_REQUIRE(((uintptr_t)A & 15) == 0 && ((uintptr_t)W & 15) == 0,
               "gemm: A and W must be 16-byte aligned");
  B200_REQUIRE(epilogue >= 0 && epilogue <= 2, "gemm: bad epilogue %d", epilogue);
  // pick the N tile so that the grid covers the 132 SMs when M is small
  const long tiles128 = (long)cdiv(M, BM) * cdiv(N, 128);
  const int bn = (tiles128 >= 112 && (N % 128) == 0) ? 128 : 64;
  CUtensorMap ta, tb;
  int rc = get_tmap(A, lda, M, K, BM, &ta);
  if (rc) return rc;
  rc = get_tmap(W, (long)K, N, K, bn, &tb);
  if (rc) return rc;
  GemmParams p{(const bf16*)bias, (const bf16*)residual, (bf16*)C, ldc, ldr, M, N, K, epilogue};
  return bn == 128 ? launch_gemm<128>(ta, tb, p, st) : launch_gemm<64>(ta, tb, p, st);
}

}  // namespace b200

extern "C" int b200_gemm_bf16_tn(const void* A, long lda, const void* W, const void* bias,
                                 const void* residual, long ldr, void* C, long ldc, int M, int N,
                                 int K, int epilogue, void* stream) {
  return b200::gemm_bf16_tn(A, lda, W, bias, residual, ldr, C, ldc, M, N, K, epilogue,
                            (cudaStream_t)stream);
}
