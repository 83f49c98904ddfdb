// kernels_wg.cu -- row GEMMs on the Hopper tensor cores (wgmma, sm_90a): the CHGNet projections and their transposes,
// the TensorNet edge MLP and distance projection, and the dense MACE products (with SiLU / SiLU' epilogues).  Weights of
// any [K][N] shape (multiples of 64) are split into this kernel's three block shapes on the host (engine.cu pack_tc, tc_mm).
//
//   * 3xTF32 split (hi*hi + lo*hi + hi*lo, fp32 accumulate in registers) keeps fp32-level accuracy;
//   * a CTA of two warpgroups owns 128-row tiles (persistent over the grid); warpgroup w multiplies rows 64w .. 64w+63
//     against all N columns (m64nNk8), both operands from shared memory;
//   * B (the weights) is pre-formatted on the host into the canonical K-major / no-swizzle core-matrix layout (8 rows x
//     16 B, hi and lo planes; engine.cu canon_split) and staged once per CTA;
//   * A is read in 64-column K chunks by coalesced float4 loads, split into tf32 hi / lo and stored in the same
//     core-matrix layout; the loads of the NEXT chunk are issued before the MMAs of the current one, so they are in
//     flight while the tensor core works;
//   * the epilogue (bias, residual / accumulate, SiLU / SiLU') runs on the accumulator registers and writes C directly
//     (each quad of threads writes 32 contiguous bytes of a row).
#include "kernels.cuh"
#include "wgmma.cuh"

namespace b2m {


// EPI (TensorNet edge MLP): 1 = keep the pre-activation in Cpre and write SiLU(value); 2 = value *= SiLU'(Pre[row][col])
// (reverse pass; applied after the accumulate, so the last K-chunk of a split product carries it).
template <int K, int N, int EPI>
__global__ void __launch_bounds__(256, 1)
    k_gemm_wg(const float* __restrict__ A, int lda, const float* __restrict__ Bcan, float* __restrict__ C, int ldc, int M,
              const float* __restrict__ bias, const float* __restrict__ R, int ldr, int accum, float* __restrict__ Cpre,
              const float* __restrict__ Pre, int ldp) {
  constexpr int KH = K / 64;
  constexpr int NR = N / 2;                           // accumulator registers per thread (m64nN, f32)
  constexpr uint32_t LBO_B = (N / 8) * 128;           // B: byte step between core matrices along K
  constexpr uint32_t LBO_A = (128 / 8) * 128;         // A chunk [128 rows][64 k]: same layout with 128 rows
  constexpr uint32_t A_PLANE = 128 * 64 * 4;          // bytes of one (hi or lo) A plane
  extern __shared__ __align__(1024) float smem[];
  float* Bs = smem;                 // [2][N*K]  hi | lo
  float* As = smem + 2 * N * K;     // [2][128*64] hi | lo
  const int tid = threadIdx.x, wg = tid >> 7, wt = tid & 127;
  const int warp = wt >> 5, lane = tid & 31;
  const int ntiles = (M + 127) / 128;

  // my share of a chunk: 8 float4, float4 f = tid + 256 i -> row (f >> 7) * 8 + (f & 7), k4 = (f >> 3) & 15
  // (8 consecutive lanes fill one 128-byte core-matrix column: conflict-free 16-byte stores)
  float4 pre[8];
  auto load_chunk = [&](int t, int kh) {
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const int f = tid + 256 * i;
      const int row = t * 128 + (f >> 7) * 8 + (f & 7);
      pre[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row < M) pre[i] = *reinterpret_cast<const float4*>(A + (size_t)row * lda + kh * 64 + ((f >> 3) & 15) * 4);
    }
  };
  if ((int)blockIdx.x < ntiles) load_chunk(blockIdx.x, 0);  // in flight while the weights are staged
  for (int i = tid; i < 2 * N * K / 4; i += 256) reinterpret_cast<float4*>(Bs)[i] = reinterpret_cast<const float4*>(Bcan)[i];
  const uint32_t a_addr = s_u32(As) + (uint32_t)wg * 1024u, b_addr = s_u32(Bs);

  float d[NR];
  for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int row0 = t * 128;
#pragma unroll 1
    for (int kh = 0; kh < KH; kh++) {
      __syncthreads();  // both warpgroups are done with the previous chunk (and the weights are staged)
#pragma unroll
      for (int i = 0; i < 8; i++) {
        const int f = tid + 256 * i;
        const int off = (((f >> 3) & 15) * 16 + (f >> 7)) * 32 + (f & 7) * 4;  // ((k/4) * 16 + m/8) * 32 + (m%8) * 4
        const float xv[4] = {pre[i].x, pre[i].y, pre[i].z, pre[i].w};
        uint32_t h[4], l[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
          h[j] = tf32_hi_bits(xv[j]);
          l[j] = __float_as_uint(xv[j] - __uint_as_float(h[j]));
        }
        *reinterpret_cast<uint4*>(As + off) = make_uint4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<uint4*>(As + 128 * 64 + off) = make_uint4(l[0], l[1], l[2], l[3]);
      }
      fence_proxy_async_smem();
      __syncthreads();
      // next chunk: the other K half of this tile, or the first half of my next tile
      if (kh + 1 < KH)
        load_chunk(t, kh + 1);
      else if (t + (int)gridDim.x < ntiles)
        load_chunk(t + gridDim.x, 0);
      acc_fence(d);
      wgmma_fence();
#pragma unroll
      for (int term = 0; term < 3; term++) {
        const uint32_t asel = a_addr + (term == 1 ? A_PLANE : 0u);
        const uint32_t bsel = b_addr + (term == 2 ? (uint32_t)(N * K) * 4u : 0u) + (uint32_t)kh * 16u * LBO_B;
#pragma unroll
        for (int ks = 0; ks < 8; ks++) {
          const uint64_t ad = gmma_desc(asel + ks * 2 * LBO_A, LBO_A, 128u);
          const uint64_t bd = gmma_desc(bsel + ks * 2 * LBO_B, LBO_B, 128u);
          const int scale_d = (kh > 0 || term > 0 || ks > 0) ? 1 : 0;
          if constexpr (N == 128)
            wgmma_tf32_n128(d, ad, bd, scale_d);
          else
            wgmma_tf32_n64(d, ad, bd, scale_d);
        }
      }
      wgmma_commit();
      wgmma_wait_all();
      acc_fence(d);
    }
    // epilogue from the accumulator fragment: d[4j + 2h + {0,1}] = (row wbase + 8h, cols 8j + 2(lane%4) + {0,1})
    const int rbase = row0 + wg * 64 + warp * 16 + (lane >> 2);
    const float* addsrc = R ? R : (accum ? C : nullptr);
    const int addld = R ? ldr : ldc;
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int row = rbase + 8 * h;
      if (row >= M) continue;
#pragma unroll
      for (int j = 0; j < N / 8; j++) {
        const int col = 8 * j + 2 * (lane & 3);
        float2 o = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
        if (bias) {
          const float2 b = *reinterpret_cast<const float2*>(bias + col);
          o.x += b.x, o.y += b.y;
        }
        if (addsrc) {
          const float2 x = *reinterpret_cast<const float2*>(addsrc + (size_t)row * addld + col);
          o.x += x.x, o.y += x.y;
        }
        float2* cp = reinterpret_cast<float2*>(C + (size_t)row * ldc + col);
        if (R && accum) {  // both at once (not used by the engine): the accumulate read stays in place
          const float2 c = *cp;
          o.x += c.x, o.y += c.y;
        }
        if constexpr (EPI == 1) {
          *reinterpret_cast<float2*>(Cpre + (size_t)row * ldc + col) = o;
          o = make_float2(silu_(o.x), silu_(o.y));
        } else if constexpr (EPI == 2) {
          const float2 pv = *reinterpret_cast<const float2*>(Pre + (size_t)row * ldp + col);
          o.x *= dsilu_(pv.x), o.y *= dsilu_(pv.y);
        }
        *cp = o;
      }
    }
  }
}

template <int K, int N, int EPI>
static void launch_gemm_wg_t(cudaStream_t st, const float* A, int lda, const float* Bcan, float* C, int ldc, int M,
                             const float* bias, const float* R, int ldr, bool accum, float* Cpre, const float* Pre,
                             int ldp, int num_sms) {
  constexpr size_t bytes = (size_t)(2 * N * K + 2 * 128 * 64) * 4;
  static_assert(bytes <= 232448, "shared memory budget");
  constexpr int per_sm = bytes <= 232448 / 2 - 1024 ? 2 : 1;
  static PerDeviceOnce attr;
  if (auto once_ = attr.first(); once_)
    B2M_CK(cudaFuncSetAttribute(k_gemm_wg<K, N, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  // float4 loads of A rows and of the weights, float2 epilogue accesses of C / bias / R / Cpre / Pre
  auto al = [](const void* p, uintptr_t n) { return p == nullptr || (((uintptr_t)p) & (n - 1)) == 0; };
  B2M_REQUIRE(lda % 4 == 0 && ldc % 2 == 0 && (R == nullptr || ldr % 2 == 0) && (Pre == nullptr || ldp % 2 == 0) &&
                  al(A, 16) && al(Bcan, 16) && al(C, 8) && al(bias, 8) && al(R, 8) && al(Cpre, 8) && al(Pre, 8),
              B2M_ERR_INVALID, "gemm_wg operand alignment");
  const int ntiles = (M + 127) / 128;
  launch(k_gemm_wg<K, N, EPI>, std::min(ntiles, per_sm * num_sms), 256, bytes, st, A, lda, Bcan, C, ldc, M, bias, R, ldr,
         accum ? 1 : 0, Cpre, Pre, ldp);
}

template <int EPI>
static void launch_gemm_wg_s(cudaStream_t st, const float* A, int lda, const float* Bcan, float* C, int ldc, int M, int N,
                             int K, const float* bias, const float* R, int ldr, bool accum, float* Cpre, const float* Pre,
                             int ldp, int num_sms) {
  if (K == 64 && N == 128)
    launch_gemm_wg_t<64, 128, EPI>(st, A, lda, Bcan, C, ldc, M, bias, R, ldr, accum, Cpre, Pre, ldp, num_sms);
  else if (K == 64 && N == 64)
    launch_gemm_wg_t<64, 64, EPI>(st, A, lda, Bcan, C, ldc, M, bias, R, ldr, accum, Cpre, Pre, ldp, num_sms);
  else if (K == 128 && N == 64)
    launch_gemm_wg_t<128, 64, EPI>(st, A, lda, Bcan, C, ldc, M, bias, R, ldr, accum, Cpre, Pre, ldp, num_sms);
  else
    throw Error(B2M_ERR_INVALID, "gemm_wg shape");
}

void launch_gemm_wg(cudaStream_t st, const float* A, int lda, const float* Bcan, float* C, int ldc, int M, int N, int K,
                    const float* bias, const float* R, int ldr, bool accum, int epi, float* Cpre, const float* Pre,
                    int ldp, int num_sms) {
  if (M <= 0) return;
  B2M_REQUIRE(epi == 1 ? Cpre != nullptr : (epi == 2 ? Pre != nullptr : epi == 0), B2M_ERR_INVALID, "gemm_wg epilogue");
  if (epi == 1)
    launch_gemm_wg_s<1>(st, A, lda, Bcan, C, ldc, M, N, K, bias, R, ldr, accum, Cpre, Pre, ldp, num_sms);
  else if (epi == 2)
    launch_gemm_wg_s<2>(st, A, lda, Bcan, C, ldc, M, N, K, bias, R, ldr, accum, Cpre, Pre, ldp, num_sms);
  else
    launch_gemm_wg_s<0>(st, A, lda, Bcan, C, ldc, M, N, K, bias, R, ldr, accum, Cpre, Pre, ldp, num_sms);
}

}  // namespace b2m
