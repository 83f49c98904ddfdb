// kernels.cu -- hand-written sm_90a kernels of the CHGNet hot path (fp32 FFMA math,
// cp.async.bulk (TMA) row gathers into shared memory, segmented scatter-adds).
// See kernels.cuh for the formulation; oracle/manual_ref.py is the CPU mirror of every stage.
#include "final_tail.cuh"
#include "kernels.cuh"
#include "wgmma.cuh"

#include <algorithm>

namespace b2m {

// ============================================================================================
// device helpers
// ============================================================================================
// MUFU.EX2 + MUFU.RCP, flush-to-zero forms (same bits as __fdividef/__expf for normal results, no range fix-ups)
__device__ __forceinline__ float sigm(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.f + e));
  return r;
}
__device__ __forceinline__ float silu_f(float x) { return x * sigm(x); }
__device__ __forceinline__ float dsilu_f(float x) {
  float s = sigm(x);
  return s * (1.f + x * (1.f - s));
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// TMA bulk copy global -> shared (one row), completion signalled on an mbarrier
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  const uint32_t addr = smem_u32(bar);
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!ok);
}
// a double-buffered stage: tile number `it` of a CTA sits in buffer it & 1, whose mbarrier completes one phase per fill,
// so that tile's consumer waits on parity (it >> 1) & 1
__device__ __forceinline__ uint32_t stage_parity(int it) { return (uint32_t)(it >> 1) & 1u; }
// one thread: a weight image (bytes a multiple of 16 KB) as 16 KB bulk copies completing on `bar`
__device__ __forceinline__ void bulk_g2s_image(float* dst, const float* src, uint32_t bytes, uint64_t* bar) {
  mbar_expect_tx(bar, bytes);
  for (uint32_t o = 0; o < bytes; o += 16384u) bulk_g2s(dst + o / 4, src + o / 4, 16384u, bar);
}

__device__ __forceinline__ float ipowf(float x, int n) {
  float r = 1.f;
  for (int i = 0; i < n; i++) r *= x;
  return r;
}
// be_k = env(rbf_k) rbf_k with the envelope applied to the rbf VALUE (chgnet.py:116-124), and d be_k / dd
__device__ __forceinline__ void rbf_env_k(float d, float freq, const RadialParams& rp, float& be, float& dbe) {
  const float invd = 1.f / d;
  const float w = freq / rp.rc;
  float s, c;
  sincosf(d * w, &s, &c);
  const float rbf = rp.norm * s * invd;
  const float drbf = rp.norm * (w * c * invd - s * invd * invd);
  const int p = rp.p;
  const float c1 = -(p + 1) * (p + 2) * 0.5f, c2 = (float)(p * (p + 2)), c3 = -p * (p + 1) * 0.5f;
  const float rho = rbf / rp.rc;
  const float rm1 = ipowf(rho, p - 1);
  const float r0 = rm1 * rho, r1 = r0 * rho, r2 = r1 * rho;
  const float env = 1.f + c1 * r0 + c2 * r1 + c3 * r2;
  const float denv = (c1 * p * rm1 + c2 * (p + 1) * r0 + c3 * (p + 2) * r1) / rp.rc;
  const bool ok = rbf <= rp.rc;
  be = ok ? env * rbf : 0.f;
  dbe = ok ? (env + rbf * denv) * drbf : 0.f;
}

// thread -> accumulator mapping of the 256-thread fused kernels: branch = warpgroup = tid>>7 (0: "layers", 1: "gates");
// a warpgroup's 128 x 64 product is two m64n64 wgmma fragments, so thread (warp w, lane l) owns rows
// r_i = 64 (i>>1) + 16 w + l/4 + 8 (i&1), i < 4, and columns c_j = 8 (j>>1) + 2 (l%4) + (j&1), j < 16
constexpr int AR = 4, AC = 16;
struct Map {
  int branch, rb, cb;
  __device__ __forceinline__ Map() {
    const int tid = threadIdx.x;
    branch = tid >> 7;
    const int lane = tid & 31;
    rb = ((tid & 127) >> 5) * 16 + (lane >> 2);
    cb = 2 * (lane & 3);
  }
  __device__ __forceinline__ int row(int i) const { return 64 * (i >> 1) + rb + 8 * (i & 1); }
  __device__ __forceinline__ int col(int j) const { return 8 * (j >> 1) + cb + (j & 1); }
};

// d = (accumulate ? d : 0) + A . B[0..63][bk .. bk+64)^T on the tensor cores (warpgroup-collective), 3xTF32 (hi.hi +
// lo.hi + hi.lo, fp32 accumulate).  x[ks]: this thread's fp32 A fragment of k block ks in the instruction's order
// (rows 16 w + l/4 and + 8 of the 64-row block, k slots l%4 and l%4 + 4).  B: canonical K-major [64 n][K k] image in
// shared memory, tf32 hi plane at b_hi and lo plane at b_lo, k permuted inside each block of 8 (slot q <- column 2q,
// slot q + 4 <- column 2q + 1; engine.cu: permute_k8), so that slots l%4 and l%4 + 4 take A's columns 8 ks + 2 (l%4)
// and + 1: the pair a thread holds in the accumulator layout, or reads from a tile as one float2.  KB < 8: the first KB
// k blocks only (the rank-9 radial products take one, K = 8).
template <int KB>
__device__ __forceinline__ void wg_mma64(const float (&x)[KB][4], uint32_t b_hi, uint32_t b_lo, int bk, bool accumulate,
                                         float (&d)[32]) {
  constexpr uint32_t LBO = 8 * 128;  // byte step between core matrices along K (N = 64)
  uint32_t ah[KB][4], al[KB][4];
#pragma unroll
  for (int ks = 0; ks < KB; ks++)
#pragma unroll
    for (int q = 0; q < 4; q++) {
      ah[ks][q] = tf32_hi_bits(x[ks][q]);
      al[ks][q] = __float_as_uint(x[ks][q] - __uint_as_float(ah[ks][q]));
    }
  const uint32_t koff = (uint32_t)(bk / 4) * LBO;
  acc_fence(d);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < KB; ks++) {
#pragma unroll
    for (int term = 0; term < 3; term++) {
      const uint64_t bd = gmma_desc((term == 2 ? b_lo : b_hi) + koff + ks * 2 * LBO, LBO, 128u);
      wgmma_tf32_n64_rA(d, term == 1 ? al[ks] : ah[ks], bd, (accumulate || ks > 0 || term > 0) ? 1 : 0);
    }
  }
  wgmma_commit();
  wgmma_wait_all();
  acc_fence(d);
}

// d = (accumulate ? d : 0) + At[row0 .. row0+63][acol .. acol+64) . B[0..63][bk .. bk+64)^T (wg_mma64).  At: fp32 in
// shared memory, row pitch lda; each k pair is one float2 read, and lda % 32 == 8 puts the 8 rows x 4 pairs of a
// half-warp on 32 distinct banks.
__device__ __forceinline__ void wg_mm64(const float* At, int lda, int row0, int acol, uint32_t b_hi, uint32_t b_lo,
                                        int bk, bool accumulate, float (&d)[32]) {
  const int lane = threadIdx.x & 31;
  const float* p0 = At + (row0 + ((threadIdx.x & 127) >> 5) * 16 + (lane >> 2)) * lda + acol + 2 * (lane & 3);
  const float* p1 = p0 + 8 * lda;
  float x[8][4];
#pragma unroll
  for (int ks = 0; ks < 8; ks++) {
    const float2 u = *reinterpret_cast<const float2*>(p0 + 8 * ks), v = *reinterpret_cast<const float2*>(p1 + 8 * ks);
    x[ks][0] = u.x, x[ks][1] = v.x, x[ks][2] = u.y, x[ks][3] = v.y;
  }
  wg_mma64(x, b_hi, b_lo, bk, accumulate, d);
}

// acc (Map layout) = At[0..127][kofs .. kofs+64) . B^T for this thread's branch; Bcan: the branch's canonical image
// (hi plane of 4096 floats, then lo plane)
__device__ __forceinline__ void gemm64(const float* At, int lda, int kofs, const float* Bcan, float (&acc)[AR][AC]) {
  const uint32_t bh = s_u32(Bcan), bl = bh + 4096u * 4u;
#pragma unroll
  for (int h = 0; h < 2; h++) {
    float d[32];
    wg_mm64(At, lda, 64 * h, kofs, bh, bl, 0, false, d);
#pragma unroll
    for (int q = 0; q < 32; q++) acc[2 * h + ((q >> 1) & 1)][2 * (q >> 2) + (q & 1)] = d[q];
  }
}

// weights -> shared memory; the fence makes the generic-proxy stores visible to wgmma after the next barrier
template <int NTH = NT>
__device__ __forceinline__ void stage_w(float* Wsm, const float* __restrict__ g, int nfloat4) {
  for (int i = threadIdx.x; i < nfloat4; i += NTH) reinterpret_cast<float4*>(Wsm)[i] = reinterpret_cast<const float4*>(g)[i];
  fence_proxy_async_smem();
}

// ============================================================================================
// small elementwise / init kernels
// ============================================================================================
__global__ void k_embed(int n, const int* __restrict__ type, const float* __restrict__ emb, float* __restrict__ x0) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)n * 16) return;
  const int r = (int)(i >> 4), c4 = (int)(i & 15);
  reinterpret_cast<float4*>(x0)[(size_t)r * 16 + c4] = reinterpret_cast<const float4*>(emb)[(size_t)type[r] * 16 + c4];
}
void launch_embed(cudaStream_t st, int n, const int* type, const float* emb, float* x0) {
  launch(k_embed, cdiv((int64_t)n * 16, 256), 256, 0, st, n, type, emb, x0);
}

// out[b][c] = sum_k be_k(d_b) W[c][k]     (32 bonds per block)
__global__ void __launch_bounds__(256) k_bond_init(int nb, const float4* __restrict__ b_vec, RadialParams rp,
                                                   const float* __restrict__ W, float* __restrict__ out) {
  __shared__ float be_s[32][12];
  __shared__ float Ws[64 * 9];
  const int b0 = blockIdx.x * 32, tid = threadIdx.x;
  for (int i = tid; i < 576; i += 256) Ws[i] = W[i];
  for (int i = tid; i < 32 * 9; i += 256) {
    const int r = i / 9, k = i % 9;
    float be = 0.f, dbe;
    if (b0 + r < nb) rbf_env_k(b_vec[b0 + r].w, rp.freq[k], rp, be, dbe);
    be_s[r][k] = be;
  }
  __syncthreads();
  for (int i = tid; i < 32 * 64; i += 256) {
    const int r = i >> 6, c = i & 63;
    if (b0 + r >= nb) continue;
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 9; k++) s = fmaf(be_s[r][k], Ws[c * 9 + k], s);
    out[(size_t)(b0 + r) * 64 + c] = s;
  }
}
void launch_bond_init(cudaStream_t st, int nb, const float4* b_vec, RadialParams rp, const float* W, float* out) {
  launch(k_bond_init, cdiv(nb, 32), 256, 0, st, nb, b_vec, rp, W, out);
}

struct AngleGeom {
  float cos_raw, cc, theta, na, nb;
  float va[3], vb[3];
};
__device__ __forceinline__ AngleGeom angle_geom(const float4 a, const float4 b) {
  // compute_theta with src_bond_sign = -1 (chgnet.py:190-194; SURVEY 9): cos = (-va . vb) / (|va||vb|)
  AngleGeom g;
  g.va[0] = a.x, g.va[1] = a.y, g.va[2] = a.z;
  g.vb[0] = b.x, g.vb[1] = b.y, g.vb[2] = b.z;
  g.na = sqrtf(a.x * a.x + a.y * a.y + a.z * a.z);
  g.nb = sqrtf(b.x * b.x + b.y * b.y + b.z * b.z);
  g.cos_raw = -(a.x * b.x + a.y * b.y + a.z * b.z) / (g.na * g.nb);
  const float lo = -1.f + 1e-7f, hi = 1.f - 1e-7f;
  g.cc = fminf(fmaxf(g.cos_raw, lo), hi);
  g.theta = acosf(g.cc);
  return g;
}

// ang0[r][c] = sum_k fourier_k(theta_r) Wae[c][k]      (128 angles per block)
__global__ void __launch_bounds__(256) k_angle_init(int64_t na, const int* __restrict__ a_in,
                                                    const int* __restrict__ a_out, const float4* __restrict__ b_vec,
                                                    const float* __restrict__ fa, const float* __restrict__ Wae,
                                                    float* __restrict__ ang0) {
  __shared__ float f_s[128][12];
  __shared__ float Ws[64 * 9];
  const int64_t r0 = (int64_t)blockIdx.x * 128;
  const int tid = threadIdx.x;
  for (int i = tid; i < 576; i += 256) Ws[i] = Wae[i];
  if (tid < 128) {
    const int64_t r = r0 + tid;
    if (r < na) {
      const AngleGeom g = angle_geom(b_vec[a_in[r]], b_vec[a_out[r]]);
      const float ipi = 0.318309886183790672f;
      // even columns cos(f_k theta), odd columns sin(f_k theta) (k>=1), all / pi   (SURVEY 9)
      for (int k = 0; k < 5; k++) {
        float s, c;
        sincosf(g.theta * fa[k], &s, &c);
        f_s[tid][2 * k] = c * ipi;
        if (k >= 1) f_s[tid][2 * k - 1] = s * ipi;
      }
    } else {
      for (int k = 0; k < 9; k++) f_s[tid][k] = 0.f;
    }
  }
  __syncthreads();
  for (int i = tid; i < 16 * 128; i += 256) {  // (4 columns, row): consecutive lanes = consecutive rows
    const int cq = i >> 7, r = i & 127;
    if (r0 + r >= na) continue;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 9; k++) {
      const float f = f_s[r][k];
#pragma unroll
      for (int j = 0; j < 4; j++) v[j] = fmaf(f, Ws[(4 * cq + j) * 9 + k], v[j]);
    }
    *reinterpret_cast<float4*>(ang0 + (size_t)(r0 + r) * 64 + 4 * cq) = make_float4(v[0], v[1], v[2], v[3]);
  }
}
void launch_angle_init(cudaStream_t st, int64_t na, const int* a_in, const int* a_out, const float4* b_vec,
                       const float* fa, const float* Wae, float* ang0) {
  launch(k_angle_init, cdiv(na, 128), 256, 0, st, na, a_in, a_out, b_vec, fa, Wae, ang0);
}

__global__ void k_silu(int64_t n, const float* __restrict__ pre, float* __restrict__ out) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) out[i] = silu_f(pre[i]);
}
__global__ void k_dsilu_mul(int64_t n, const float* __restrict__ pre, float* __restrict__ g) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) g[i] *= dsilu_f(pre[i]);
}
void launch_silu(cudaStream_t st, int64_t n, const float* pre, float* out) {
  launch(k_silu, cdiv(n, 256), 256, 0, st, n, pre, out);
}
void launch_dsilu_mul(cudaStream_t st, int64_t n, const float* pre, float* g) {
  launch(k_dsilu_mul, cdiv(n, 256), 256, 0, st, n, pre, g);
}
void launch_zero_rows(cudaStream_t st, float* p, int64_t nfloats) {
  if (nfloats > 0) B2M_CK(cudaMemsetAsync(p, 0, nfloats * sizeof(float), st));
}

// ============================================================================================
// atom conv: shared pieces of the persistent forward and backward
// ============================================================================================
// Both kernels are persistent, one CTA per SM, and split the work per warpgroup over 64-edge tiles (below): every
// tile's A[src] rows arrive by per-row bulk copies into the warpgroup's one [TW][LDE] buffer, issued once the previous
// tile's scatter pass is done with it; the tile's indices load one tile earlier still, into registers (EdgeRow).
//
// Every per-element phase works in the accumulator layout (Map): a thread owns 2 rows x 16 columns of each branch b,
// whose first-layer columns are 64 b .. 64 b + 63.  Such a thread touches the tile only at its own positions
// (row(i), 64 b + col(j)), as float2 pairs
// (col(2 jj), col(2 jj) + 1); the pitch LDE = 136 (8 mod 32 floats) puts the 8 rows x 4 pairs of a half-warp on 32
// distinct banks.  The line-graph tiles use the same pitch and layout.
constexpr int LDE = 136;

struct EdgeRow {
  int src, dst, bond;
  float d;
};
// edge e's indices and distance, for a thread that owns a row of its tile (has_row) and e < E; else an empty row
__device__ __forceinline__ EdgeRow edge_row(const AtomConvArgs& a, int64_t e, bool has_row) {
  EdgeRow r{-1, -1, -1, 1.f};
  if (has_row && e < a.E) {
    r.src = a.e_src[e];
    r.dst = a.e_dst[e];
    r.bond = a.e_bond[e];
    r.d = a.e_vec[e].w;
  }
  return r;
}
// the threads with rows lr = 0..ROWS-1 of a ROWS-row tile t publish their row (indices, distance) and start its A[src]
// copy into `buf`; the caller has made sure, with a barrier, that nobody reads `buf` or the index arrays of this stage
// any more
template <int ROWS>
__device__ __forceinline__ void issue_gather(const AtomConvArgs& a, int64_t t, const EdgeRow& row, int lr, float* buf,
                                             uint64_t* bar, int* s_src, int* s_dst, int* s_bond, float* s_d) {
  if (lr == 0) mbar_expect_tx(bar, (uint32_t)min((int64_t)ROWS, a.E - t * ROWS) * 512u);
  if (lr < ROWS) {
    if (s_src != nullptr) s_src[lr] = row.src;
    s_dst[lr] = row.dst;
    s_bond[lr] = row.bond;
    s_d[lr] = row.d;
    if (row.src >= 0) bulk_g2s(buf + lr * LDE, a.Aproj + (size_t)row.src * D2, 512u, bar);
  }
}
// be_k(d_r) (and d be_k / dd) of a ROWS-row tile's rows by 2 ROWS threads (rows r, radial halves): k = 0..7 into be_s
// [ROWS][8] (the A operand of the radial products), k = 8 into be8 [ROWS]
template <int ROWS>
__device__ __forceinline__ void radial_rows(const AtomConvArgs& a, const float* s_d, int nvalid, float* be_s, float* be8,
                                            float* dbe_s, float* dbe8) {
  const int r = threadIdx.x % ROWS, half = (threadIdx.x / ROWS) & 1;
  const float d = s_d[r];
  const int k0 = half ? 5 : 0, k1 = half ? 9 : 5;
  for (int k = k0; k < k1; k++) {
    float be = 0.f, dbe = 0.f;
    if (r < nvalid) rbf_env_k(d, a.rp.freq[k], a.rp, be, dbe);
    *(k < 8 ? be_s + r * 8 + k : be8 + r) = be;
    if (dbe_s != nullptr) *(k < 8 ? dbe_s + r * 8 + k : dbe8 + r) = dbe;
  }
}
__device__ __forceinline__ float2 ld_f2(const float* p) { return *reinterpret_cast<const float2*>(p); }
__device__ __forceinline__ void st_f2(float* p, float x, float y) { *reinterpret_cast<float2*>(p) = make_float2(x, y); }

// index into a wg_mma64 result of this thread's element (row(2h + ii), col(j)) of the 64-row half h (Map layout)
__device__ __forceinline__ constexpr int fq(int ii, int j) { return 4 * (j >> 1) + 2 * ii + (j & 1); }

// d = x[rows of half h][0..7] . B^T on the tensor cores: x is be_s or dbe_s ([TM][8]; a thread's k pair of a row is one
// float2, conflict-free at pitch 8 within a half-warp), img a [64 n][8 k] image of the radial block (AtomConvArgs).
// The ninth column is the caller's: d + x_8 B[.][8].
__device__ __forceinline__ void radial_mma(const Map& m, int h, const float* x_s, const float* img, float (&d)[32]) {
  const float2 u = ld_f2(x_s + m.row(2 * h) * 8 + m.cb), v = ld_f2(x_s + m.row(2 * h + 1) * 8 + m.cb);
  const float x[1][4] = {{u.x, v.x, u.y, v.y}};
  uint32_t b = s_u32(img);
  asm volatile("" : "+r"(b));  // formed here: descriptors hoisted out of the tile loop would hold registers throughout
  wg_mma64(x, b, b + 512u * 4u, 0, false, d);
}

// pre of this thread's rows of 64-row half h (acc[2h], acc[2h + 1], Map layout): A[src] (in the tile) + C[dst] +
// (Q[bond] | be.M^T), summed in that order; rows r >= nvalid are 0.  be.M^T is k = 0..7 on the tensor cores plus
// be_8 M[.][8].  Index work is per row; the C / Q values of both rows (32 float2 loads) are in flight under the product.
template <int R>
__device__ __forceinline__ void first_layer_half(const AtomConvArgs& a, const Map& m, int h, const float* tile,
                                                 const int* s_dst, const int* s_bond, const float* be_s,
                                                 const float* be8, const float* rad, int nvalid,
                                                 float (&acc)[R][AC]) {
  const int c0 = 64 * m.branch + m.cb;
  float2 cv[2][AC / 2], qv[2][AC / 2];
  float b8[2];
  bool viaQ[2], ok[2];
#pragma unroll
  for (int ii = 0; ii < 2; ii++) {
    const int r = m.row(2 * h + ii);
    const int dst = s_dst[r], bond = s_bond[r];
    ok[ii] = r < nvalid;
    viaQ[ii] = a.Qproj != nullptr && bond >= 0;
    const float* cp = a.Cproj + (size_t)max(dst, 0) * D2 + c0;
#pragma unroll
    for (int jj = 0; jj < AC / 2; jj++) cv[ii][jj] = dst >= 0 ? __ldg(reinterpret_cast<const float2*>(cp + 8 * jj)) : make_float2(0.f, 0.f);
    if (viaQ[ii]) {
      const float* qp = a.Qproj + (size_t)bond * D2 + c0;
#pragma unroll
      for (int jj = 0; jj < AC / 2; jj++) qv[ii][jj] = __ldg(reinterpret_cast<const float2*>(qp + 8 * jj));
    } else {
#pragma unroll
      for (int jj = 0; jj < AC / 2; jj++) qv[ii][jj] = make_float2(0.f, 0.f);
    }
    b8[ii] = be8[r];
  }
  float d[32];
  radial_mma(m, h, be_s, rad + ATOM_RAD_M + 1024 * m.branch, d);
#pragma unroll
  for (int j = 0; j < AC; j++) {
    const float m8 = rad[ATOM_RAD_M8 + 64 * m.branch + m.col(j)];
#pragma unroll
    for (int ii = 0; ii < 2; ii++) {
      const int r = m.row(2 * h + ii);
      const float x = tile[r * LDE + 64 * m.branch + m.col(j)];
      const float2 c2 = cv[ii][j >> 1], q2 = qv[ii][j >> 1];
      const float t = viaQ[ii] ? ((j & 1) ? q2.y : q2.x) : fmaf(b8[ii], m8, d[fq(ii, j)]);
      acc[2 * h + ii][j] = ok[ii] ? x + ((j & 1) ? c2.y : c2.x) + t : 0.f;
    }
  }
}

// x rows of half h (2h, 2h + 1) in the accumulator layout as the register A fragment of wg_mma64: in k block ks a
// thread holds columns 8 ks + 2 (l%4) and + 1, the k pair its slots take in the k-permuted images
template <int R>
__device__ __forceinline__ void acc_frag(const float (&x)[R][AC], int h, float (&v)[8][4]) {
#pragma unroll
  for (int ks = 0; ks < 8; ks++) {
    v[ks][0] = x[2 * h][2 * ks], v[ks][1] = x[2 * h + 1][2 * ks];
    v[ks][2] = x[2 * h][2 * ks + 1], v[ks][3] = x[2 * h + 1][2 * ks + 1];
  }
}
// a wg_mma64 result d as rows 2h, 2h + 1 of acc (accumulator layout)
template <int R>
__device__ __forceinline__ void frag_acc(const float (&d)[32], int h, float (&acc)[R][AC]) {
#pragma unroll
  for (int q = 0; q < 32; q++) acc[2 * h + ((q >> 1) & 1)][2 * (q >> 2) + (q & 1)] = d[q];
}

// acc rows of half h (2h, 2h + 1) = x rows of half h . B^T (wg_mma64).  x is in the accumulator layout and is the
// register A fragment as it stands (acc_frag).  Bcan: the branch's k-permuted canonical image (hi plane of 4096
// floats, then lo).  x and acc may be the same array.
template <int R>
__device__ __forceinline__ void wg_mm64_acc(const float (&x)[R][AC], int h, const float* Bcan, float (&acc)[R][AC]) {
  float v[8][4];
  acc_frag(x, h, v);
  const uint32_t b_hi = s_u32(Bcan);
  float d[32];
  wg_mma64(v, b_hi, b_hi + 4096u * 4u, 0, false, d);
  frag_acc(d, h, acc);
}

// v[i] (row m.row(i)) summed over the 4 lanes of a quad, which share rows: lane l gets the sum of row l & 3
__device__ __forceinline__ float quad_row_sum(const float (&v)[AR]) {
  const int l = threadIdx.x & 3;
  const bool b0 = l & 1, b1 = l & 2;
  float w[2];
#pragma unroll
  for (int h = 0; h < 2; h++)
    w[h] = (b0 ? v[2 * h + 1] : v[2 * h]) + __shfl_xor_sync(0xffffffffu, b0 ? v[2 * h] : v[2 * h + 1], 1);
  return (b1 ? w[1] : w[0]) + __shfl_xor_sync(0xffffffffu, b1 ? w[0] : w[1], 2);
}

__device__ __forceinline__ void red_add_v4(float* p, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

// one row of a running segmented sum: `sum` collects the rows of key `cur` and is reduced into out[cur] when the key
// changes; rows with k < 0 contribute nothing.  The lane owns columns col .. col + 3 of out's rows of `width` floats.
__device__ __forceinline__ void seg_add(float* out, int width, int col, int k, const float4& v, int& cur, float4& sum) {
  if (k != cur) {
    if (cur >= 0) red_add_v4(out + (size_t)cur * width + col, sum);
    cur = k;
    sum = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (k >= 0) sum.x += v.x, sum.y += v.y, sum.z += v.z, sum.w += v.w;
}

// Scatter phase of a [ROWS][LDE] tile by NTH threads (threadIdx.x % NTH), columns 0 .. 4 LPR - 1, in one pass: LPR
// lanes take a row (lane q its columns 4 q .. 4 q + 3, one LDS.128; a row is contiguous, so the loads are conflict-free
// at any pitch) and a thread walks R = ROWS LPR / NTH consecutive rows.  Its float4 of row r
//   - is added to gat[gidx[r]]                                                    (gat != nullptr, gidx[r] >= 0),
//   - goes into one running sum per key array, reduced into out0[key0[.]] / out1[key1[.]] when the key changes and
//     after the thread's last row                                                 (out != nullptr, key >= 0),
//   - is stored to sto[sidx[r]]: for rows whose index occurs once in the whole pass (sto != nullptr, sidx[r] >= 0).
// Outputs are rows of 4 LPR floats, and every addition to them is one red.v4.  Rows past the end of a partial tile have
// all indices < 0.  The indices are equal in the lanes that share a row, so with LPR = 32 no branch diverges.  A run of
// equal keys that crosses the R-row boundary between two threads is reduced in two parts.  Values and indices are
// loaded eight rows at a time before those rows are walked: the reductions (asm volatile) keep loads in program order.
template <int LPR, int ROWS = TM, int NTH = NT>
__device__ __forceinline__ void scatter_rows(const float* tile, const int* key0, float* out0, const int* key1,
                                             float* out1, const int* gidx, float* gat, const int* sidx = nullptr,
                                             float* sto = nullptr) {
  constexpr int R = ROWS * LPR / NTH, W = 4 * LPR, B = 8;
  static_assert(R % B == 0 && B % 4 == 0, "batches of B rows, their indices read as int4");
  const int t = threadIdx.x % NTH, q = t % LPR, r0 = t / LPR * R;
  float4 s0 = make_float4(0.f, 0.f, 0.f, 0.f), s1 = s0;
  int c0 = -1, c1 = -1;
#pragma unroll
  for (int b = 0; b < R; b += B) {
    float4 v[B];
    int k0[B], k1[B], kg[B], ks[B];
#pragma unroll
    for (int i = 0; i < B; i++) v[i] = *reinterpret_cast<const float4*>(tile + (r0 + b + i) * LDE + 4 * q);
    auto ld_idx = [&](const int* idx, bool on, int(&k)[B]) {
#pragma unroll
      for (int i = 0; i < B; i += 4) {
        const int4 x = on ? *reinterpret_cast<const int4*>(idx + r0 + b + i) : make_int4(-1, -1, -1, -1);
        k[i] = x.x, k[i + 1] = x.y, k[i + 2] = x.z, k[i + 3] = x.w;
      }
    };
    ld_idx(key0, out0 != nullptr, k0);
    ld_idx(key1, out1 != nullptr, k1);
    ld_idx(gidx, gat != nullptr, kg);
    ld_idx(sidx, sto != nullptr, ks);
#pragma unroll
    for (int i = 0; i < B; i++) {
      if (ks[i] >= 0) *reinterpret_cast<float4*>(sto + (size_t)ks[i] * W + 4 * q) = v[i];
      if (kg[i] >= 0) red_add_v4(gat + (size_t)kg[i] * W + 4 * q, v[i]);
      seg_add(out0, W, 4 * q, k0[i], v[i], c0, s0);
      seg_add(out1, W, 4 * q, k1[i], v[i], c1, s1);
    }
  }
  if (c0 >= 0) red_add_v4(out0 + (size_t)c0 * W + 4 * q, s0);
  if (c1 >= 0) red_add_v4(out1 + (size_t)c1 * W + 4 * q, s1);
}

// ============================================================================================
// atom conv: forward
// ============================================================================================
// The three warpgroups of a CTA do not wait for each other: warpgroup w of CTA c owns the 64-edge tiles g, g + 3 grid,
// g + 6 grid, ... (g = 3 c + w) and computes both branches of each, so that some warpgroups' gathers, loads and
// activations run while another's products are on the tensor cores.  Each warpgroup has its own [TW][LDE] gather buffer
// (the k-th fill completes phase k of its mbarrier), its own index, distance and be slots, and its own named barrier;
// the W2 images, the radial block and b2 are staged once per CTA behind the only CTA-wide barrier and are read-only
// afterwards.  The next tile's gather is issued once the scatter pass is done with the buffer: one buffer per
// warpgroup is what lets three warpgroups fit next to the W2 image, and the other warpgroups' work covers the wait.  A
// thread holds rows m.row(0), m.row(1) of the tile and columns m.col(j) of both branches: the layers' 32 outputs L stay
// in registers while the gates' first layer and product run, and m = L . (G . w_ab) is formed in registers and stored
// at the thread's own positions (columns 0..63) for the scatter pass.  Three warpgroups of 128 threads leave each
// thread at most 168 registers.
constexpr int TW = 64;               // rows of a warpgroup's forward tile
constexpr int WGF = 3, NTF = 128 * WGF;  // warpgroups and threads of a forward CTA
struct AtomSmemFwd {
  static constexpr int kTile = 32;                   // [WGF][TW][LDE] gather buffers (first 128 B: their mbarriers)
  static constexpr int kW = kTile + WGF * TW * LDE;  // wgmma images of W2 (2 branches x hi | lo, k permuted), staged once
  static constexpr int kRad = kW + 16384;            // radial block (M, W_ab: AtomConvArgs::radial), staged once
  static constexpr int kBe = kRad + ATOM_RAD;        // be [WGF][TW][8] (k < 8)
  static constexpr int kBe8 = kBe + WGF * TW * 8;    // be [WGF][TW] (k = 8)
  static constexpr int kB2 = kBe8 + WGF * TW;
  static constexpr int kD = kB2 + 128;               // d [WGF][TW]
  static constexpr int kIdx = kD + WGF * TW;         // dst [WGF][TW], then bond [WGF][TW]
  static constexpr int kTotal = kIdx + 2 * WGF * TW;
  static constexpr size_t bytes = (size_t)kTotal * 4;
};
static_assert(AtomSmemFwd::bytes <= 232448, "atom-conv forward shared memory");
static_assert(AtomSmemFwd::kW % 4 == 0 && AtomSmemFwd::kRad % 4 == 0 && AtomSmemFwd::kBe % 4 == 0 &&
                  AtomSmemFwd::kIdx % 4 == 0,
              "16-byte aligned images, radial rows and index slots");

// barrier of warpgroup w's 128 threads alone (named barrier 1 + w; barrier 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(int w) { asm volatile("bar.sync %0, 128;" ::"r"(1 + w) : "memory"); }

__global__ void __launch_bounds__(NTF, 1) k_atomconv_fwd(const AtomConvArgs a) {
  extern __shared__ __align__(128) float smem[];
  const int tid = threadIdx.x, w = tid >> 7, lr = tid & 127;  // warpgroup; thread lr < TW gathers row lr
  uint64_t* mbar = reinterpret_cast<uint64_t*>(smem) + w;      // this warpgroup's gather buffer
  const float* Wsm = smem + AtomSmemFwd::kW;
  const float* rad = smem + AtomSmemFwd::kRad;
  const float* b2s = smem + AtomSmemFwd::kB2;
  float* tile = smem + AtomSmemFwd::kTile + w * TW * LDE;
  float* be_s = smem + AtomSmemFwd::kBe + w * TW * 8;
  float* be8 = smem + AtomSmemFwd::kBe8 + w * TW;
  float* s_d = smem + AtomSmemFwd::kD + w * TW;
  int* s_dst = reinterpret_cast<int*>(smem + AtomSmemFwd::kIdx) + w * TW;
  int* s_bond = reinterpret_cast<int*>(smem + AtomSmemFwd::kIdx) + (WGF + w) * TW;

  const int64_t ntiles = (a.E + TW - 1) / TW, first = WGF * (int64_t)blockIdx.x + w, step = WGF * (int64_t)gridDim.x;
  if (tid == 0) {
    for (int i = 0; i < WGF; i++) mbar_init(reinterpret_cast<uint64_t*>(smem) + i, 1);
    fence_barrier_init();
  }
  EdgeRow nxt = edge_row(a, first * TW + lr, lr < TW);
  // loop-invariant operands, once per CTA
  stage_w<NTF>(smem + AtomSmemFwd::kW, a.W2can, 4096);
  stage_w<NTF>(smem + AtomSmemFwd::kRad, a.radial, ATOM_RAD / 4);
  if (tid < 128) smem[AtomSmemFwd::kB2 + tid] = a.b2[tid];
  __syncthreads();
  if (first < ntiles)  // the last CTA's later warpgroups have no tile when the tile count is not a multiple of WGF
    issue_gather<TW>(a, first, nxt, lr, tile, mbar, nullptr, s_dst, s_bond, s_d);
  nxt = edge_row(a, (first + step) * TW + lr, lr < TW);

  const Map m;
  Map mL = m, mG = m;  // the first layer's columns and radial image of each branch
  mL.branch = 0;
  mG.branch = 1;
  int it = 0;
  for (int64_t t = first; t < ntiles; t += step, it++) {
    const int nvalid = (int)min((int64_t)TW, a.E - t * TW);
    wg_sync(w);  // the tile's indices and distances are published
    radial_rows<TW>(a, s_d, nvalid, be_s, be8, nullptr, nullptr);
    mbar_wait(mbar, (uint32_t)it & 1u);
    wg_sync(w);
    // per branch: pre = A[src] + C[dst] + (be.M^T | Q[bond]); silu(pre) straight into the second layer; + b2
    float L[2][AC];
    first_layer_half(a, mL, 0, tile, s_dst, s_bond, be_s, be8, rad, nvalid, L);
#pragma unroll
    for (int ii = 0; ii < 2; ii++)
#pragma unroll
      for (int j = 0; j < AC; j++) L[ii][j] = silu_f(L[ii][j]);
    wg_mm64_acc(L, 0, Wsm, L);
#pragma unroll
    for (int ii = 0; ii < 2; ii++)
#pragma unroll
      for (int j = 0; j < AC; j++) L[ii][j] = silu_f(L[ii][j] + b2s[m.col(j)]);
    float G[2][AC];
    first_layer_half(a, mG, 0, tile, s_dst, s_bond, be_s, be8, rad, nvalid, G);
#pragma unroll
    for (int ii = 0; ii < 2; ii++)
#pragma unroll
      for (int j = 0; j < AC; j++) G[ii][j] = silu_f(G[ii][j]);
    wg_mm64_acc(G, 0, Wsm + 8192, G);
    // m = L . (G . w_ab), w_ab = be.W_ab^T on the tensor cores, over the A[src] values of columns 0..63
    float wab[32];
    radial_mma(m, 0, be_s, rad + ATOM_RAD_WAB, wab);
#pragma unroll
    for (int ii = 0; ii < 2; ii++) {
      const int r = m.row(ii);
      const float b8 = be8[r];
      float mv[AC];
#pragma unroll
      for (int j = 0; j < AC; j++) {
        const float g = sigm(G[ii][j] + b2s[64 + m.col(j)]) * fmaf(b8, rad[ATOM_RAD_WAB8 + m.col(j)], wab[fq(ii, j)]);
        mv[j] = L[ii][j] * g;
      }
#pragma unroll
      for (int jj = 0; jj < AC / 2; jj++) st_f2(tile + r * LDE + m.col(2 * jj), mv[2 * jj], mv[2 * jj + 1]);
    }
    wg_sync(w);
    scatter_rows<16, TW, 128>(tile, s_dst, a.agg, nullptr, nullptr, nullptr, nullptr);  // agg[dst] += m
    fence_proxy_async_smem();  // this thread's generic accesses of the buffer come before its bulk refill
    wg_sync(w);                // the warpgroup is done with the buffer, the indices and be_s
    if (t + step < ntiles) {
      issue_gather<TW>(a, t + step, nxt, lr, tile, mbar, nullptr, s_dst, s_bond, s_d);
      nxt = edge_row(a, (t + 2 * step) * TW + lr, lr < TW);
    }
  }
}

void launch_atomconv_fwd(cudaStream_t st, const AtomConvArgs& a, int num_sms) {
  if (a.E <= 0) return;
  static PerDeviceOnce attr;
  if (auto once_ = attr.first(); once_) {
    B2M_CK(cudaFuncSetAttribute(k_atomconv_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AtomSmemFwd::bytes));
  }
  launch(k_atomconv_fwd, std::min(cdiv(cdiv(a.E, TW), WGF), num_sms), NTF, AtomSmemFwd::bytes, st, a);
}

// ============================================================================================
// atom conv: backward (recompute forward in-tile, then hand-derived reverse pass)
// ============================================================================================
// Laid out like the forward: the two warpgroups of a CTA do not wait for each other.  Warpgroup w of CTA c owns the
// 64-edge tiles g, g + 2 grid, g + 4 grid, ... (g = 2 c + w) and computes both branches of each.  Each warpgroup has
// its own [TW][LDE] buffer P, mbarrier, index, distance, be and d be / dd slots and named barrier.  Both weight images
// (W2 for the recompute, W2^T for g . W2), the radial block and b2 are staged once per CTA behind the only CTA-wide
// barrier; one buffer per warpgroup is what lets two warpgroups fit next to 128 KB of images.  The tile's A[src] rows
// arrive in P; each thread overwrites its own A[src] values with the pre-activations, and later with their adjoints
// gpre, which the scatter pass reads row-major.  A thread holds rows m.row(0), m.row(1) and columns m.col(j) of both
// branches, so the second layer's outputs -- u (L) and oG = sigm(v + b2) (G), 32 floats each -- stay in registers
// through the elementwise reverse, which forms dE/du, dE/dv and dE/dw_ab in place over u, oG and w_ab.  The next
// tile's gather is issued once the scatter pass is done with P, and the other warpgroup's work covers the wait.
constexpr int WGB = 2, NTB = 128 * WGB;  // warpgroups and threads of a backward CTA
struct AtomSmemBwd {
  static constexpr int kTile = 32;                      // [WGB][TW][LDE] buffers P (first 128 B: their mbarriers)
  static constexpr int kW = kTile + WGB * TW * LDE;     // wgmma images of W2 (2 branches x hi | lo, k permuted) ...
  static constexpr int kWT = kW + 16384;                // ... and of W2^T, both staged once
  static constexpr int kRad = kWT + 16384;              // radial block (M, W_ab: AtomConvArgs::radial), staged once
  static constexpr int kBe = kRad + ATOM_RAD;           // be [WGB][TW][8] (k < 8)
  static constexpr int kDbe = kBe + WGB * TW * 8;       // d be / dd [WGB][TW][8]
  static constexpr int kBe8 = kDbe + WGB * TW * 8;      // be [WGB][TW] (k = 8)
  static constexpr int kDbe8 = kBe8 + WGB * TW;         // d be / dd [WGB][TW] (k = 8)
  static constexpr int kB2 = kDbe8 + WGB * TW;
  static constexpr int kD = kB2 + 128;                  // d [WGB][TW]
  static constexpr int kIdx = kD + WGB * TW;            // src, dst, bond: [WGB][TW] each
  static constexpr int kTotal = kIdx + 3 * WGB * TW;
  static constexpr size_t bytes = (size_t)kTotal * 4;
};
static_assert(AtomSmemBwd::bytes <= 232448, "atom-conv backward shared memory");
static_assert(AtomSmemBwd::kW % 4 == 0 && AtomSmemBwd::kWT % 4 == 0 && AtomSmemBwd::kRad % 4 == 0 &&
                  AtomSmemBwd::kBe % 4 == 0 && AtomSmemBwd::kDbe % 4 == 0 && AtomSmemBwd::kIdx % 4 == 0,
              "16-byte aligned images, radial rows and index slots");

__global__ void __launch_bounds__(NTB, 1) k_atomconv_bwd(const AtomConvArgs a) {
  extern __shared__ __align__(128) float smem[];
  const int tid = threadIdx.x, w = tid >> 7, lr = tid & 127;  // warpgroup; thread lr < TW gathers row lr
  uint64_t* mbar = reinterpret_cast<uint64_t*>(smem) + w;      // this warpgroup's buffer
  const float* W2s = smem + AtomSmemBwd::kW;
  const float* W2Ts = smem + AtomSmemBwd::kWT;
  const float* rad_base = smem + AtomSmemBwd::kRad;
  const float* b2s = smem + AtomSmemBwd::kB2;
  float* P = smem + AtomSmemBwd::kTile + w * TW * LDE;
  float* be_s = smem + AtomSmemBwd::kBe + w * TW * 8;
  float* dbe_s = smem + AtomSmemBwd::kDbe + w * TW * 8;
  float* be8 = smem + AtomSmemBwd::kBe8 + w * TW;
  float* dbe8 = smem + AtomSmemBwd::kDbe8 + w * TW;
  float* s_d = smem + AtomSmemBwd::kD + w * TW;
  int* s_src = reinterpret_cast<int*>(smem + AtomSmemBwd::kIdx) + w * TW;
  int* s_dst = reinterpret_cast<int*>(smem + AtomSmemBwd::kIdx) + (WGB + w) * TW;
  int* s_bond = reinterpret_cast<int*>(smem + AtomSmemBwd::kIdx) + (2 * WGB + w) * TW;

  const int64_t ntiles = (a.E + TW - 1) / TW, first = WGB * (int64_t)blockIdx.x + w, step = WGB * (int64_t)gridDim.x;
  const bool useQ = a.Qproj != nullptr;
  if (tid == 0) {
    for (int i = 0; i < WGB; i++) mbar_init(reinterpret_cast<uint64_t*>(smem) + i, 1);
    fence_barrier_init();
  }
  EdgeRow nxt = edge_row(a, first * TW + lr, lr < TW);
  // loop-invariant operands, once per CTA
  stage_w<NTB>(smem + AtomSmemBwd::kW, a.W2can, 4096);
  stage_w<NTB>(smem + AtomSmemBwd::kWT, a.W2Tcan, 4096);
  stage_w<NTB>(smem + AtomSmemBwd::kRad, a.radial, ATOM_RAD / 4);
  if (tid < 128) smem[AtomSmemBwd::kB2 + tid] = a.b2[tid];
  __syncthreads();
  if (first < ntiles)  // the last CTA's second warpgroup has no tile when the tile count is odd
    issue_gather<TW>(a, first, nxt, lr, P, mbar, s_src, s_dst, s_bond, s_d);
  nxt = edge_row(a, (first + step) * TW + lr, lr < TW);

  const Map m;
  Map mL = m, mG = m;  // the first layer's columns and radial image of each branch
  mL.branch = 0;
  mG.branch = 1;
  int it = 0;
  for (int64_t t = first; t < ntiles; t += step, it++) {
    const float* rad = rad_base;
    asm volatile("" : "+l"(rad));  // radial addresses formed per tile: hoisted out of the loop they hold registers
    const int64_t e0 = t * TW;
    const int nvalid = (int)min((int64_t)TW, a.E - e0);
    wg_sync(w);  // the tile's indices and distances are published
    radial_rows<TW>(a, s_d, nvalid, be_s, be8, dbe_s, dbe8);
    mbar_wait(mbar, (uint32_t)it & 1u);
    wg_sync(w);
    // recompute, per branch: pre (kept in P at the thread's own positions), silu(pre) . W2^T + b2 = u (L) / v (G);
    // L keeps u, G keeps oG = sigm(v)
    float L[2][AC], G[2][AC];
    auto recompute = [&](const Map& mb, float(&x)[2][AC]) {
      first_layer_half(a, mb, 0, P, s_dst, s_bond, be_s, be8, rad, nvalid, x);
#pragma unroll
      for (int ii = 0; ii < 2; ii++)
#pragma unroll
        for (int jj = 0; jj < AC / 2; jj++) {
          float& x0 = x[ii][2 * jj];
          float& x1 = x[ii][2 * jj + 1];
          st_f2(P + m.row(ii) * LDE + 64 * mb.branch + m.col(2 * jj), x0, x1);
          x0 = silu_f(x0);
          x1 = silu_f(x1);
        }
      wg_mm64_acc(x, 0, W2s + mb.branch * 8192, x);
    };
    recompute(mL, L);
#pragma unroll
    for (int ii = 0; ii < 2; ii++)
#pragma unroll
      for (int j = 0; j < AC; j++) L[ii][j] += b2s[m.col(j)];
    recompute(mG, G);
#pragma unroll
    for (int ii = 0; ii < 2; ii++)
#pragma unroll
      for (int j = 0; j < AC; j++) G[ii][j] = sigm(G[ii][j] + b2s[64 + m.col(j)]);
    // elementwise reverse, in place: L <- dE/du, G <- dE/dv, w <- w_ab = be.W_ab^T (tensor cores) <- dE/dw_ab.  Both
    // rows' 16 dE/dagg values are loaded before any is used.
    int dst[2];
    float2 gm2[2][AC / 2];
#pragma unroll
    for (int ii = 0; ii < 2; ii++) {
      dst[ii] = s_dst[m.row(ii)];
      const float* gp = a.gagg + (size_t)max(dst[ii], 0) * D + m.cb;
#pragma unroll
      for (int jj = 0; jj < AC / 2; jj++)
        gm2[ii][jj] = dst[ii] >= 0 ? __ldg(reinterpret_cast<const float2*>(gp + 8 * jj)) : make_float2(0.f, 0.f);
    }
    float wv[32];
    radial_mma(m, 0, be_s, rad + ATOM_RAD_WAB, wv);
#pragma unroll
    for (int ii = 0; ii < 2; ii++) {
      const float b8 = be8[m.row(ii)];
#pragma unroll
      for (int jj = 0; jj < AC / 2; jj++) {
        const float2 wk2 = ld_f2(rad + ATOM_RAD_WAB8 + m.col(2 * jj));
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const int j = 2 * jj + e;
          const float u = L[ii][j], oG = G[ii][j];
          const float gm = e ? gm2[ii][jj].y : gm2[ii][jj].x;
          const float wab = fmaf(b8, e ? wk2.y : wk2.x, wv[fq(ii, j)]);
          float gu = 0.f, gv = 0.f, gwv = 0.f;
          if (dst[ii] >= 0) {
            const float sg = sigm(u);
            const float oL = u * sg;
            gwv = gm * oL * oG;                                 // d/d w_ab
            gu = gm * oG * wab * (sg * (1.f + u * (1.f - sg)));  // d/du
            gv = gm * oL * wab * oG * (1.f - oG);                // d/dv
          }
          L[ii][j] = gu;
          G[ii][j] = gv;
          wv[fq(ii, j)] = gwv;
        }
      }
    }
    // dE/dd of row m.row(ii), one sum per branch over this thread's columns: branch 0 sum_c dE/dw_ab[r][c]
    // (dbe.W_ab^T)[r][c]; rows fed by M (not bond rows fed by Q) add sum_j gpre[r][j] (dbe.M^T)[r][j] of each branch
    float sd[AR];  // [2 b + ii]
    {
      float dw[32];
      radial_mma(m, 0, dbe_s, rad + ATOM_RAD_WAB, dw);
#pragma unroll
      for (int ii = 0; ii < 2; ii++) {
        const float db8 = dbe8[m.row(ii)];
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < AC; j++) s = fmaf(wv[fq(ii, j)], fmaf(db8, rad[ATOM_RAD_WAB8 + m.col(j)], dw[fq(ii, j)]), s);
        sd[ii] = s;
        sd[2 + ii] = 0.f;
      }
    }
    // per branch: gpre = (g . W2) * dsilu(pre), into P at the thread's own positions
    auto reverse = [&](const Map& mb, float(&x)[2][AC]) {
      const int c0 = 64 * mb.branch;
      wg_mm64_acc(x, 0, W2Ts + mb.branch * 8192, x);
#pragma unroll
      for (int ii = 0; ii < 2; ii++)
#pragma unroll
        for (int jj = 0; jj < AC / 2; jj++) {
          float* p = P + m.row(ii) * LDE + c0 + m.col(2 * jj);
          const float2 pre = ld_f2(p);
          float& x0 = x[ii][2 * jj];
          float& x1 = x[ii][2 * jj + 1];
          x0 *= dsilu_f(pre.x);
          x1 *= dsilu_f(pre.y);
          st_f2(p, x0, x1);
        }
      float dm[32];
      radial_mma(m, 0, dbe_s, rad + ATOM_RAD_M + 1024 * mb.branch, dm);
#pragma unroll
      for (int ii = 0; ii < 2; ii++) {
        const int r = m.row(ii);
        const float db8 = dbe8[r];
        float s = 0.f;
#pragma unroll
        for (int jj = 0; jj < AC / 2; jj++) {
          const float2 mk = ld_f2(rad + ATOM_RAD_M8 + c0 + m.col(2 * jj));
          s = fmaf(x[ii][2 * jj], fmaf(db8, mk.x, dm[fq(ii, 2 * jj)]), s);
          s = fmaf(x[ii][2 * jj + 1], fmaf(db8, mk.y, dm[fq(ii, 2 * jj + 1)]), s);
        }
        if (r < nvalid && !(useQ && s_bond[r] >= 0)) sd[2 * mb.branch + ii] += s;
      }
    };
    reverse(mL, L);
    reverse(mG, G);
    {  // quad_row_sum: lane l gets branch l >> 1's sum of row m.row(l & 1); then branch 0's + branch 1's
      const float v = quad_row_sum(sd);
      const float v1 = __shfl_xor_sync(0xffffffffu, v, 2);
      const int r = m.row(tid & 1);
      if ((tid & 2) == 0 && r < nvalid) a.gd[e0 + r] += v + v1;
    }
    wg_sync(w);  // P holds the tile's gpre
    // gC[dst] += gpre (segmented), gA[src] += gpre, gQ[bond] = gpre (each bond row occurs once): one pass over P
    scatter_rows<32, TW, 128>(P, s_dst, a.gA != nullptr ? a.gC : nullptr, nullptr, nullptr, s_src, a.gA, s_bond,
                              useQ ? a.gQ : nullptr);
    fence_proxy_async_smem();  // this thread's generic accesses of the buffer come before its bulk refill
    wg_sync(w);                // the warpgroup is done with the buffer, the indices and the radial slots
    if (t + step < ntiles) {
      issue_gather<TW>(a, t + step, nxt, lr, P, mbar, s_src, s_dst, s_bond, s_d);
      nxt = edge_row(a, (t + 2 * step) * TW + lr, lr < TW);
    }
  }
}

void launch_atomconv_bwd(cudaStream_t st, const AtomConvArgs& a, int num_sms) {
  if (a.E <= 0) return;
  static PerDeviceOnce attr;
  if (auto once_ = attr.first(); once_) {
    B2M_CK(cudaFuncSetAttribute(k_atomconv_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AtomSmemBwd::bytes));
  }
  launch(k_atomconv_bwd, std::min(cdiv(cdiv(a.E, TW), WGB), num_sms), NTB, AtomSmemBwd::bytes, st, a);
}

// ============================================================================================
// line-graph kernels: bond conv (HIDDEN) and angle update (!HIDDEN)
// ============================================================================================
// The forward and the angle-update backward run in independent warpgroups over 64-angle tiles (LineSmemWg, below).
// The bond-conv backward's four weight images do not fit in a CTA next to one buffer per warpgroup, so it keeps the
// layout described here (LineSmem, LineSm, line_prologue).  Persistent like the atom conv: min(tiles, SMs) CTAs, CTA c
// takes 128-angle tiles c, c + grid, ...  Two [TM][LDE] buffers alternate: tile number `it` of a CTA has its Ha[a]
// rows in buffer it & 1 (P) and its own angle rows in columns 64..127 of the other buffer (Q).  Each copy completes on the barrier of its tile's stage (hbar / abar [it & 1], parity
// stage_parity(it)).  One 64 KB weight slot holds the image the next product needs; images that share it are refilled
// by bulk copies as soon as the product before has read the slot, and waited on (wbar, one phase per fill, in fill
// order) just before the product that reads them.
//
// Every per-element phase works in the accumulator layout (Map), as in the atom conv: a thread touches the tiles only at
// its own positions (row(i), 64 b + col(j)), as float2 pairs, and the A operands of the products are either its
// accumulator fragments (hid . W2^T, g . W2) or float2 pairs of a tile (ang . Wg^T, gpre . Wg; wg_mm64).  All B images
// are k-permuted (engine.cu: permute_k8).
struct LineSmem {
  static constexpr int kBuf = 32;               // two [TM][LDE] buffers (first 128 B: hbar[2], abar[2], wbar)
  static constexpr int kW = kBuf + 2 * TM * LDE;  // one weight image (2 branches x hi | lo, or Wg^T hi | lo)
  static constexpr int kB2 = kW + 16384;
  static constexpr int kIdx = kB2 + 128;       // a_in, a_out, a_ctr: [2][TM] each
  static constexpr int kTotal = kIdx + 6 * TM;
  static constexpr size_t bytes = (size_t)kTotal * 4;
};
static_assert(LineSmem::bytes <= 232448, "line-graph shared memory");

struct LineSm {
  float* smem;
  __device__ __forceinline__ uint64_t* hbar() const { return reinterpret_cast<uint64_t*>(smem); }
  __device__ __forceinline__ uint64_t* abar() const { return hbar() + 2; }
  __device__ __forceinline__ uint64_t* wbar() const { return hbar() + 4; }
  __device__ __forceinline__ float* buf(int s) const { return smem + LineSmem::kBuf + s * TM * LDE; }
  __device__ __forceinline__ float* W() const { return smem + LineSmem::kW; }
  __device__ __forceinline__ float* b2() const { return smem + LineSmem::kB2; }
  __device__ __forceinline__ int* idx(int s, int k) const {  // k: 0 a_in, 1 a_out, 2 a_ctr
    return reinterpret_cast<int*>(smem + LineSmem::kIdx) + (2 * k + s) * TM;
  }
};

struct AngleIdx {
  int a, b, c;
};
// angle r's indices, for a thread that owns a row of its tile (has_row) and r < A; else an empty row
__device__ __forceinline__ AngleIdx angle_row(const LineArgs& a, int64_t r, bool has_row) {
  AngleIdx x{-1, -1, -1};
  if (has_row && r < a.A) {
    x.a = a.a_in[r];
    x.b = a.a_out[r];
    x.c = a.a_ctr[r];
  }
  return x;
}
__device__ __forceinline__ AngleIdx angle_idx(const LineArgs& a, int64_t r) { return angle_row(a, r, threadIdx.x < TM); }
// threads 0..TM-1 publish their row of tile t into stage s's index arrays and start its Ha[a] copy into `buf`; the
// caller has made sure, with a proxy fence and a barrier, that nobody reads `buf` or those arrays any more
__device__ __forceinline__ void line_issue_ha(const LineArgs& a, const LineSm& sm, int64_t t, const AngleIdx& x,
                                             float* buf, int s) {
  const int tid = threadIdx.x;
  if (tid == 0) mbar_expect_tx(&sm.hbar()[s], (uint32_t)min((int64_t)TM, a.A - t * TM) * 512u);
  if (tid < TM) {
    sm.idx(s, 0)[tid] = x.a;
    sm.idx(s, 1)[tid] = x.b;
    sm.idx(s, 2)[tid] = x.c;
    if (x.a >= 0) bulk_g2s(buf + tid * LDE, a.Ha + (size_t)x.a * D2, 512u, &sm.hbar()[s]);
  }
}
// the 256 B angle rows of tile t into columns 64..127 of `buf`, completing on abar[s]
__device__ __forceinline__ void line_issue_ang(const LineArgs& a, const LineSm& sm, int64_t t, float* buf, int s) {
  const int tid = threadIdx.x;
  const int nvalid = (int)min((int64_t)TM, a.A - t * TM);
  if (tid == 0) mbar_expect_tx(&sm.abar()[s], (uint32_t)nvalid * 256u);
  if (tid < nvalid) bulk_g2s(buf + tid * LDE + 64, a.ang + (size_t)(t * TM + tid) * D, 256u, &sm.abar()[s]);
}
// barriers, b2, the first weight image and the copies of the CTA's first tile (Ha into buffer 0, angles into buffer 1)
__device__ __forceinline__ AngleIdx line_prologue(const LineArgs& a, const LineSm& sm) {
  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int i = 0; i < 5; i++) mbar_init(&sm.hbar()[i], 1);
    fence_barrier_init();
  }
  AngleIdx x = angle_idx(a, (int64_t)blockIdx.x * TM + tid);
  if (tid < 128) sm.b2()[tid] = a.b2 ? a.b2[tid] : 0.f;
  __syncthreads();
  if (tid == 0) bulk_g2s_image(sm.W(), a.Wgcan, 16384 * 4, sm.wbar());
  line_issue_ha(a, sm, blockIdx.x, x, sm.buf(0), 0);
  line_issue_ang(a, sm, blockIdx.x, sm.buf(1), 0);
  return angle_idx(a, ((int64_t)blockIdx.x + gridDim.x) * TM + tid);
}

// pre = ((Ha[a] + ang.Wg^T) + Hb[b]) + Xc[c] in place of acc (which holds ang.Wg^T), in the accumulator layout: Ha from
// P at the thread's own positions, a row's 16 Hb and 16 Xc values as float2 loads issued before any is used.  Rows
// r >= nvalid get 0.  R = AR: the four rows of a 128-row tile; R = 2: the two of a 64-row tile.
template <int R>
__device__ __forceinline__ void line_first_layer(const LineArgs& a, const Map& m, const float* P, const int* s_b,
                                                 const int* s_c, int nvalid, float (&acc)[R][AC]) {
  const int c0 = 64 * m.branch + m.cb;
#pragma unroll
  for (int i = 0; i < R; i++) {
    const int r = m.row(i);
    const bool ok = r < nvalid;
    const float* hb = a.Hb + (size_t)(ok ? s_b[r] : 0) * D2 + c0;
    const float* xc = a.Xc + (size_t)(ok ? s_c[r] : 0) * D2 + c0;
    float2 hv[AC / 2], xv[AC / 2];
#pragma unroll
    for (int jj = 0; jj < AC / 2; jj++) {
      hv[jj] = ok ? __ldg(reinterpret_cast<const float2*>(hb + 8 * jj)) : make_float2(0.f, 0.f);
      xv[jj] = ok ? __ldg(reinterpret_cast<const float2*>(xc + 8 * jj)) : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int jj = 0; jj < AC / 2; jj++) {
      const float2 ha = ok ? ld_f2(P + r * LDE + c0 + 8 * jj) : make_float2(0.f, 0.f);
      float& x0 = acc[i][2 * jj];
      float& x1 = acc[i][2 * jj + 1];
      x0 = ok ? ha.x + x0 + hv[jj].x + xv[jj].x : 0.f;
      x1 = ok ? ha.y + x1 + hv[jj].y + xv[jj].y : 0.f;
    }
  }
}

__device__ __forceinline__ void red_add_v2(float* p, float x, float y) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(x), "f"(y) : "memory");
}

// ---- the forward and the angle-update backward: independent warpgroups ----
// Laid out like the atom conv: the warpgroups of a CTA do not wait for each other.  Warpgroup w of CTA c owns the
// 64-angle tiles g, g + WG grid, g + 2 WG grid, ... (g = WG c + w, grid = min(ceil(tiles / WG), SMs)) and computes both
// branches of each.  Each warpgroup has its own [TW][LDE] buffer for the tile's Ha[a] rows (per-row bulk copies; the
// k-th fill completes phase k of its mbarrier), its own a_in / a_out / a_ctr slots and its own named barrier; the
// weight images (and b2) are staged once per CTA behind the only CTA-wide barrier and are read-only afterwards.  The
// next tile's indices load one tile ahead into registers, and its Ha copy is issued as soon as the warpgroup is done
// with the buffer.  The angle rows need no stage: with the k-permuted images a thread's k pair of an angle row is one
// float2 of that row, so they go from global memory straight into the register A fragments of ang . Wg^T
// (line_ang_frag), and both branches' products share one tf32 split of them (wg_mma64_pair).
template <int WG, int NIMG>
struct LineSmemWg {
  static constexpr int kBuf = 32;                  // [WG][TW][LDE] buffers (first 128 B: their mbarriers)
  static constexpr int kW = kBuf + WG * TW * LDE;  // NIMG wgmma images of 16384 floats, staged once
  static constexpr int kB2 = kW + NIMG * 16384;
  static constexpr int kIdx = kB2 + 128;           // a_in, a_out, a_ctr: [WG][TW] each
  static constexpr int kTotal = kIdx + 3 * WG * TW;
  static constexpr size_t bytes = (size_t)kTotal * 4;
  static_assert(bytes <= 232448, "line-graph shared memory");
  static_assert(kW % 32 == 0 && kIdx % 4 == 0, "128-byte aligned images, 16-byte aligned index slots");
};
// forward: HIDDEN (bond conv) keeps Wg and W2 resident next to two buffers; !HIDDEN (angle update) has only Wg, and
// three buffers fit next to it (three warpgroups, at most 168 registers per thread)
template <bool HIDDEN>
struct LineFwd {
  static constexpr int WG = HIDDEN ? 2 : 3;
  using Smem = LineSmemWg<WG, HIDDEN ? 2 : 1>;
};
// angle-update backward: Wg (recompute) and Wg^T (gang += gpre . Wg) resident, two warpgroups
constexpr int LBWG = 2;
using LineBwdSmem = LineSmemWg<LBWG, 2>;

// the threads with rows lr = 0..TW-1 of 64-angle tile t publish their row's indices and start its Ha[a] copy into
// `buf`, completing on `bar`; the caller has made sure, with a proxy fence and a barrier, that nobody reads `buf` or
// the index slots any more
__device__ __forceinline__ void line_issue_ha_wg(const LineArgs& a, int64_t t, const AngleIdx& x, int lr, float* buf,
                                                 uint64_t* bar, int* s_a, int* s_b, int* s_c) {
  if (lr == 0) mbar_expect_tx(bar, (uint32_t)min((int64_t)TW, a.A - t * TW) * 512u);
  if (lr < TW) {
    s_a[lr] = x.a;
    s_b[lr] = x.b;
    s_c[lr] = x.c;
    if (x.a >= 0) bulk_g2s(buf + lr * LDE, a.Ha + (size_t)x.a * D2, 512u, bar);
  }
}
// this thread's A fragment of ang . Wg^T for the 64-angle tile at row r0 (wg_mma64): rows m.row(0), m.row(1), and of
// each the k pair 8 ks + cb, + 1 as one float2; rows r >= nvalid are 0
__device__ __forceinline__ void line_ang_frag(const LineArgs& a, const Map& m, int64_t r0, int nvalid, float (&x)[8][4]) {
  float2 u[2][8];
#pragma unroll
  for (int ii = 0; ii < 2; ii++) {
    const int r = m.row(ii);
    const bool ok = r < nvalid;
    const float* p = a.ang + (size_t)(r0 + (ok ? r : 0)) * D + m.cb;
#pragma unroll
    for (int ks = 0; ks < 8; ks++) u[ii][ks] = ok ? __ldg(reinterpret_cast<const float2*>(p + 8 * ks)) : make_float2(0.f, 0.f);
  }
#pragma unroll
  for (int ks = 0; ks < 8; ks++) x[ks][0] = u[0][ks].x, x[ks][1] = u[1][ks].x, x[ks][2] = u[0][ks].y, x[ks][3] = u[1][ks].y;
}
// L / G (rows 0, 1 of a 64-row tile, accumulator layout) = x . B^T for the two branch images of Bcan (hi plane of
// 4096 floats, then lo, per branch): wg_mma64 twice, with one tf32 split of x and one commit
__device__ __forceinline__ void wg_mma64_pair(const float (&x)[8][4], const float* Bcan, float (&L)[2][AC],
                                              float (&G)[2][AC]) {
  constexpr uint32_t LBO = 8 * 128;
  uint32_t ah[8][4], al[8][4];
#pragma unroll
  for (int ks = 0; ks < 8; ks++)
#pragma unroll
    for (int q = 0; q < 4; q++) {
      ah[ks][q] = tf32_hi_bits(x[ks][q]);
      al[ks][q] = __float_as_uint(x[ks][q] - __uint_as_float(ah[ks][q]));
    }
  float dL[32], dG[32];
  auto mma = [&](float(&d)[32], uint32_t b_hi) {
#pragma unroll
    for (int ks = 0; ks < 8; ks++)
#pragma unroll
      for (int term = 0; term < 3; term++) {
        const uint64_t bd = gmma_desc((term == 2 ? b_hi + 4096u * 4u : b_hi) + ks * 2 * LBO, LBO, 128u);
        wgmma_tf32_n64_rA(d, term == 1 ? al[ks] : ah[ks], bd, (ks > 0 || term > 0) ? 1 : 0);
      }
  };
  const uint32_t b = s_u32(Bcan);
  acc_fence(dL);
  acc_fence(dG);
  wgmma_fence();
  mma(dL, b);
  mma(dG, b + 8192u * 4u);
  wgmma_commit();
  wgmma_wait_all();
  acc_fence(dL);
  acc_fence(dG);
  frag_acc(dL, 0, L);
  frag_acc(dG, 0, G);
}

// Forward.  Per tile: ang . Wg^T of both branches (registers) while the Ha rows land; pre = ((Ha + ang.Wg^T) + Hb) +
// Xc of both branches (line_first_layer).  !HIDDEN: the buffer is free from here on, so the next tile's Ha copy is
// issued before ang_out = ang + silu(pre_L) sigm(pre_G) is formed in registers and stored.  HIDDEN: silu(pre) . W2^T
// + b2 per branch (register A operands), m = silu(u) sigm(v) in registers, stored over the thread's own Ha values of
// columns 0..63, and aggB[b] += m in one scatter pass over the warpgroup's 64 rows; then the next tile's copy.
template <bool HIDDEN>
__global__ void __launch_bounds__(128 * LineFwd<HIDDEN>::WG, 1) k_line_fwd(const LineArgs a) {
  using S = typename LineFwd<HIDDEN>::Smem;
  constexpr int WG = LineFwd<HIDDEN>::WG;
  extern __shared__ __align__(128) float smem[];
  const int tid = threadIdx.x, w = tid >> 7, lr = tid & 127;  // warpgroup; thread lr < TW copies row lr
  uint64_t* mbar = reinterpret_cast<uint64_t*>(smem) + w;      // this warpgroup's buffer
  const float* Wg = smem + S::kW;
  const float* W2 = smem + S::kW + 16384;  // HIDDEN
  const float* b2s = smem + S::kB2;        // HIDDEN
  float* P = smem + S::kBuf + w * TW * LDE;
  int* s_a = reinterpret_cast<int*>(smem + S::kIdx) + w * TW;
  int* s_b = reinterpret_cast<int*>(smem + S::kIdx) + (WG + w) * TW;
  int* s_c = reinterpret_cast<int*>(smem + S::kIdx) + (2 * WG + w) * TW;

  // tile numbers in 32 bits (up to 2^37 angles): the three-warpgroup forward has no register to spare
  const int ntiles = (int)((a.A + TW - 1) / TW), first = WG * blockIdx.x + w, step = WG * gridDim.x;
  if (tid == 0) {
    for (int i = 0; i < WG; i++) mbar_init(reinterpret_cast<uint64_t*>(smem) + i, 1);
    fence_barrier_init();
  }
  AngleIdx nxt = angle_row(a, (int64_t)first * TW + lr, lr < TW);
  // loop-invariant operands, once per CTA
  stage_w<128 * WG>(smem + S::kW, a.Wgcan, 4096);
  if (HIDDEN) {
    stage_w<128 * WG>(smem + S::kW + 16384, a.W2can, 4096);
    if (tid < 128) smem[S::kB2 + tid] = a.b2[tid];
  }
  __syncthreads();
  if (first < ntiles)  // the last CTA's later warpgroups have no tile when the tile count is not a multiple of WG
    line_issue_ha_wg(a, first, nxt, lr, P, mbar, s_a, s_b, s_c);
  nxt = angle_row(a, (int64_t)(first + step) * TW + lr, lr < TW);

  const Map m;
  Map mL = m, mG = m;  // the first layer's columns of each branch
  mL.branch = 0;
  mG.branch = 1;
  int it = 0;
  for (int t = first; t < ntiles; t += step, it++) {
    int64_t r0 = (int64_t)t * TW;
    asm volatile("" : "+l"(r0));  // row addresses formed per tile: carried across tiles they hold registers
    const int nvalid = (int)min((int64_t)TW, a.A - r0);
    float L[2][AC], G[2][AC];
    {
      float x[8][4];
      line_ang_frag(a, m, r0, nvalid, x);
      wg_sync(w);  // the tile's indices are published
      wg_mma64_pair(x, Wg, L, G);
    }
    mbar_wait(mbar, (uint32_t)it & 1u);
    line_first_layer(a, mL, P, s_b, s_c, nvalid, L);
    line_first_layer(a, mG, P, s_b, s_c, nvalid, G);
    if constexpr (!HIDDEN) {
      fence_proxy_async_smem();  // this thread's generic accesses of the buffer come before its bulk refill
      wg_sync(w);                // the warpgroup is done with the buffer and the indices
      if (t + step < ntiles) {
        line_issue_ha_wg(a, t + step, nxt, lr, P, mbar, s_a, s_b, s_c);
        nxt = angle_row(a, ((int64_t)t + 2 * step) * TW + lr, lr < TW);
      }
      // ang_out = ang + silu(pre_L) sigm(pre_G), the angle rows re-read (L2) as float2 pairs
#pragma unroll
      for (int ii = 0; ii < 2; ii++) {
        const int r = m.row(ii);
        if (r >= nvalid) continue;
        const float* ang = a.ang + (size_t)(r0 + r) * D;
        float* out = a.ang_out + (size_t)(r0 + r) * D;
        float2 av[AC / 2];
#pragma unroll
        for (int jj = 0; jj < AC / 2; jj++) av[jj] = __ldg(reinterpret_cast<const float2*>(ang + m.col(2 * jj)));
#pragma unroll
        for (int jj = 0; jj < AC / 2; jj++) {
          const float l0 = silu_f(L[ii][2 * jj]), l1 = silu_f(L[ii][2 * jj + 1]);
          const float g0 = sigm(G[ii][2 * jj]), g1 = sigm(G[ii][2 * jj + 1]);
          st_f2(out + m.col(2 * jj), av[jj].x + l0 * g0, av[jj].y + l1 * g1);
        }
      }
    } else {
      // hid = silu(pre) straight into the second layer; u (L) and v (G) + b2
#pragma unroll
      for (int ii = 0; ii < 2; ii++)
#pragma unroll
        for (int j = 0; j < AC; j++) L[ii][j] = silu_f(L[ii][j]);
      wg_mm64_acc(L, 0, W2, L);
#pragma unroll
      for (int ii = 0; ii < 2; ii++)
#pragma unroll
        for (int j = 0; j < AC; j++) L[ii][j] = silu_f(L[ii][j] + b2s[m.col(j)]);
#pragma unroll
      for (int ii = 0; ii < 2; ii++)
#pragma unroll
        for (int j = 0; j < AC; j++) G[ii][j] = silu_f(G[ii][j]);
      wg_mm64_acc(G, 0, W2 + 8192, G);
      // m = silu(u) sigm(v), over the thread's own Ha values of columns 0..63
#pragma unroll
      for (int ii = 0; ii < 2; ii++)
#pragma unroll
        for (int jj = 0; jj < AC / 2; jj++) {
          const float g0 = sigm(G[ii][2 * jj] + b2s[64 + m.col(2 * jj)]);
          const float g1 = sigm(G[ii][2 * jj + 1] + b2s[64 + m.col(2 * jj + 1)]);
          st_f2(P + m.row(ii) * LDE + m.col(2 * jj), L[ii][2 * jj] * g0, L[ii][2 * jj + 1] * g1);
        }
      wg_sync(w);
      scatter_rows<16, TW, 128>(P, s_b, a.aggB, nullptr, nullptr, nullptr, nullptr);  // aggB[b] += m
      fence_proxy_async_smem();  // this thread's generic accesses of the buffer come before its bulk refill
      wg_sync(w);                // the warpgroup is done with the buffer and the indices
      if (t + step < ntiles) {
        line_issue_ha_wg(a, t + step, nxt, lr, P, mbar, s_a, s_b, s_c);
        nxt = angle_row(a, ((int64_t)t + 2 * step) * TW + lr, lr < TW);
      }
    }
  }
}

// Bond-conv backward (HIDDEN), in the 128-angle layout (LineSmem): its four weight images (Wg, W2, W2^T, Wg^T) do not
// fit next to one buffer per warpgroup, so they take turns in the one slot.  P (buffer it & 1) holds the tile's Ha rows,
// then its pre-activations, each thread's over its own Ha values, then their adjoints gpre, which the scatter phase and
// gpre.Wg read row-major; H (the other buffer) holds the angle rows, then the last layer's outputs parked at each
// thread's own positions -- u (L), oG = sigm(v) (G) -- so that the reverse keeps one 64-row half of accumulators live
// at a time and reads its own and its partner's values back.  Both products of the hidden layer take their A operand
// from registers.  Once H has been read for the last time (by the elementwise reverse), the next tile's Ha rows are
// copied into it (H becomes the next tile's P); once the scatter phase and gang += gpre.Wg have read P, the next
// tile's angle rows go into its columns 64..127 (P becomes the next tile's H).  Weight images through the one slot: Wg
// -> W2 -> W2^T -> Wg^T per tile.
__device__ __forceinline__ void line_bwd_bond(const LineArgs& a) {
  extern __shared__ __align__(128) float smem[];
  const LineSm sm{smem};
  const float* b2s = sm.b2();
  const int tid = threadIdx.x;
  const int64_t ntiles = (a.A + TM - 1) / TM, step = gridDim.x;
  AngleIdx nxt = line_prologue(a, sm);
  uint32_t wpar = 0;

  int it = 0;
  for (int64_t t = blockIdx.x; t < ntiles; t += step, it++) {
    const int s = it & 1;
    float* P = sm.buf(s);
    float* H = sm.buf(s ^ 1);
    const int* s_a = sm.idx(s, 0);
    const int* s_b = sm.idx(s, 1);
    const int* s_c = sm.idx(s, 2);
    const int64_t r0 = t * TM;
    const int nvalid = (int)min((int64_t)TM, a.A - r0);
    const bool more = t + step < ntiles;
    const Map m;
    float acc[AR][AC];
    mbar_wait(&sm.abar()[s], stage_parity(it));
    mbar_wait(sm.wbar(), wpar);  // Wg
    wpar ^= 1;
    gemm64(H, LDE, 64, sm.W() + m.branch * 8192, acc);
    __syncthreads();  // both warpgroups have read the angle rows and Wg: H and the slot may be written
    if (tid == 0) bulk_g2s_image(sm.W(), a.W2can, 16384 * 4, sm.wbar());
    mbar_wait(&sm.hbar()[s], stage_parity(it));
    line_first_layer(a, m, P, s_b, s_c, nvalid, acc);
    // pre overwrites the thread's own Ha values in P (same thread, same addresses); silu(pre) . W2^T + b2 = u | v
#pragma unroll
    for (int i = 0; i < AR; i++)
#pragma unroll
      for (int jj = 0; jj < AC / 2; jj++) {
        float& x0 = acc[i][2 * jj];
        float& x1 = acc[i][2 * jj + 1];
        st_f2(P + m.row(i) * LDE + m.branch * 64 + m.col(2 * jj), x0, x1);
        x0 = silu_f(x0);
        x1 = silu_f(x1);
      }
    mbar_wait(sm.wbar(), wpar);  // W2
    wpar ^= 1;
    // the pre-activation of the last layer of this GatedMLP (u | v = silu(pre) . W2^T + b2, one 64-row half at a
    // time), parked in H at the thread's own positions as u (L) and oG = sigm(v) (G)
#pragma unroll
    for (int h = 0; h < 2; h++) {
      wg_mm64_acc(acc, h, sm.W() + m.branch * 8192, acc);
#pragma unroll
      for (int ii = 0; ii < 2; ii++)
#pragma unroll
        for (int jj = 0; jj < AC / 2; jj++) {
          const int i = 2 * h + ii;
          const float u0 = acc[i][2 * jj] + b2s[m.branch * 64 + m.col(2 * jj)];
          const float u1 = acc[i][2 * jj + 1] + b2s[m.branch * 64 + m.col(2 * jj + 1)];
          st_f2(H + m.row(i) * LDE + m.branch * 64 + m.col(2 * jj), m.branch == 0 ? u0 : sigm(u0),
                m.branch == 0 ? u1 : sigm(u1));
        }
    }
    __syncthreads();  // H holds both branches' values and W2 has been read
    if (tid == 0) bulk_g2s_image(sm.W(), a.W2Tcan, 16384 * 4, sm.wbar());
    // reverse, per 64-row half: acc = dE/du (L) / dE/dv (G) from the values parked in H (the partner's sigm(v) /
    // silu(u) formed from them); ghid = [gu . W2L, gv . W2G] from the adjoints in registers and gpre = ghid *
    // dsilu(pre), into P over pre
#pragma unroll
    for (int h = 0; h < 2; h++) {
      bool ok[2];
      float2 gm2[2][AC / 2];  // both rows' 16 upstream gradients, loaded as float2 pairs before any is used
#pragma unroll
      for (int ii = 0; ii < 2; ii++) {
        const int r = m.row(2 * h + ii);
        ok[ii] = r < nvalid;
        const float* gsrc = a.gaggB + (size_t)(ok[ii] ? s_b[r] : 0) * D;
#pragma unroll
        for (int jj = 0; jj < AC / 2; jj++)
          gm2[ii][jj] = ok[ii] ? *reinterpret_cast<const float2*>(gsrc + m.col(2 * jj)) : make_float2(0.f, 0.f);
      }
#pragma unroll
      for (int ii = 0; ii < 2; ii++) {
        const int i = 2 * h + ii;
        const int r = m.row(i);
#pragma unroll
        for (int j = 0; j < AC; j++) {
          const float2 ow2 = ld_f2(H + r * LDE + m.branch * 64 + m.col(j & ~1));        // u (L) / oG (G)
          const float2 pt2 = ld_f2(H + r * LDE + (1 - m.branch) * 64 + m.col(j & ~1));  // the partner's
          const float x = (j & 1) ? ow2.y : ow2.x;
          const float pt = (j & 1) ? pt2.y : pt2.x;
          float g = 0.f;
          if (ok[ii]) {
            const float gm = (j & 1) ? gm2[ii][j >> 1].y : gm2[ii][j >> 1].x;
            if (m.branch == 0) {
              const float sg = sigm(x);
              g = gm * pt * (sg * (1.f + x * (1.f - sg)));
            } else {
              const float oL = silu_f(pt);
              g = gm * oL * x * (1.f - x);
            }
          }
          acc[i][j] = g;
        }
      }
      if (h == 0) mbar_wait(sm.wbar(), wpar);  // W2^T
      wg_mm64_acc(acc, h, sm.W() + m.branch * 8192, acc);
#pragma unroll
      for (int ii = 0; ii < 2; ii++)
#pragma unroll
        for (int jj = 0; jj < AC / 2; jj++) {
          const int i = 2 * h + ii;
          float* p = P + m.row(i) * LDE + m.branch * 64 + m.col(2 * jj);
          const float2 pre = ld_f2(p);
          st_f2(p, acc[i][2 * jj] * dsilu_f(pre.x), acc[i][2 * jj + 1] * dsilu_f(pre.y));
        }
    }
    wpar ^= 1;
    fence_proxy_async_smem();  // this thread's generic accesses of H come before its bulk refill
    __syncthreads();           // H, its stage's index arrays and W2^T are free; P holds gpre
    if (more) {
      line_issue_ha(a, sm, t + step, nxt, H, s ^ 1);
      nxt = angle_idx(a, (t + 2 * step) * TM + tid);
    }
    if (tid == 0) bulk_g2s_image(sm.W(), a.WgTcan, 16384 * 4, sm.wbar());
    // ---- scatter phase (reads P and this tile's index arrays) ----
    // gHb[b] += gpre and gXc[c] += gpre (segmented), gHa[a] += gpre: one pass over P
    scatter_rows<32>(P, s_b, a.gHb, s_c, a.gXc, s_a, a.gHa);
    // gang += gpre @ Wg   (K = 128, N = 64) on the tensor cores: warpgroup w takes rows 64 w .. 64 w + 63.  Each angle
    // row belongs to this tile alone, so the update is a fire-and-forget reduction: one addition per element, as a
    // load-add-store would do.
    mbar_wait(sm.wbar(), wpar);  // Wg^T
    wpar ^= 1;
    {
      float d[32];
      const uint32_t bh = s_u32(sm.W()), bl = bh + 64u * 128u * 4u;
      wg_mm64(P, LDE, 64 * m.branch, 0, bh, bl, 0, false, d);
      wg_mm64(P, LDE, 64 * m.branch, 64, bh, bl, 64, true, d);
#pragma unroll
      for (int q = 0; q < 32; q += 2) {
        const int r = 64 * m.branch + m.rb + 8 * ((q >> 1) & 1), c = 8 * (q >> 2) + m.cb;
        if (r < nvalid) red_add_v2(&a.gang[(size_t)(r0 + r) * D + c], d[q], d[q + 1]);
      }
    }
    fence_proxy_async_smem();  // this thread's generic accesses of P come before its bulk refill
    __syncthreads();           // P and Wg^T are free
    if (more) {
      line_issue_ang(a, sm, t + step, P, s ^ 1);
      if (tid == 0) bulk_g2s_image(sm.W(), a.Wgcan, 16384 * 4, sm.wbar());
    }
  }
}

// Angle-update backward (!HIDDEN), in the warpgroup layout of the forward with Wg and Wg^T resident.  Per tile: pre of
// both branches as in the forward (u = pre_L, v = pre_G); the elementwise reverse in registers, with oG = sigm(v) and g
// the tile's own rows of gang (loaded at the top of the tile with the angle rows): gpre_L = dE/du = g oG dsilu(u),
// gpre_G = dE/dv = g silu(u) oG (1 - oG), stored over the thread's own Ha values; gHb[b] += gpre and gXc[c] += gpre
// (segmented) and gHa[a] += gpre in one scatter pass over the warpgroup's 64 rows; the next tile's copy; then, while it
// flies, gang += gpre . Wg (K = 128) with gpre as the register A operand, one K half per branch.  The thread that adds
// into a gang element has read its upstream value at the top of the tile, so the update is a fire-and-forget
// reduction: one addition per element, as a load-add-store would do.
__device__ __forceinline__ void line_bwd_angle(const LineArgs& a) {
  using S = LineBwdSmem;
  constexpr int WG = LBWG;
  extern __shared__ __align__(128) float smem[];
  const int tid = threadIdx.x, w = tid >> 7, lr = tid & 127;  // warpgroup; thread lr < TW copies row lr
  uint64_t* mbar = reinterpret_cast<uint64_t*>(smem) + w;      // this warpgroup's buffer
  const float* Wg = smem + S::kW;
  const float* WgT = smem + S::kW + 16384;
  float* P = smem + S::kBuf + w * TW * LDE;
  int* s_a = reinterpret_cast<int*>(smem + S::kIdx) + w * TW;
  int* s_b = reinterpret_cast<int*>(smem + S::kIdx) + (WG + w) * TW;
  int* s_c = reinterpret_cast<int*>(smem + S::kIdx) + (2 * WG + w) * TW;

  // tile numbers in 32 bits (up to 2^37 angles): the three-warpgroup forward has no register to spare
  const int ntiles = (int)((a.A + TW - 1) / TW), first = WG * blockIdx.x + w, step = WG * gridDim.x;
  if (tid == 0) {
    for (int i = 0; i < WG; i++) mbar_init(reinterpret_cast<uint64_t*>(smem) + i, 1);
    fence_barrier_init();
  }
  AngleIdx nxt = angle_row(a, (int64_t)first * TW + lr, lr < TW);
  // loop-invariant operands, once per CTA
  stage_w<128 * WG>(smem + S::kW, a.Wgcan, 4096);
  stage_w<128 * WG>(smem + S::kW + 16384, a.WgTcan, 4096);
  __syncthreads();
  if (first < ntiles)  // the last CTA's second warpgroup has no tile when the tile count is odd
    line_issue_ha_wg(a, first, nxt, lr, P, mbar, s_a, s_b, s_c);
  nxt = angle_row(a, (int64_t)(first + step) * TW + lr, lr < TW);

  const Map m;
  Map mL = m, mG = m;  // the first layer's columns of each branch
  mL.branch = 0;
  mG.branch = 1;
  int it = 0;
  for (int t = first; t < ntiles; t += step, it++) {
    int64_t r0 = (int64_t)t * TW;
    asm volatile("" : "+l"(r0));  // row addresses formed per tile: carried across tiles they hold registers
    const int nvalid = (int)min((int64_t)TW, a.A - r0);
    // the upstream gradients (both rows' 16 gang pairs) load with the angle rows, before anything waits
    bool ok[2];
    float2 gm2[2][AC / 2];
#pragma unroll
    for (int ii = 0; ii < 2; ii++) {
      const int r = m.row(ii);
      ok[ii] = r < nvalid;
      const float* gsrc = a.gang + (size_t)(r0 + (ok[ii] ? r : 0)) * D;
#pragma unroll
      for (int jj = 0; jj < AC / 2; jj++)
        gm2[ii][jj] = ok[ii] ? *reinterpret_cast<const float2*>(gsrc + m.col(2 * jj)) : make_float2(0.f, 0.f);
    }
    float L[2][AC], G[2][AC];
    {
      float x[8][4];
      line_ang_frag(a, m, r0, nvalid, x);
      wg_sync(w);  // the tile's indices are published
      wg_mma64_pair(x, Wg, L, G);
    }
    mbar_wait(mbar, (uint32_t)it & 1u);
    line_first_layer(a, mL, P, s_b, s_c, nvalid, L);
    line_first_layer(a, mG, P, s_b, s_c, nvalid, G);
    // elementwise reverse, in place: L <- gpre_L, G <- gpre_G
#pragma unroll
    for (int ii = 0; ii < 2; ii++) {
#pragma unroll
      for (int j = 0; j < AC; j++) {
        const float u = L[ii][j], oG = sigm(G[ii][j]);
        float gu = 0.f, gv = 0.f;
        if (ok[ii]) {
          const float gm = (j & 1) ? gm2[ii][j >> 1].y : gm2[ii][j >> 1].x;
          const float sg = sigm(u);
          gu = gm * oG * (sg * (1.f + u * (1.f - sg)));
          gv = gm * silu_f(u) * oG * (1.f - oG);
        }
        L[ii][j] = gu;
        G[ii][j] = gv;
      }
#pragma unroll
      for (int jj = 0; jj < AC / 2; jj++) {
        st_f2(P + m.row(ii) * LDE + m.col(2 * jj), L[ii][2 * jj], L[ii][2 * jj + 1]);
        st_f2(P + m.row(ii) * LDE + 64 + m.col(2 * jj), G[ii][2 * jj], G[ii][2 * jj + 1]);
      }
    }
    wg_sync(w);  // P holds the tile's gpre
    scatter_rows<32, TW, 128>(P, s_b, a.gHb, s_c, a.gXc, s_a, a.gHa);
    fence_proxy_async_smem();  // this thread's generic accesses of the buffer come before its bulk refill
    wg_sync(w);                // the warpgroup is done with the buffer and the indices
    if (t + step < ntiles) {
      line_issue_ha_wg(a, t + step, nxt, lr, P, mbar, s_a, s_b, s_c);
      nxt = angle_row(a, ((int64_t)t + 2 * step) * TW + lr, lr < TW);
    }
    // gang += gpre . Wg   (K = 128, N = 64) on the tensor cores, from the registers while the next tile's copy flies
    {
      float v[8][4], d[32];
      const uint32_t bh = s_u32(WgT), bl = bh + 64u * 128u * 4u;
      acc_frag(L, 0, v);
      wg_mma64(v, bh, bl, 0, false, d);
      acc_frag(G, 0, v);
      wg_mma64(v, bh, bl, 64, true, d);
#pragma unroll
      for (int q = 0; q < 32; q += 2) {
        const int r = m.rb + 8 * ((q >> 1) & 1), c = 8 * (q >> 2) + m.cb;
        if (r < nvalid) red_add_v2(&a.gang[(size_t)(r0 + r) * D + c], d[q], d[q + 1]);
      }
    }
  }
}

static_assert(128 * LBWG == NT, "both backward kernels run 256-thread CTAs");
template <bool HIDDEN>
__global__ void __launch_bounds__(NT, 1) k_line_bwd(const LineArgs a) {
  if constexpr (HIDDEN)
    line_bwd_bond(a);
  else
    line_bwd_angle(a);
}

void launch_line_fwd(cudaStream_t st, const LineArgs& a, bool hidden, int num_sms) {
  if (a.A <= 0) return;
  static PerDeviceOnce attr;
  if (auto once_ = attr.first(); once_) {
    B2M_CK(cudaFuncSetAttribute(k_line_fwd<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)LineFwd<true>::Smem::bytes));
    B2M_CK(cudaFuncSetAttribute(k_line_fwd<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)LineFwd<false>::Smem::bytes));
  }
  with_flags(
      [&](auto kHidden) {
        using F = LineFwd<decltype(kHidden)::value>;
        launch(k_line_fwd<kHidden>, std::min(cdiv(cdiv(a.A, TW), F::WG), num_sms), 128 * F::WG, F::Smem::bytes, st, a);
      },
      hidden);
}
void launch_line_bwd(cudaStream_t st, const LineArgs& a, bool hidden, int num_sms) {
  if (a.A <= 0) return;
  static PerDeviceOnce attr;
  if (auto once_ = attr.first(); once_) {
    B2M_CK(cudaFuncSetAttribute(k_line_bwd<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LineSmem::bytes));
    B2M_CK(cudaFuncSetAttribute(k_line_bwd<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LineBwdSmem::bytes));
  }
  if (hidden)
    launch(k_line_bwd<true>, std::min(cdiv(a.A, TM), num_sms), NT, LineSmem::bytes, st, a);
  else
    launch(k_line_bwd<false>, std::min(cdiv(cdiv(a.A, TW), LBWG), num_sms), NT, LineBwdSmem::bytes, st, a);
}

// ============================================================================================
// bond update (node-level, after the W_out GEMM):  h' = h + upd * w3b(d_b)
// ============================================================================================
// 128 bonds per block, 16-byte accesses: these are pure streaming kernels (300 MB per launch at 97 k atoms) and ran at a
// third of the HBM rate with 32 bonds per block and 4-byte accesses
constexpr int BNR = 128;  // bonds per block
template <int MODE>  // 0: fwd, 1: bwd (gupd, gdb), 2: h0 backward (gdb only)
__global__ void __launch_bounds__(256) k_bond_node(int nb, const float4* __restrict__ b_vec, RadialParams rp,
                                                   const float* __restrict__ W /*[64][9]*/,
                                                   const float* __restrict__ x0 /*h | gh | gh0*/,
                                                   const float* __restrict__ x1 /*upd*/, float* __restrict__ out,
                                                   float* __restrict__ gdb) {
  extern __shared__ float bn_smem[];
  float(*be_s)[12] = reinterpret_cast<float(*)[12]>(bn_smem);                 // [BNR][12]
  float(*dbe_s)[12] = reinterpret_cast<float(*)[12]>(bn_smem + BNR * 12);     // [BNR][12]
  float* Ws = bn_smem + 2 * BNR * 12;                                         // [64][9]
  float(*P)[68] = reinterpret_cast<float(*)[68]>(bn_smem + 2 * BNR * 12 + 576);  // [BNR][68]  MODE 1: gh*upd, MODE 2: gh0
  const int b0 = blockIdx.x * BNR, tid = threadIdx.x;
  for (int i = tid; i < 576; i += 256) Ws[i] = W[i];
  for (int i = tid; i < BNR * 9; i += 256) {
    const int r = i / 9, k = i % 9;
    float be = 0.f, dbe = 0.f;
    if (b0 + r < nb) rbf_env_k(b_vec[b0 + r].w, rp.freq[k], rp, be, dbe);
    be_s[r][k] = be;
    dbe_s[r][k] = dbe;
  }
  __syncthreads();
  for (int i = tid; i < BNR * 16; i += 256) {  // (row, 4 columns) per item
    const int r = i >> 4, c = (i & 15) * 4;
    float4 pv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (b0 + r < nb) {
      const size_t o = (size_t)(b0 + r) * 64 + c;
      const float4 a0 = *reinterpret_cast<const float4*>(x0 + o);
      if (MODE == 2) {
        pv = a0;
      } else {
        float w[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int k = 0; k < 9; k++) {
          const float b = be_s[r][k];
#pragma unroll
          for (int j = 0; j < 4; j++) w[j] = fmaf(b, Ws[(c + j) * 9 + k], w[j]);
        }
        const float4 a1 = *reinterpret_cast<const float4*>(x1 + o);
        if (MODE == 0) {
          *reinterpret_cast<float4*>(out + o) = make_float4(a0.x + a1.x * w[0], a0.y + a1.y * w[1], a0.z + a1.z * w[2], a0.w + a1.w * w[3]);
        } else {
          *reinterpret_cast<float4*>(out + o) = make_float4(a0.x * w[0], a0.y * w[1], a0.z * w[2], a0.w * w[3]);
          pv = make_float4(a0.x * a1.x, a0.y * a1.y, a0.z * a1.z, a0.w * a1.w);
        }
      }
    }
    if (MODE != 0) *reinterpret_cast<float4*>(&P[r][c]) = pv;
  }
  if (MODE == 1 || MODE == 2) {
    __syncthreads();
    // gdb[r] += sum_k (sum_c P[r][c] W[c][k]) dbe_k : two threads per bond (k parity), partial sums combined by shuffle
    {
      const int r = tid >> 1, par = tid & 1;
      float tot = 0.f;
      for (int k = par; k < 9; k += 2) {
        float sacc = 0.f;
#pragma unroll 8
        for (int c = 0; c < 64; c++) sacc = fmaf(P[r][c], Ws[c * 9 + k], sacc);
        tot += sacc * dbe_s[r][k];
      }
      tot += __shfl_xor_sync(0xffffffffu, tot, 1);
      if (par == 0 && b0 + r < nb) gdb[b0 + r] += tot;
    }
  }
}
constexpr size_t kBondNodeSmem = (size_t)(2 * BNR * 12 + 576 + BNR * 68) * sizeof(float);
template <int MODE>
static void launch_bond_node(cudaStream_t st, int nb, const float4* b_vec, RadialParams rp, const float* W, const float* x0,
                             const float* x1, float* out, float* gdb) {
  static PerDeviceOnce attr;
  if (auto once_ = attr.first(); once_)
    B2M_CK(cudaFuncSetAttribute(k_bond_node<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBondNodeSmem));
  launch(k_bond_node<MODE>, cdiv(nb, BNR), 256, kBondNodeSmem, st, nb, b_vec, rp, W, x0, x1, out, gdb);
}
void launch_bond_update_fwd(cudaStream_t st, int nb, const float4* b_vec, RadialParams rp3, const float* W3bw,
                            const float* h, const float* upd, float* hout) {
  if (nb <= 0) return;
  launch_bond_node<0>(st, nb, b_vec, rp3, W3bw, h, upd, hout, nullptr);
}
void launch_bond_update_bwd(cudaStream_t st, int nb, const float4* b_vec, RadialParams rp3, const float* W3bw,
                            const float* gh, const float* upd, float* gupd, float* gdb) {
  if (nb <= 0) return;
  launch_bond_node<1>(st, nb, b_vec, rp3, W3bw, gh, upd, gupd, gdb);
}
void launch_h0_bwd(cudaStream_t st, int nb, const float4* b_vec, RadialParams rp, const float* Wbe, const float* gh0,
                   float* gdb) {
  if (nb <= 0) return;
  launch_bond_node<2>(st, nb, b_vec, rp, Wbe, gh0, nullptr, nullptr, gdb);
}

// theta / Fourier backward (128 angles per block)
constexpr int ANR = 128;
__global__ void __launch_bounds__(256) k_angle_init_bwd(int64_t na, const int* __restrict__ a_in,
                                                        const int* __restrict__ a_out,
                                                        const float4* __restrict__ b_vec, const float* __restrict__ fa,
                                                        const float* __restrict__ Wae, const float* __restrict__ gang0,
                                                        float* __restrict__ gbvec) {
  extern __shared__ float ab_smem[];
  float(*G)[65] = reinterpret_cast<float(*)[65]>(ab_smem);                  // [ANR][65]
  float(*gf_s)[12] = reinterpret_cast<float(*)[12]>(ab_smem + ANR * 65);    // [ANR][12]
  float* Ws = ab_smem + ANR * 65 + ANR * 12;                                // [64][9]
  const int64_t r0 = (int64_t)blockIdx.x * ANR;
  const int tid = threadIdx.x;
  for (int i = tid; i < 576; i += 256) Ws[i] = Wae[i];
  for (int i = tid; i < ANR * 64; i += 256) {
    const int r = i >> 6, c = i & 63;
    G[r][c] = (r0 + r < na) ? gang0[(size_t)(r0 + r) * 64 + c] : 0.f;
  }
  __syncthreads();
  for (int i = tid; i < ANR * 9; i += 256) {
    const int r = i / 9, k = i % 9;
    float s = 0.f;
#pragma unroll 8
    for (int c = 0; c < 64; c++) s = fmaf(G[r][c], Ws[c * 9 + k], s);
    gf_s[r][k] = s;
  }
  __syncthreads();
  if (tid < ANR && r0 + tid < na) {
    const int64_t r = r0 + tid;
    const int ia = a_in[r], ib = a_out[r];
    const AngleGeom g = angle_geom(b_vec[ia], b_vec[ib]);
    const float ipi = 0.318309886183790672f;
    float gth = 0.f;
    for (int k = 0; k < 5; k++) {
      float s, c;
      sincosf(g.theta * fa[k], &s, &c);
      gth -= gf_s[tid][2 * k] * fa[k] * s;
      if (k >= 1) gth += gf_s[tid][2 * k - 1] * fa[k] * c;
    }
    gth *= ipi;
    const float lo = -1.f + 1e-7f, hi = 1.f - 1e-7f;
    float gcos = 0.f;
    if (g.cos_raw >= lo && g.cos_raw <= hi) gcos = -gth / sqrtf(1.f - g.cc * g.cc);
    const float inn = 1.f / (g.na * g.nb);
    const float ia2 = 1.f / (g.na * g.na), ib2 = 1.f / (g.nb * g.nb);
    for (int x = 0; x < 3; x++) {
      const float dva = -g.vb[x] * inn - g.cos_raw * g.va[x] * ia2;
      const float dvb = -g.va[x] * inn - g.cos_raw * g.vb[x] * ib2;
      atomicAdd(&gbvec[(size_t)ia * 3 + x], gcos * dva);
      atomicAdd(&gbvec[(size_t)ib * 3 + x], gcos * dvb);
    }
  }
}
constexpr size_t kAngleBwdSmem = (size_t)(ANR * 65 + ANR * 12 + 576) * sizeof(float);
void launch_angle_init_bwd(cudaStream_t st, int64_t na, const int* a_in, const int* a_out, const float4* b_vec,
                           const float* fa, const float* Wae, const float* gang0, float* gbvec) {
  if (na <= 0) return;
  static PerDeviceOnce attr;
  if (auto once_ = attr.first(); once_)
    B2M_CK(cudaFuncSetAttribute(k_angle_init_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAngleBwdSmem));
  launch(k_angle_init_bwd, cdiv(na, ANR), 256, kAngleBwdSmem, st, na, a_in, a_out, b_vec, fa, Wae, gang0, gbvec);
}

// ============================================================================================
// readout
// ============================================================================================
// kAtomic: also the per-atom energy of every row, atom_e[gid[row]] = scale * v + elem_ref + mean_per_atom
// kWeighted: every row's energy (and per-atom energy) times wgt[gid[row]] (heat flux: cell mask or position seed)
template <bool kAtomic, bool kWeighted = false>
__global__ void __launch_bounds__(256) k_rowdot(int n, const float* __restrict__ X, const float* __restrict__ w,
                                                float bias, float* __restrict__ out, double* __restrict__ sum,
                                                const int* __restrict__ type, const double* __restrict__ elem_ref,
                                                float scale, const int* __restrict__ gid, double* __restrict__ atom_e,
                                                double mean_per_atom, const float* __restrict__ wgt) {
  // one warp per row
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  float v = 0.f;
  if (warp < n) {
    const float2 x = reinterpret_cast<const float2*>(X + (size_t)warp * 64)[lane];
    const float2 ww = reinterpret_cast<const float2*>(w)[lane];
    v = x.x * ww.x + x.y * ww.y;
  }
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __shared__ double part[8];
  double contrib = 0.0;
  if (warp < n && lane == 0) {
    v += bias;
    if (out) out[warp] = v;
    contrib = readout_energy<kAtomic, kWeighted>(warp, v, scale, type, elem_ref, gid, atom_e, mean_per_atom, wgt);
  }
  if (sum) {
    if (lane == 0) part[threadIdx.x >> 5] = contrib;
    __syncthreads();
    if (threadIdx.x == 0) {
      double s = 0.0;
      for (int i = 0; i < 8; i++) s += part[i];
      atomicAdd(sum, s);
    }
  }
}
void launch_rowdot(cudaStream_t st, int n, const float* X, const float* w, float bias, float* out, double* sum,
                   const int* type, const double* elem_ref, float scale, const int* gid, double* atom_e,
                   double mean_per_atom, const float* wgt) {
  with_flags(
      [&](auto kAtomic, auto kWeighted) {
        launch(k_rowdot<kAtomic, kWeighted>, cdiv((int64_t)n * 32, 256), 256, 0, st, n, X, w, bias, out, sum, type,
               elem_ref, scale, gid, atom_e, mean_per_atom, wgt);
      },
      atom_e != nullptr, wgt != nullptr);
}
// kWeighted: row r's seed times wgt[gid[r]]
template <bool kWeighted = false>
__global__ void k_readout_seed(int n, const float* __restrict__ pre, const float* __restrict__ w, float scale,
                               float* __restrict__ g, const int* __restrict__ gid, const float* __restrict__ wgt) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)n * 64) return;
  if constexpr (kWeighted) scale *= wgt[gid[i >> 6]];
  g[i] = scale * w[i & 63] * dsilu_f(pre[i]);
}
void launch_readout_seed(cudaStream_t st, int n, const float* pre, const float* w, float scale, float* g,
                         const int* gid, const float* wgt) {
  with_flags(
      [&](auto kWeighted) {
        launch(k_readout_seed<kWeighted>, cdiv((int64_t)n * 64, 256), 256, 0, st, n, pre, w, scale, g, gid, wgt);
      },
      wgt != nullptr);
}

// ============================================================================================
// final geometry backward: forces and virial
// ============================================================================================
// kAtomic: also 1/2 v (x) g into both endpoints' rows of the per-atom virial array (final_tail.cuh)
template <bool kAtomic>
__global__ void __launch_bounds__(256) k_edge_final(int64_t E, const int* __restrict__ e_src,
                                                    const int* __restrict__ e_dst, const int* __restrict__ e_bond,
                                                    const float4* __restrict__ e_vec, const int* __restrict__ gid,
                                                    const float* __restrict__ gd, const float* __restrict__ gdb,
                                                    const float* __restrict__ gbvec, float* __restrict__ forces,
                                                    double* __restrict__ virial, float* __restrict__ atom_vir) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  float vir[9];
#pragma unroll
  for (int k = 0; k < 9; k++) vir[k] = 0.f;
  int asrc = 0, adst = -1;
  if (e < E) {
    const float4 v = e_vec[e];
    float g = gd[e];
    float gx = 0.f, gy = 0.f, gz = 0.f;
    const int b = e_bond[e];
    if (b >= 0) {
      g += gdb[b];
      gx = gbvec[(size_t)b * 3], gy = gbvec[(size_t)b * 3 + 1], gz = gbvec[(size_t)b * 3 + 2];
    }
    const float s = g / v.w;
    gx += s * v.x, gy += s * v.y, gz += s * v.z;
    const int gdst = gid[e_dst[e]], gsrc = gid[e_src[e]];
    scatter_edge(forces, gsrc, gdst, v, make_float3(gx, gy, gz), vir);
    if constexpr (kAtomic) asrc = gsrc, adst = gdst;
  }
  edge_virial_tail<kAtomic>(atom_vir, asrc, adst, vir, virial);
}
void launch_edge_final(cudaStream_t st, int64_t E, const int* e_src, const int* e_dst, const int* e_bond,
                       const float4* e_vec, const int* gid, const float* gd, const float* gdb, const float* gbvec,
                       float* forces, double* virial, float* atom_vir) {
  with_flags(
      [&](auto kAtomic) {
        launch(k_edge_final<kAtomic>, cdiv(E, 256), 256, 0, st, E, e_src, e_dst, e_bond, e_vec, gid, gd, gdb, gbvec,
               forces, virial, atom_vir);
      },
      atom_vir != nullptr);
}

// kAtomic: also 1/2 v (x) g of this partition's part of g into both endpoints' per-atom virial rows (the bond's
// owner adds its own part in k_edge_final, so the sum over partitions is exact)
template <bool kAtomic>
__global__ void __launch_bounds__(256) k_halo_bond_final(int b0, int b1, const int* __restrict__ b_src_gid,
                                                         const int* __restrict__ b_dst, const float4* __restrict__ b_vec,
                                                         const int* __restrict__ gid, const float* __restrict__ gdb,
                                                         const float* __restrict__ gbvec, float* __restrict__ forces,
                                                         double* __restrict__ virial, float* __restrict__ atom_vir) {
  const int b = b0 + blockIdx.x * blockDim.x + threadIdx.x;
  float vir[9];
#pragma unroll
  for (int k = 0; k < 9; k++) vir[k] = 0.f;
  if (b < b1) {
    const float4 v = b_vec[b];
    const float s = gdb[b] / v.w;
    const float gx = gbvec[(size_t)b * 3] + s * v.x, gy = gbvec[(size_t)b * 3 + 1] + s * v.y,
                gz = gbvec[(size_t)b * 3 + 2] + s * v.z;
    const int gdst = gid[b_dst[b]], gsrc = b_src_gid[b];
    scatter_edge(forces, gsrc, gdst, v, make_float3(gx, gy, gz), vir);
    if constexpr (kAtomic) {
      float w[9];
#pragma unroll
      for (int k = 0; k < 9; k++) w[k] = 0.5f * vir[k];
      red_add_virial(atom_vir, gdst, w);
      red_add_virial(atom_vir, gsrc, w);
    }
  }
  block_sum_add(vir, virial);
}
void launch_halo_bond_final(cudaStream_t st, int b0, int b1, const int* b_src_gid, const int* b_dst,
                            const float4* b_vec, const int* gid, const float* gdb, const float* gbvec, float* forces,
                            double* virial, float* atom_vir) {
  if (b1 <= b0) return;
  with_flags(
      [&](auto kAtomic) {
        launch(k_halo_bond_final<kAtomic>, cdiv(b1 - b0, 256), 256, 0, st, b0, b1, b_src_gid, b_dst, b_vec, gid, gdb,
               gbvec, forces, virial, atom_vir);
      },
      atom_vir != nullptr);
}

// ============================================================================================
// halo pack / unpack
// ============================================================================================
__global__ void k_gather_rows(int n, int w4, const int* __restrict__ idx, const float4* __restrict__ src,
                              float4* __restrict__ dst) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)n * w4) return;
  const int r = (int)(i / w4), c = (int)(i % w4);
  dst[i] = src[(size_t)idx[r] * w4 + c];
}
__global__ void k_scatter_add_rows(int n, int w, const int* __restrict__ idx, const float* __restrict__ src,
                                   float* __restrict__ dst) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)n * w) return;
  const int r = (int)(i / w), c = (int)(i % w);
  dst[(size_t)idx[r] * w + c] += src[i];  // to-lists hold unique rows
}
void launch_gather_rows(cudaStream_t st, int n, int width, const int* idx, const float* src, float* dst) {
  const int w4 = width / 4;
  launch(k_gather_rows, cdiv((int64_t)n * w4, 256), 256, 0, st, n, w4, idx, reinterpret_cast<const float4*>(src),
         reinterpret_cast<float4*>(dst));
}
void launch_scatter_add_rows(cudaStream_t st, int n, int width, const int* idx, const float* src, float* dst) {
  launch(k_scatter_add_rows, cdiv((int64_t)n * width, 256), 256, 0, st, n, width, idx, src, dst);
}

}  // namespace b2m
