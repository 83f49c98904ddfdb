// kernels_mace.cu -- MACE with hidden features C x 0e, C x 0e + C x 1o or C x 0e + C x 1o + C x 2e on the same
// partitioned CSR graph as the CHGNet and TensorNet paths.  Arithmetic as oracle/mace_ref.py and, for 0e+1o features,
// tests/mace_eq_ref.py and, for 0e+1o+2e, tests/mace_l2_ref.py state it (the conventions are written down there once),
// and the ZBL pair term and Agnesi transform as tests/mace_zbl_ref.py
// states them; engine_mace.inl runs these kernels stage by stage.
//
// First generation: the node- and edge-level products (radial MLP, linear_up, the per-l mixes, the product linear) run
// on the wgmma row GEMM of the other paths (kernels_wg.cu, engine.cu tc_mm); the element-dependent mixes
// (skip_tp) read the element's C x C block per atom; the symmetric contraction is one thread per (atom, channel) that
// walks the nonzero terms of U, which every channel shares.  Aggregations walk the CSR-by-destination rows (no atomics
// in the forward); the reverse scatters to sources with atomics.
#include <utility>

#include "final_tail.cuh"
#include "mace_cg.cuh"
#include "mace_cg_l2.cuh"
#include "mace_state.cuh"

namespace b2m {

namespace {

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + __expf(-x)); }
__device__ __forceinline__ float silu_f(float x) { return x * sigm(x); }
__device__ __forceinline__ float dsilu_f(float x) {
  const float s = sigm(x);
  return s * (1.f + x * (1.f - s));
}

// ============================================================================================
// edge geometry: spherical harmonics (oracle/mace_ref.py sh_basis) and Bessel x polynomial cutoff
// ============================================================================================
// value and gradient (w.r.t. the unit vector's components) carried together
struct Dual {
  float v, x, y, z;
};
__device__ __forceinline__ Dual operator*(Dual a, Dual b) {
  return {a.v * b.v, a.x * b.v + a.v * b.x, a.y * b.v + a.v * b.y, a.z * b.v + a.v * b.z};
}
__device__ __forceinline__ Dual operator*(float s, Dual a) { return {s * a.v, s * a.x, s * a.y, s * a.z}; }
__device__ __forceinline__ Dual operator-(Dual a, Dual b) { return {a.v - b.v, a.x - b.x, a.y - b.y, a.z - b.z}; }

template <class T>
__device__ __forceinline__ T smul(float s, T a) { return s * a; }

// Y[0..nsh) of the unit vector (x, y, z); T = float or Dual
template <class T>
__device__ __forceinline__ void sh16(T x, T y, T z, T one, int nsh, T* Y) {
  Y[0] = one;
  if (nsh <= 1) return;
  const float s3 = 1.7320508075688772f;
  Y[1] = smul(s3, x), Y[2] = smul(s3, y), Y[3] = smul(s3, z);
  if (nsh <= 4) return;
  const float s15 = 3.872983346207417f, s5h = 1.118033988749895f, s15h = 1.9364916731037085f;
  const T xx = x * x, yy = y * y, zz = z * z;
  Y[4] = smul(s15, x * y), Y[5] = smul(s15, y * z), Y[6] = smul(s5h, smul(2.f, zz) - xx - yy), Y[7] = smul(s15, x * z);
  Y[8] = smul(s15h, xx - yy);
  if (nsh <= 9) return;
  const float a = 2.091650066335189f, b = 10.246950765959598f, c = 1.6201851746019651f, d = 1.3228756555322954f;
  const T q = smul(4.f, zz) - xx - yy;
  Y[9] = smul(a, y * (smul(3.f, xx) - yy));
  Y[10] = smul(b, x * y * z);
  Y[11] = smul(c, y * q);
  Y[12] = smul(d, z * (smul(2.f, zz) - smul(3.f, xx) - smul(3.f, yy)));
  Y[13] = smul(c, x * q);
  Y[14] = smul(0.5f * b, z * (xx - yy));
  Y[15] = smul(a, x * (xx - smul(3.f, yy)));
}

// mace's polynomial envelope of d / r (exponent p, zero from d = r on) and its derivative in d
__device__ __forceinline__ void poly_env(float d, float r, int ip, float& f, float& df) {
  const float x = d / r;
  if (x >= 1.f) {
    f = 0.f, df = 0.f;
    return;
  }
  const float p = (float)ip;
  const float xp1 = __powf(x, p - 1.f), xp = xp1 * x, xp1p = xp * x, xp2 = xp1p * x;
  f = 1.f - 0.5f * (p + 1.f) * (p + 2.f) * xp + p * (p + 2.f) * xp1p - 0.5f * p * (p + 1.f) * xp2;
  df = (-0.5f * (p + 1.f) * (p + 2.f) * p * xp1 + p * (p + 2.f) * (p + 1.f) * xp - 0.5f * p * (p + 1.f) * (p + 2.f) * xp1p) /
       r;
}

// polynomial cutoff of the radial basis and its derivative in d
__device__ __forceinline__ void poly_cut(float d, const MaceRadial& rp, float& f, float& df) {
  poly_env(d, rp.r_max, rp.p, f, df);
}

// Agnesi transform x = 1 + a s^q / (1 + s^(q - p)), s = d / r0, and dx/dd
__device__ __forceinline__ void agnesi(float d, float r0, const MaceCore& c, float& x, float& dx) {
  const float s = d / r0, sq = powf(s, c.aq), sqp = powf(s, c.aq - c.ap), den = 1.f / (1.f + sqp);
  x = 1.f + c.aa * sq * den;
  dx = c.aa * (sq / s) * (c.aq + c.ap * sqp) * den * den / r0;
}

// ZBL energy of one directed edge u -> v, V = 1/2 14.3996 Z_u Z_v / d phi(d / a_uv) env_p(d / (rho'_u + rho'_v)), and dV/dd
__device__ __forceinline__ void zbl(float d, float4 eu, float4 ev, const MaceCore& c, float& V, float& dV) {
  float env, denv;
  poly_env(d, eu.z + ev.z, c.zp, env, denv);
  const float ia = (eu.y + ev.y) / c.za, t = d * ia;  // 1 / a_uv
  const float x0 = expf(-3.2f * t), x1 = expf(-0.9423f * t), x2 = expf(-0.4029f * t), x3 = expf(-0.2016f * t);
  const float phi = c.zc[0] * x0 + c.zc[1] * x1 + c.zc[2] * x2 + c.zc[3] * x3;
  const float dphi = -ia * (3.2f * c.zc[0] * x0 + 0.9423f * c.zc[1] * x1 + 0.4029f * c.zc[2] * x2 + 0.2016f * c.zc[3] * x3);
  const float k = 0.5f * 14.3996f * eu.x * ev.x, rd = 1.f / d;
  V = k * rd * phi * env;
  dV = k * rd * ((dphi - phi * rd) * env + phi * denv);
}

template <bool kSpecies>
__global__ void k_mace_edge_geom(int64_t E, const float4* __restrict__ e_vec, MaceRadial rp, int nsh,
                                 float* __restrict__ Y, float* __restrict__ eb, const int* __restrict__ e_src,
                                 const int* __restrict__ e_dst, const int* __restrict__ type, MaceCore core) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= E) return;
  const float4 v = e_vec[e];
  const float d = v.w, rd = 1.f / d;
  float y[kMaceMaxNsh];
  sh16<float>(v.x * rd, v.y * rd, v.z * rd, 1.f, nsh, y);
#pragma unroll
  for (int k = 0; k < kMaceMaxNsh; k++) Y[e * kMaceMaxNsh + k] = k < nsh ? y[k] : 0.f;
  float f, df;
  poly_cut(d, rp, f, df);
  float xb = d, rxb = rd;  // the Bessel argument: d, or (kSpecies: Agnesi on) the transformed x; f stays f(d)
  if constexpr (kSpecies) {
    float dx;
    agnesi(d, 0.5f * (core.elem[type[e_src[e]]].w + core.elem[type[e_dst[e]]].w), core, xb, dx);
    rxb = 1.f / xb;
  }
  for (int n = 0; n < rp.nbp; n++) eb[e * rp.nbp + n] = n < rp.nb ? rp.pref * sinf(rp.w[n] * xb) * rxb * f : 0.f;
}

// one thread per owned atom i: e_lin[i] += sum_{e -> i} V_e in CSR row order, before any readout adds to it
__global__ void k_mace_zbl(int n_own, const int* __restrict__ row_ptr, const int* __restrict__ e_src,
                           const float4* __restrict__ e_vec, const int* __restrict__ type, MaceCore core,
                           float* __restrict__ e_lin) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_own) return;
  const float4 ev = core.elem[type[i]];
  float s = 0.f;
  for (int e = row_ptr[i]; e < row_ptr[i + 1]; e++) {
    float V, dV;
    zbl(e_vec[e].w, core.elem[type[e_src[e]]], ev, core, V, dV);
    s += V;
  }
  e_lin[i] += s;
}

__global__ void k_mace_embed(int n, int C, const int* __restrict__ type, const float* __restrict__ W,
                             float* __restrict__ h0) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)n * C) return;
  const int r = (int)(i / C), c = (int)(i % C);
  h0[i] = W[(size_t)type[r] * C + c];
}

// A[lm][t][c] = sum_{e -> t} R[e][l(lm) C + c] Y[e][lm] u[src(e)][c]
__global__ void k_mace_msg(int n_own, int C, int L1, const int* __restrict__ row_ptr, const int* __restrict__ e_src,
                           const float* __restrict__ R, const float* __restrict__ Y, const float* __restrict__ u,
                           float* __restrict__ A) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)n_own * C) return;
  const int t = (int)(i / C), c = (int)(i % C), nsh = L1 * L1, RW = L1 * C;
  float acc[kMaceMaxNsh];
#pragma unroll
  for (int k = 0; k < kMaceMaxNsh; k++) acc[k] = 0.f;
  for (int e = row_ptr[t]; e < row_ptr[t + 1]; e++) {
    const float uc = u[(size_t)e_src[e] * C + c];
    const float* re = R + (size_t)e * RW + c;
    const float* ye = Y + (size_t)e * kMaceMaxNsh;
#pragma unroll
    for (int l = 0; l < 4; l++) {
      if (l >= L1) break;
      const float r = re[l * C] * uc;
      for (int m = l * l; m < (l + 1) * (l + 1); m++) acc[m] = fmaf(r, ye[m], acc[m]);
    }
  }
  const size_t plane = (size_t)n_own * C;
#pragma unroll
  for (int k = 0; k < kMaceMaxNsh; k++)
    if (k < nsh) A[k * plane + i] = acc[k];
}

// reverse of k_mace_msg: gR[e][l C + c] = u sum_{m in l} gA[m] Y[m] ; gY[e][m] += sum_c gA[m] R[l] u (warp sums over
// 32 channels of one destination, then one atomic) ; gu[src][c] += sum_m gA[m] R[l(m)] Y[m]
__global__ void k_mace_msg_bwd(int n_own, int C, int L1, const int* __restrict__ row_ptr, const int* __restrict__ e_src,
                               const float* __restrict__ R, const float* __restrict__ Y, const float* __restrict__ u,
                               const float* __restrict__ gA, float* __restrict__ gR, float* __restrict__ gY,
                               float* __restrict__ gu) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)n_own * C) return;  // n_own * C is a multiple of 32: whole warps leave together
  const int t = (int)(i / C), c = (int)(i % C), nsh = L1 * L1, RW = L1 * C, lane = threadIdx.x & 31;
  const size_t plane = (size_t)n_own * C;
  float ga[kMaceMaxNsh];
#pragma unroll
  for (int k = 0; k < kMaceMaxNsh; k++) ga[k] = k < nsh ? gA[k * plane + i] : 0.f;
  for (int e = row_ptr[t]; e < row_ptr[t + 1]; e++) {
    const int s = e_src[e];
    const float uc = u[(size_t)s * C + c];
    const float* re = R + (size_t)e * RW + c;
    const float* ye = Y + (size_t)e * kMaceMaxNsh;
    float gus = 0.f;
#pragma unroll
    for (int l = 0; l < 4; l++) {
      if (l >= L1) break;
      const float r = re[l * C];
      float gr = 0.f;
      for (int m = l * l; m < (l + 1) * (l + 1); m++) {
        const float y = ye[m];
        gr = fmaf(ga[m], y, gr);
        float gy = ga[m] * r * uc;
        for (int o = 16; o > 0; o >>= 1) gy += __shfl_xor_sync(0xffffffffu, gy, o);
        if (lane == 0) atomicAdd(&gY[(size_t)e * kMaceMaxNsh + m], gy);
      }
      gR[(size_t)e * RW + l * C + c] = gr * uc;
      gus = fmaf(gr, r, gus);
    }
    atomicAdd(&gu[(size_t)s * C + c], gus);
  }
}

// out[lm][i][:] (+)= in[lm][i][:] @ W[type[i]][l(lm)] : one block of C threads per row i; each weight element is read
// once per row and applied to the 2l + 1 components of its l
__global__ void k_mace_elem_mix(int n, int C, int L1, int nsh, const int* __restrict__ type, const float* __restrict__ W,
                                const float* __restrict__ in, float* __restrict__ out, int accum) {
  __shared__ float x[7][128];
  const int i = blockIdx.x, c2 = threadIdx.x;
  const int z = type[i];
  const size_t plane = (size_t)n * C;
  const int Lw = nsh == 1 ? 1 : L1;
  for (int l = 0; l < Lw; l++) {
    const int m0 = l * l, nm = 2 * l + 1;
    __syncthreads();
    for (int m = 0; m < nm; m++) x[m][c2] = in[(m0 + m) * plane + (size_t)i * C + c2];
    __syncthreads();
    const float* Wb = W + ((size_t)z * Lw + l) * C * C + c2;
    float acc[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int c = 0; c < C; c++) {
      const float w = Wb[(size_t)c * C];
#pragma unroll
      for (int m = 0; m < 7; m++)
        if (m < nm) acc[m] = fmaf(w, x[m][c], acc[m]);
    }
    for (int m = 0; m < nm; m++) {
      float* o = out + (m0 + m) * plane + (size_t)i * C + c2;
      *o = accum ? *o + acc[m] : acc[m];
    }
  }
}

// symmetric contraction, one thread per (atom, channel): the channel's 16 components of A sit in shared memory (column
// per thread), the terms are read by every thread of the warp at the same address
template <bool kBwd>
__global__ void __launch_bounds__(128) k_mace_symc(int n_own, int C, int nsh, int Ktot, const int* __restrict__ type,
                                                   const float* __restrict__ A, const MaceTerm* __restrict__ terms,
                                                   int nterms, const float* __restrict__ w, const float* __restrict__ gB,
                                                   float* __restrict__ out) {
  __shared__ float a[kMaceMaxNsh][128];
  __shared__ float ga[kBwd ? kMaceMaxNsh : 1][128];
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)n_own * C) return;
  const int tid = threadIdx.x, t = (int)(i / C), c = (int)(i % C);
  const size_t plane = (size_t)n_own * C;
#pragma unroll
  for (int k = 0; k < kMaceMaxNsh; k++) {
    a[k][tid] = k < nsh ? A[k * plane + i] : 0.f;
    if constexpr (kBwd) ga[k][tid] = 0.f;
  }
  const float* wz = w + (size_t)type[t] * Ktot * C + c;
  const float g = kBwd ? gB[i] : 0.f;
  float acc = 0.f;
  for (int j = 0; j < nterms; j++) {
    const MaceTerm tm = terms[j];
    const int nu = tm.idx >> 24, i1 = tm.idx & 255, i2 = (tm.idx >> 8) & 255, i3 = (tm.idx >> 16) & 255;
    const float cw = tm.coef * wz[(size_t)tm.kg * C];
    const float a1 = a[i1][tid], a2 = nu >= 2 ? a[i2][tid] : 1.f, a3 = nu >= 3 ? a[i3][tid] : 1.f;
    if constexpr (!kBwd) {
      acc = fmaf(cw, a1 * a2 * a3, acc);
    } else {
      const float s = cw * g;
      ga[i1][tid] += s * a2 * a3;
      if (nu >= 2) ga[i2][tid] += s * a1 * a3;
      if (nu >= 3) ga[i3][tid] += s * a1 * a2;
    }
  }
  if constexpr (!kBwd) {
    out[i] = acc;
  } else {
#pragma unroll
    for (int k = 0; k < kMaceMaxNsh; k++)
      if (k < nsh) out[k * plane + i] = ga[k][tid];
  }
}

// ============================================================================================
// 0e+1o node features (layers t >= 1 of a model with hidden_irreps C x 0e + C x 1o)
// ============================================================================================
// the coupling list of one max_ell (mace_cg.cuh), expanded with X
#define MACE_CG_EXPAND(L, X) \
  if constexpr ((L) == 1) { MACE_CG_1(X) } else if constexpr ((L) == 2) { MACE_CG_2(X) } else { MACE_CG_3(X) }

// Am[slot(l_out, m, j)] = sum_{e -> t} R[e][p] sum CG u[src][l_in m1] Y[e][l_sh m2] over the paths p of conv_paths,
// one thread per (atom, channel) with the 4 + npaths + nsh operands of an edge in registers; no atomics
template <int kL>
__global__ void __launch_bounds__(256) k_mace_msg_eq(int n_own, int C, const int* __restrict__ row_ptr,
                                                     const int* __restrict__ e_src, const float* __restrict__ R,
                                                     const float* __restrict__ Y, const float* __restrict__ u,
                                                     float* __restrict__ Am) {
  constexpr int NP = mace_npaths(kL, 1), NS = mace_nslots(kL, 1), NSH = (kL + 1) * (kL + 1);
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)n_own * C) return;
  const int t = (int)(i / C), c = (int)(i % C);
  float acc[NS];
#pragma unroll
  for (int k = 0; k < NS; k++) acc[k] = 0.f;
  for (int e = row_ptr[t]; e < row_ptr[t + 1]; e++) {
    const float* us = u + (size_t)e_src[e] * 4 * C + c;
    const float uu[4] = {us[0], us[C], us[2 * C], us[3 * C]};
    const float* re = R + (size_t)e * NP * C + c;
    float r[NP];
#pragma unroll
    for (int p = 0; p < NP; p++) r[p] = re[p * C];
    const float* ye = Y + (size_t)e * kMaceMaxNsh;
    float y[NSH];
#pragma unroll
    for (int k = 0; k < NSH; k++) y[k] = ye[k];
#define MACE_X(p, iu, iy, s, cf) acc[s] = fmaf((cf) * r[p], uu[iu] * y[iy], acc[s]);
    MACE_CG_EXPAND(kL, MACE_X)
#undef MACE_X
  }
  int s = 0;
#pragma unroll
  for (int l = 0; l <= kL; l++) {
    const int np = mace_np_l(kL, l, 1);
    float* blk = Am + (size_t)mace_slot_base(kL, l, 1) * n_own * C;
#pragma unroll
    for (int m = 0; m < 2 * l + 1; m++)
#pragma unroll
      for (int j = 0; j < np; j++) blk[(((size_t)m * n_own + t) * np + j) * C + c] = acc[s++];
  }
}

// reverse of k_mace_msg_eq: gR over R in place (the thread of (dst, c) is the only reader and writer of R[e][.][c] for
// its edges), gY[e][k] += the warp's 32 channels (one atomic per warp), gu[src][4][c] += (atomics)
template <int kL>
__global__ void __launch_bounds__(256) k_mace_msg_eq_bwd(int n_own, int C, const int* __restrict__ row_ptr,
                                                         const int* __restrict__ e_src, float* __restrict__ R,
                                                         const float* __restrict__ Y, const float* __restrict__ u,
                                                         const float* __restrict__ gAm, float* __restrict__ gY,
                                                         float* __restrict__ gu) {
  constexpr int NP = mace_npaths(kL, 1), NS = mace_nslots(kL, 1), NSH = (kL + 1) * (kL + 1);
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)n_own * C) return;  // n_own * C is a multiple of 32: whole warps leave together
  const int t = (int)(i / C), c = (int)(i % C), lane = threadIdx.x & 31;
  float ga[NS];
  {
    int s = 0;
#pragma unroll
    for (int l = 0; l <= kL; l++) {
      const int np = mace_np_l(kL, l, 1);
      const float* blk = gAm + (size_t)mace_slot_base(kL, l, 1) * n_own * C;
#pragma unroll
      for (int m = 0; m < 2 * l + 1; m++)
#pragma unroll
        for (int j = 0; j < np; j++) ga[s++] = blk[(((size_t)m * n_own + t) * np + j) * C + c];
    }
  }
  for (int e = row_ptr[t]; e < row_ptr[t + 1]; e++) {
    const int src = e_src[e];
    const float* us = u + (size_t)src * 4 * C + c;
    const float uu[4] = {us[0], us[C], us[2 * C], us[3 * C]};
    float* re = R + (size_t)e * NP * C + c;
    float r[NP], gr[NP];
#pragma unroll
    for (int p = 0; p < NP; p++) r[p] = re[p * C], gr[p] = 0.f;
    const float* ye = Y + (size_t)e * kMaceMaxNsh;
    float y[NSH], gy[NSH];
#pragma unroll
    for (int k = 0; k < NSH; k++) y[k] = ye[k], gy[k] = 0.f;
    float g4[4] = {0.f, 0.f, 0.f, 0.f};
#define MACE_X(p, iu, iy, s, cf)                  \
  {                                               \
    const float g = (cf) * ga[s];                 \
    gr[p] = fmaf(g, uu[iu] * y[iy], gr[p]);       \
    const float gq = g * r[p];                    \
    g4[iu] = fmaf(gq, y[iy], g4[iu]);             \
    gy[iy] = fmaf(gq, uu[iu], gy[iy]);            \
  }
    MACE_CG_EXPAND(kL, MACE_X)
#undef MACE_X
#pragma unroll
    for (int p = 0; p < NP; p++) re[p * C] = gr[p];
#pragma unroll
    for (int k = 1; k < NSH; k++) {  // Y[0] = 1 carries no gradient
      float v = gy[k];
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) atomicAdd(&gY[(size_t)e * kMaceMaxNsh + k], v);
    }
    float* gs = gu + (size_t)src * 4 * C + c;
#pragma unroll
    for (int k = 0; k < 4; k++) atomicAdd(gs + k * C, g4[k]);
  }
}

// out[i][m][:] (+)= in[i][m][:] @ W[type[i]][l(m)], m < ncomp (1 or 4; k2e: 9), rows of pitch ldi / ldo: one block of C
// threads per row, each weight element read once per row and applied to the components of its l
template <bool k2e>
__global__ void k_mace_elem_mix_rows(int n, int C, int ncomp, int ldi, int ldo, const int* __restrict__ type,
                                     const float* __restrict__ W, const float* __restrict__ in, float* __restrict__ out,
                                     int accum) {
  __shared__ float x[k2e ? 9 : 4][128];
  const int i = blockIdx.x, c2 = threadIdx.x;
  if constexpr (k2e) {
    const int z = type[i];
    for (int m = 0; m < 9; m++) x[m][c2] = in[(size_t)i * ldi + m * C + c2];
    __syncthreads();
    const float* W0 = W + (size_t)z * 3 * C * C + c2;
    const float *W1 = W0 + (size_t)C * C, *W2 = W1 + (size_t)C * C;
    float a[9];
#pragma unroll
    for (int m = 0; m < 9; m++) a[m] = 0.f;
    for (int c = 0; c < C; c++) {
      const float w0 = W0[(size_t)c * C], w1 = W1[(size_t)c * C], w2 = W2[(size_t)c * C];
      a[0] = fmaf(w0, x[0][c], a[0]);
#pragma unroll
      for (int m = 1; m < 4; m++) a[m] = fmaf(w1, x[m][c], a[m]);
#pragma unroll
      for (int m = 4; m < 9; m++) a[m] = fmaf(w2, x[m][c], a[m]);
    }
#pragma unroll
    for (int m = 0; m < 9; m++) {
      float* o = out + (size_t)i * ldo + m * C + c2;
      *o = accum ? *o + a[m] : a[m];
    }
  } else {
    const int z = type[i], Lw = ncomp == 4 ? 2 : 1;
    for (int m = 0; m < ncomp; m++) x[m][c2] = in[(size_t)i * ldi + m * C + c2];
    __syncthreads();
    const float* W0 = W + (size_t)z * Lw * C * C + c2;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    if (ncomp == 4) {
      const float* W1 = W0 + (size_t)C * C;
      for (int c = 0; c < C; c++) {
        const float w0 = W0[(size_t)c * C], w1 = W1[(size_t)c * C];
        a0 = fmaf(w0, x[0][c], a0), a1 = fmaf(w1, x[1][c], a1), a2 = fmaf(w1, x[2][c], a2), a3 = fmaf(w1, x[3][c], a3);
      }
    } else {
      for (int c = 0; c < C; c++) a0 = fmaf(W0[(size_t)c * C], x[0][c], a0);
    }
    const float a[4] = {a0, a1, a2, a3};
    for (int m = 0; m < ncomp; m++) {
      float* o = out + (size_t)i * ldo + m * C + c2;
      *o = accum ? *o + a[m] : a[m];
    }
  }
}

// symmetric contraction with a 1o (kNo = 4) or 1o and 2e (kNo = 9) output: as k_mace_symc, with the term's output
// slot o (MaceTerm) selecting one of kNo accumulators (forward) or upstream adjoints (reverse); B / gB [kNo][n_own][C]
template <bool kBwd, int kNo>
__global__ void __launch_bounds__(128) k_mace_symc_eq(int n_own, int C, int nsh, int Ktot, const int* __restrict__ type,
                                                      const float* __restrict__ A, const MaceTerm* __restrict__ terms,
                                                      int nterms, const float* __restrict__ w,
                                                      const float* __restrict__ gB, float* __restrict__ out) {
  static_assert(kNo == 4 || kNo == 9, "output slots of a 0e+1o or 0e+1o+2e product");
  __shared__ float a[kMaceMaxNsh][128];
  __shared__ float ga[kBwd ? kMaceMaxNsh : 1][128];
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)n_own * C) return;
  const int tid = threadIdx.x, t = (int)(i / C), c = (int)(i % C);
  const size_t plane = (size_t)n_own * C;
#pragma unroll
  for (int k = 0; k < kMaceMaxNsh; k++) {
    a[k][tid] = k < nsh ? A[k * plane + i] : 0.f;
    if constexpr (kBwd) ga[k][tid] = 0.f;
  }
  const float* wz = w + (size_t)type[t] * Ktot * C + c;
  float g[kNo];
#pragma unroll
  for (int o = 0; o < kNo; o++) g[o] = 0.f;
  if constexpr (kBwd) {
#pragma unroll
    for (int o = 0; o < kNo; o++) g[o] = gB[o * plane + i];
  }
  float acc[kNo];
#pragma unroll
  for (int o = 0; o < kNo; o++) acc[o] = 0.f;
  for (int j = 0; j < nterms; j++) {
    const MaceTerm tm = terms[j];
    // slots 0..3 keep bits 28..29 (bit 31 stays clear); slot 8 sets bit 31, hence the unsigned field for kNo = 9
    const int nu = (tm.idx >> 24) & 3, o = kNo == 4 ? (tm.idx >> 28) & 3 : (int)((uint32_t)tm.idx >> 28);
    const int i1 = tm.idx & 255, i2 = (tm.idx >> 8) & 255, i3 = (tm.idx >> 16) & 255;
    const float cw = tm.coef * wz[(size_t)tm.kg * C];
    const float a1 = a[i1][tid], a2 = nu >= 2 ? a[i2][tid] : 1.f, a3 = nu >= 3 ? a[i3][tid] : 1.f;
    if constexpr (!kBwd) {
      const float v = cw * (a1 * a2 * a3);  // the same o for the whole warp: the selects do not diverge
      if constexpr (kNo == 4) {
        acc[0] += o == 0 ? v : 0.f, acc[1] += o == 1 ? v : 0.f, acc[2] += o == 2 ? v : 0.f, acc[3] += o == 3 ? v : 0.f;
      } else {
#pragma unroll
        for (int k = 0; k < kNo; k++) acc[k] += o == k ? v : 0.f;
      }
    } else {
      float go = g[kNo - 1];
      if constexpr (kNo == 4) {
        go = o == 0 ? g[0] : o == 1 ? g[1] : o == 2 ? g[2] : g[3];
      } else {
#pragma unroll
        for (int k = kNo - 2; k >= 0; k--) go = o == k ? g[k] : go;
      }
      const float s = cw * go;
      ga[i1][tid] += s * a2 * a3;
      if (nu >= 2) ga[i2][tid] += s * a1 * a3;
      if (nu >= 3) ga[i3][tid] += s * a1 * a2;
    }
  }
  if constexpr (!kBwd) {
#pragma unroll
    for (int o = 0; o < kNo; o++) out[o * plane + i] = acc[o];
  } else {
#pragma unroll
    for (int k = 0; k < kMaceMaxNsh; k++)
      if (k < nsh) out[k * plane + i] = ga[k][tid];
  }
}

// ============================================================================================
// 0e+1o+2e node features (layers t >= 1 of a model with hidden_irreps C x 0e + C x 1o + C x 2e)
// ============================================================================================
#define MACE_CG_L2_EXPAND(L, X) \
  if constexpr ((L) == 2) { MACE_CG_L2_2(X) } else { MACE_CG_L2_3(X) }

// the slots [S0, S0 + NS) of output l kLo and the paths [P0, P0 + NPL) that reach it, and which u / Y components those
// paths read (bit masks, from the coupling list)
template <int kL, int kLo>
struct MaceL2Group {
  static constexpr int NP = mace_npaths(kL, 2), NPL = mace_np_l(kL, kLo, 2), P0 = mace_path_base(kL, kLo, 2);
  static constexpr int S0 = mace_slot_base(kL, kLo, 2), NS = (2 * kLo + 1) * NPL, NSH = (kL + 1) * (kL + 1);
  static constexpr uint32_t mask(bool y) {
    uint32_t m = 0;
#define MACE_X(p, iu, iy, s, cf) \
  if ((s) >= S0 && (s) < S0 + NS) m |= 1u << (y ? (iy) : (iu));
    MACE_CG_L2_EXPAND(kL, MACE_X)
#undef MACE_X
    return m;
  }
  static constexpr uint32_t UM = mask(false), YM = mask(true);
};

// Am[slot(l_out = kLo, m, j)] = sum_{e -> t} R[e][p] sum CG u[src][l_in m1] Y[e][l_sh m2] over the paths p of that l_out:
// one launch per l_out (all 71 slots of max_ell 3 in one thread would not fit the register file with the edge operands;
// DESIGN.md §11.3), one thread per (atom, channel), no atomics
template <int kL, int kLo>
__global__ void __launch_bounds__(256) k_mace_msg_l2(int n_own, int C, const int* __restrict__ row_ptr,
                                                     const int* __restrict__ e_src, const float* __restrict__ R,
                                                     const float* __restrict__ Y, const float* __restrict__ u,
                                                     float* __restrict__ Am) {
  using G = MaceL2Group<kL, kLo>;
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)n_own * C) return;
  const int t = (int)(i / C), c = (int)(i % C);
  float acc[G::NS];
#pragma unroll
  for (int k = 0; k < G::NS; k++) acc[k] = 0.f;
  for (int e = row_ptr[t]; e < row_ptr[t + 1]; e++) {
    const float* us = u + (size_t)e_src[e] * 9 * C + c;
    float uu[9];
#pragma unroll
    for (int k = 0; k < 9; k++) uu[k] = (G::UM >> k) & 1 ? us[k * C] : 0.f;
    const float* re = R + (size_t)e * G::NP * C + c;
    float r[G::NP];
#pragma unroll
    for (int p = 0; p < G::NP; p++) r[p] = p >= G::P0 && p < G::P0 + G::NPL ? re[p * C] : 0.f;
    const float* ye = Y + (size_t)e * kMaceMaxNsh;
    float y[G::NSH];
#pragma unroll
    for (int k = 0; k < G::NSH; k++) y[k] = (G::YM >> k) & 1 ? ye[k] : 0.f;
#define MACE_X(p, iu, iy, s, cf) \
  if constexpr ((s) >= G::S0 && (s) < G::S0 + G::NS) acc[(s) - G::S0] = fmaf((cf) * r[p], uu[iu] * y[iy], acc[(s) - G::S0]);
    MACE_CG_L2_EXPAND(kL, MACE_X)
#undef MACE_X
  }
  float* blk = Am + (size_t)G::S0 * n_own * C;
#pragma unroll
  for (int m = 0; m < 2 * kLo + 1; m++)
#pragma unroll
    for (int j = 0; j < G::NPL; j++) blk[(((size_t)m * n_own + t) * G::NPL + j) * C + c] = acc[m * G::NPL + j];
}

// reverse of k_mace_msg_l2 for output l kLo: gR over R in place for the paths of that l_out (the thread of (dst, c) is
// the only reader and writer of R[e][p][c], and no other launch touches those paths), gY[e][k] += the warp's 32 channels
// (one atomic per warp), gu[src][9][c] += (atomics)
template <int kL, int kLo>
__global__ void __launch_bounds__(256) k_mace_msg_l2_bwd(int n_own, int C, const int* __restrict__ row_ptr,
                                                         const int* __restrict__ e_src, float* __restrict__ R,
                                                         const float* __restrict__ Y, const float* __restrict__ u,
                                                         const float* __restrict__ gAm, float* __restrict__ gY,
                                                         float* __restrict__ gu) {
  using G = MaceL2Group<kL, kLo>;
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)n_own * C) return;  // n_own * C is a multiple of 32: whole warps leave together
  const int t = (int)(i / C), c = (int)(i % C), lane = threadIdx.x & 31;
  float ga[G::NS];
  {
    const float* blk = gAm + (size_t)G::S0 * n_own * C;
#pragma unroll
    for (int m = 0; m < 2 * kLo + 1; m++)
#pragma unroll
      for (int j = 0; j < G::NPL; j++) ga[m * G::NPL + j] = blk[(((size_t)m * n_own + t) * G::NPL + j) * C + c];
  }
  for (int e = row_ptr[t]; e < row_ptr[t + 1]; e++) {
    const int src = e_src[e];
    const float* us = u + (size_t)src * 9 * C + c;
    float uu[9], g9[9];
#pragma unroll
    for (int k = 0; k < 9; k++) uu[k] = (G::UM >> k) & 1 ? us[k * C] : 0.f, g9[k] = 0.f;
    float* re = R + (size_t)e * G::NP * C + c;
    float r[G::NP], gr[G::NP];
#pragma unroll
    for (int p = 0; p < G::NP; p++) r[p] = p >= G::P0 && p < G::P0 + G::NPL ? re[p * C] : 0.f, gr[p] = 0.f;
    const float* ye = Y + (size_t)e * kMaceMaxNsh;
    float y[G::NSH], gy[G::NSH];
#pragma unroll
    for (int k = 0; k < G::NSH; k++) y[k] = (G::YM >> k) & 1 ? ye[k] : 0.f, gy[k] = 0.f;
#define MACE_X(p, iu, iy, s, cf)                    \
  if constexpr ((s) >= G::S0 && (s) < G::S0 + G::NS) { \
    const float g = (cf) * ga[(s) - G::S0];         \
    gr[p] = fmaf(g, uu[iu] * y[iy], gr[p]);         \
    const float gq = g * r[p];                      \
    g9[iu] = fmaf(gq, y[iy], g9[iu]);               \
    gy[iy] = fmaf(gq, uu[iu], gy[iy]);              \
  }
    MACE_CG_L2_EXPAND(kL, MACE_X)
#undef MACE_X
#pragma unroll
    for (int p = G::P0; p < G::P0 + G::NPL; p++) re[p * C] = gr[p];
#pragma unroll
    for (int k = 1; k < G::NSH; k++) {  // Y[0] = 1 carries no gradient
      if (!((G::YM >> k) & 1)) continue;
      float v = gy[k];
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) atomicAdd(&gY[(size_t)e * kMaceMaxNsh + k], v);
    }
    float* gs = gu + (size_t)src * 9 * C + c;
#pragma unroll
    for (int k = 0; k < 9; k++)
      if ((G::UM >> k) & 1) atomicAdd(gs + k * C, g9[k]);
  }
}

// ============================================================================================
// readouts
// ============================================================================================
__global__ void k_mace_readout_lin(int n_own, int C, int ld, const float* __restrict__ h, const float* __restrict__ w,
                                   float* __restrict__ e_lin) {
  const int r = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (r >= n_own) return;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s = fmaf(h[(size_t)r * ld + c], w[c], s);
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) e_lin[r] += s;
}

// kWeighted: eps_i (E0, scale and shift included) times wgt[gid[r]] in the energy sum and atom_e (heat flux: cell mask or
// position seed); e_lin is weighted here, so k_mace_readout_lin and k_mace_zbl stay unweighted
template <bool kAtomic, bool kWeighted = false>
__global__ void k_mace_readout_final(int n_own, int C, int H, const float* __restrict__ h, const float* __restrict__ W1,
                                     const float* __restrict__ w2, const float* __restrict__ e_lin,
                                     const int* __restrict__ type, const double* __restrict__ E0, double scale,
                                     double shift, float* __restrict__ pre, double* __restrict__ energy,
                                     const int* __restrict__ gid, double* __restrict__ atom_e,
                                     const float* __restrict__ wgt) {
  const int r = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (r >= n_own) return;
  float e = 0.f;
  for (int j = 0; j < H; j++) {
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s = fmaf(h[(size_t)r * C + c], W1[(size_t)c * H + j], s);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) pre[(size_t)r * H + j] = s;
    e = fmaf(silu_f(s), w2[j], e);
  }
  if (lane == 0) {
    double eps = E0[type[r]] + scale * ((double)e_lin[r] + (double)e) + shift;
    if constexpr (kWeighted) eps *= (double)wgt[gid[r]];
    if constexpr (kAtomic) atom_e[gid[r]] = eps;
    atomicAdd(energy, eps);
  }
}

// kWeighted: row r's seed times wgt[gid[r]]
template <bool kWeighted = false>
__global__ void k_mace_readout_seed(int n_own, int C, int H, const float* __restrict__ pre, const float* __restrict__ W1,
                                    const float* __restrict__ w2, float scale, float* __restrict__ gh,
                                    const int* __restrict__ gid, const float* __restrict__ wgt) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)n_own * C) return;
  const int r = (int)(i / C), c = (int)(i % C);
  if constexpr (kWeighted) scale *= wgt[gid[r]];
  float s = 0.f;
  for (int j = 0; j < H; j++) s = fmaf(W1[(size_t)c * H + j] * w2[j], dsilu_f(pre[(size_t)r * H + j]), s);
  gh[i] = scale * s;
}

// adjoint of a linear readout; kWeighted: row r's term times wgt[gid[r]]
template <bool kWeighted = false>
__global__ void k_mace_add_row(int n_own, int C, int ld, const float* __restrict__ w, float scale,
                               float* __restrict__ gh, const int* __restrict__ gid, const float* __restrict__ wgt) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)n_own * C) return;
  if constexpr (kWeighted) scale *= wgt[gid[i / C]];
  gh[(i / C) * ld + i % C] += scale * w[i % C];
}

// ============================================================================================
// final geometry reverse: dE/dv from the adjoints of the radial basis (g_eb) and of the harmonics (gY)
// ============================================================================================
// kSpecies: the ZBL term (core.zbl) and the chain rule through the Agnesi transform (core.agnesi), switched at run time
// kWeighted (with kSpecies): the ZBL term times wgt[gid[dst]], the readout weight of the atom its pair energy belongs to;
// g_eb and gY carry the weights already (they are adjoints of the weighted readouts)
template <bool kAtomic, bool kSpecies, bool kWeighted = false>
__global__ void __launch_bounds__(256) k_mace_edge_final(int64_t E, int nsh, const int* __restrict__ e_src,
                                                         const int* __restrict__ e_dst, const float4* __restrict__ e_vec,
                                                         const int* __restrict__ gid, MaceRadial rp,
                                                         const float* __restrict__ g_eb, const float* __restrict__ gY,
                                                         float* __restrict__ forces, double* __restrict__ virial,
                                                         float* __restrict__ atom_vir, const int* __restrict__ type,
                                                         MaceCore core, const float* __restrict__ wgt) {
  static_assert(kSpecies || !kWeighted, "only the ZBL term needs the weight");
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  float vir[9];
#pragma unroll
  for (int k = 0; k < 9; k++) vir[k] = 0.f;
  int asrc = 0, adst = -1;
  if (e < E) {
    const float4 v = e_vec[e];
    const float d = v.w, rd = 1.f / d;
    const float x = v.x * rd, y = v.y * rd, z = v.z * rd;
    float f, df;
    poly_cut(d, rp, f, df);
    float xb = d, rxb = rd, dxb = 1.f;  // Bessel argument, its inverse and d(xb)/dd
    float4 eu, ev;
    if constexpr (kSpecies) {
      eu = core.elem[type[e_src[e]]], ev = core.elem[type[e_dst[e]]];
      if (core.agnesi) {
        agnesi(d, 0.5f * (eu.w + ev.w), core, xb, dxb);
        rxb = 1.f / xb;
      }
    }
    float gd = 0.f;
    for (int n = 0; n < rp.nb; n++) {
      float sn, cn;
      sincosf(rp.w[n] * xb, &sn, &cn);  // w_n d reaches num_bessel * pi: the accurate range reduction
      const float b = rp.pref * sn * rxb, db = rp.pref * (rp.w[n] * cn - sn * rxb) * rxb * dxb;
      gd = fmaf(g_eb[(size_t)e * rp.nbp + n], db * f + b * df, gd);
    }
    if constexpr (kSpecies) {
      if (core.zbl) {
        float V, dV;
        zbl(d, eu, ev, core, V, dV);
        float zs = core.zscale;
        if constexpr (kWeighted) zs *= wgt[gid[e_dst[e]]];
        gd = fmaf(zs, dV, gd);
      }
    }
    Dual Yd[kMaceMaxNsh];
    sh16<Dual>(Dual{x, 1.f, 0.f, 0.f}, Dual{y, 0.f, 1.f, 0.f}, Dual{z, 0.f, 0.f, 1.f}, Dual{1.f, 0.f, 0.f, 0.f}, nsh, Yd);
    float hx = 0.f, hy = 0.f, hz = 0.f;
    for (int m = 1; m < nsh; m++) {
      const float gy = gY[(size_t)e * kMaceMaxNsh + m];
      hx = fmaf(gy, Yd[m].x, hx), hy = fmaf(gy, Yd[m].y, hy), hz = fmaf(gy, Yd[m].z, hz);
    }
    const float3 g = unit_vector_chain(gd, make_float3(x, y, z), rd, make_float3(hx, hy, hz));
    const int gdst = gid[e_dst[e]], gsrc = gid[e_src[e]];
    scatter_edge(forces, gsrc, gdst, v, g, vir);
    if constexpr (kAtomic) asrc = gsrc, adst = gdst;
  }
  edge_virial_tail<kAtomic>(atom_vir, asrc, adst, vir, virial);
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------
void launch_mace_edge_geom(cudaStream_t st, int64_t E, const float4* e_vec, const MaceRadial& rp, int nsh, float* Y,
                           float* eb, const int* e_src, const int* e_dst, const int* type, const MaceCore& core) {
  with_flags(
      [&](auto kSpecies) {
        launch(k_mace_edge_geom<kSpecies>, cdiv(E, 256), 256, 0, st, E, e_vec, rp, nsh, Y, eb, e_src, e_dst, type, core);
      },
      core.agnesi != 0);
}
void launch_mace_zbl(cudaStream_t st, int n_own, const int* row_ptr, const int* e_src, const float4* e_vec,
                     const int* type, const MaceCore& core, float* e_lin) {
  launch(k_mace_zbl, cdiv(n_own, 128), 128, 0, st, n_own, row_ptr, e_src, e_vec, type, core, e_lin);
}
void launch_mace_embed(cudaStream_t st, int n, int C, const int* type, const float* W, float* h0) {
  launch(k_mace_embed, cdiv((int64_t)n * C, 256), 256, 0, st, n, C, type, W, h0);
}
void launch_mace_msg(cudaStream_t st, int n_own, int C, int L1, const int* row_ptr, const int* e_src, const float* R,
                     const float* Y, const float* u, float* A) {
  launch(k_mace_msg, cdiv((int64_t)n_own * C, 256), 256, 0, st, n_own, C, L1, row_ptr, e_src, R, Y, u, A);
}
void launch_mace_msg_bwd(cudaStream_t st, int n_own, int C, int L1, const int* row_ptr, const int* e_src, const float* R,
                         const float* Y, const float* u, const float* gA, float* gR, float* gY, float* gu) {
  launch(k_mace_msg_bwd, cdiv((int64_t)n_own * C, 256), 256, 0, st, n_own, C, L1, row_ptr, e_src, R, Y, u, gA, gR, gY,
         gu);
}
void launch_mace_elem_mix(cudaStream_t st, int n, int C, int L1, int nsh, const int* type, const float* W,
                          const float* in, float* out, bool accum) {
  if (n <= 0) return;
  B2M_REQUIRE(C <= 128, B2M_ERR_INVALID, "mace elem mix: C <= 128");
  launch(k_mace_elem_mix, n, C, 0, st, n, C, L1, nsh, type, W, in, out, accum ? 1 : 0);
}
void launch_mace_symc(cudaStream_t st, int n_own, int C, int nsh, int Ktot, const int* type, const float* A,
                      const MaceTerm* terms, int nterms, const float* w, float* B) {
  launch(k_mace_symc<false>, cdiv((int64_t)n_own * C, 128), 128, 0, st, n_own, C, nsh, Ktot, type, A, terms, nterms, w,
         nullptr, B);
}
void launch_mace_symc_bwd(cudaStream_t st, int n_own, int C, int nsh, int Ktot, const int* type, const float* A,
                          const MaceTerm* terms, int nterms, const float* w, const float* gB, float* gA) {
  launch(k_mace_symc<true>, cdiv((int64_t)n_own * C, 128), 128, 0, st, n_own, C, nsh, Ktot, type, A, terms, nterms, w,
         gB, gA);
}
void launch_mace_readout_lin(cudaStream_t st, int n_own, int C, int ld, const float* h, const float* w, float* e_lin) {
  launch(k_mace_readout_lin, cdiv((int64_t)n_own * 32, 256), 256, 0, st, n_own, C, ld, h, w, e_lin);
}
void launch_mace_readout_final(cudaStream_t st, int n_own, int C, int H, const float* h, const float* W1, const float* w2,
                               const float* e_lin, const int* type, const double* E0, double scale, double shift,
                               float* pre, double* energy, const int* gid, double* atom_e, const float* wgt) {
  with_flags(
      [&](auto kAtomic, auto kWeighted) {
        launch(k_mace_readout_final<kAtomic, kWeighted>, cdiv((int64_t)n_own * 32, 256), 256, 0, st, n_own, C, H, h, W1,
               w2, e_lin, type, E0, scale, shift, pre, energy, gid, atom_e, wgt);
      },
      atom_e != nullptr, wgt != nullptr);
}
void launch_mace_readout_seed(cudaStream_t st, int n_own, int C, int H, const float* pre, const float* W1,
                              const float* w2, float scale, float* gh, const int* gid, const float* wgt) {
  with_flags(
      [&](auto kWeighted) {
        launch(k_mace_readout_seed<kWeighted>, cdiv((int64_t)n_own * C, 256), 256, 0, st, n_own, C, H, pre, W1, w2,
               scale, gh, gid, wgt);
      },
      wgt != nullptr);
}
void launch_mace_add_row(cudaStream_t st, int n_own, int C, int ld, const float* w, float scale, float* gh,
                         const int* gid, const float* wgt) {
  with_flags(
      [&](auto kWeighted) {
        launch(k_mace_add_row<kWeighted>, cdiv((int64_t)n_own * C, 256), 256, 0, st, n_own, C, ld, w, scale, gh, gid,
               wgt);
      },
      wgt != nullptr);
}
void launch_mace_msg_eq(cudaStream_t st, int max_ell, int n_own, int C, const int* row_ptr, const int* e_src,
                        const float* R, const float* Y, const float* u, float* Am) {
  B2M_REQUIRE(max_ell >= 1 && max_ell <= 3, B2M_ERR_INVALID, "mace message with 0e+1o features: max_ell must be 1..3");
  const auto kern = max_ell == 1 ? k_mace_msg_eq<1> : max_ell == 2 ? k_mace_msg_eq<2> : k_mace_msg_eq<3>;
  launch(kern, cdiv((int64_t)n_own * C, 256), 256, 0, st, n_own, C, row_ptr, e_src, R, Y, u, Am);
}
void launch_mace_msg_eq_bwd(cudaStream_t st, int max_ell, int n_own, int C, const int* row_ptr, const int* e_src,
                            float* R, const float* Y, const float* u, const float* gAm, float* gY, float* gu) {
  B2M_REQUIRE(max_ell >= 1 && max_ell <= 3, B2M_ERR_INVALID, "mace message with 0e+1o features: max_ell must be 1..3");
  const auto kern = max_ell == 1 ? k_mace_msg_eq_bwd<1> : max_ell == 2 ? k_mace_msg_eq_bwd<2> : k_mace_msg_eq_bwd<3>;
  launch(kern, cdiv((int64_t)n_own * C, 256), 256, 0, st, n_own, C, row_ptr, e_src, R, Y, u, gAm, gY, gu);
}
void launch_mace_elem_mix_rows(cudaStream_t st, int n, int C, int ncomp, int ldi, int ldo, const int* type,
                               const float* W, const float* in, float* out, bool accum) {
  if (n <= 0) return;
  B2M_REQUIRE(C <= 128 && (ncomp == 1 || ncomp == 4 || ncomp == 9), B2M_ERR_INVALID,
              "mace elem mix: C <= 128, 1, 4 or 9 components");
  const auto kern = ncomp == 9 ? k_mace_elem_mix_rows<true> : k_mace_elem_mix_rows<false>;
  launch(kern, n, C, 0, st, n, C, ncomp, ldi, ldo, type, W, in, out, accum ? 1 : 0);
}
void launch_mace_symc_eq(cudaStream_t st, int n_own, int C, int nsh, int Ktot, const int* type, const float* A,
                         const MaceTerm* terms, int nterms, const float* w, float* B) {
  launch(k_mace_symc_eq<false, 4>, cdiv((int64_t)n_own * C, 128), 128, 0, st, n_own, C, nsh, Ktot, type, A, terms,
         nterms, w, nullptr, B);
}
void launch_mace_symc_eq_bwd(cudaStream_t st, int n_own, int C, int nsh, int Ktot, const int* type, const float* A,
                             const MaceTerm* terms, int nterms, const float* w, const float* gB, float* gA) {
  launch(k_mace_symc_eq<true, 4>, cdiv((int64_t)n_own * C, 128), 128, 0, st, n_own, C, nsh, Ktot, type, A, terms,
         nterms, w, gB, gA);
}
void launch_mace_symc_l2(cudaStream_t st, int n_own, int C, int nsh, int Ktot, const int* type, const float* A,
                         const MaceTerm* terms, int nterms, const float* w, float* B) {
  launch(k_mace_symc_eq<false, 9>, cdiv((int64_t)n_own * C, 128), 128, 0, st, n_own, C, nsh, Ktot, type, A, terms,
         nterms, w, nullptr, B);
}
void launch_mace_symc_l2_bwd(cudaStream_t st, int n_own, int C, int nsh, int Ktot, const int* type, const float* A,
                             const MaceTerm* terms, int nterms, const float* w, const float* gB, float* gA) {
  launch(k_mace_symc_eq<true, 9>, cdiv((int64_t)n_own * C, 128), 128, 0, st, n_own, C, nsh, Ktot, type, A, terms,
         nterms, w, gB, gA);
}
// one launch per output l of the 0e+1o+2e message (kernel<kL, 0>, .., kernel<kL, kL>)
template <int kL, bool kBwd, int... kLo>
static void msg_l2_groups(std::integer_sequence<int, kLo...>, cudaStream_t st, int n_own, int C, const int* row_ptr,
                          const int* e_src, float* R, const float* Y, const float* u, float* Am, const float* gAm,
                          float* gY, float* gu) {
  const int grid = cdiv((int64_t)n_own * C, 256);
  if constexpr (kBwd)
    (launch(k_mace_msg_l2_bwd<kL, kLo>, grid, 256, 0, st, n_own, C, row_ptr, e_src, R, Y, u, gAm, gY, gu), ...);
  else
    (launch(k_mace_msg_l2<kL, kLo>, grid, 256, 0, st, n_own, C, row_ptr, e_src, R, Y, u, Am), ...);
}
void launch_mace_msg_l2(cudaStream_t st, int max_ell, int n_own, int C, const int* row_ptr, const int* e_src,
                        const float* R, const float* Y, const float* u, float* Am) {
  B2M_REQUIRE(max_ell == 2 || max_ell == 3, B2M_ERR_INVALID,
              "mace message with 0e+1o+2e features: max_ell must be 2 or 3");
  float* Rm = const_cast<float*>(R);  // read only in the forward
  if (max_ell == 2)
    msg_l2_groups<2, false>(std::make_integer_sequence<int, 3>{}, st, n_own, C, row_ptr, e_src, Rm, Y, u, Am, nullptr,
                            nullptr, nullptr);
  else
    msg_l2_groups<3, false>(std::make_integer_sequence<int, 4>{}, st, n_own, C, row_ptr, e_src, Rm, Y, u, Am, nullptr,
                            nullptr, nullptr);
}
void launch_mace_msg_l2_bwd(cudaStream_t st, int max_ell, int n_own, int C, const int* row_ptr, const int* e_src,
                            float* R, const float* Y, const float* u, const float* gAm, float* gY, float* gu) {
  B2M_REQUIRE(max_ell == 2 || max_ell == 3, B2M_ERR_INVALID,
              "mace message with 0e+1o+2e features: max_ell must be 2 or 3");
  if (max_ell == 2)
    msg_l2_groups<2, true>(std::make_integer_sequence<int, 3>{}, st, n_own, C, row_ptr, e_src, R, Y, u, nullptr, gAm, gY,
                           gu);
  else
    msg_l2_groups<3, true>(std::make_integer_sequence<int, 4>{}, st, n_own, C, row_ptr, e_src, R, Y, u, nullptr, gAm, gY,
                           gu);
}
// kSpecies with the pair term or the Agnesi transform; kWeighted with the pair term and readout weights (without the
// pair term the weights are all in g_eb and gY)
void launch_mace_edge_final(cudaStream_t st, int64_t E, int nsh, const int* e_src, const int* e_dst, const float4* e_vec,
                            const int* gid, const int* type, const MaceRadial& rp, const MaceCore& core,
                            const float* g_eb, const float* gY, float* forces, double* virial, float* atom_vir,
                            const float* wgt) {
  with_flags(
      [&](auto kAtomic, auto kSpecies, auto kWeighted) {
        launch(k_mace_edge_final<kAtomic, kSpecies || kWeighted, kWeighted>, cdiv(E, 256), 256, 0, st, E, nsh, e_src,
               e_dst, e_vec, gid, rp, g_eb, gY, forces, virial, atom_vir, type, core, wgt);
      },
      atom_vir != nullptr, core.zbl || core.agnesi, wgt != nullptr && core.zbl);
}

}  // namespace b2m
