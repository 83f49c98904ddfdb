// kernels_mace.cu -- MACE with hidden features C x 0e or C x 0e + C x 1o on the same partitioned CSR graph as the
// CHGNet and TensorNet paths.  Arithmetic as oracle/mace_ref.py and, for 0e+1o features, tests/mace_eq_ref.py state it
// (the conventions are written down there once), and the ZBL pair term and Agnesi transform as tests/mace_zbl_ref.py
// states them; engine_mace.inl runs these kernels stage by stage.
//
// First generation: the node- and edge-level products (radial MLP, linear_up, the per-l mixes, the product linear) run
// on the wgmma row GEMM of the other paths (kernels_wg.cu, engine.cu tc_mm); the element-dependent mixes
// (skip_tp) read the element's C x C block per atom; the symmetric contraction is one thread per (atom, channel) that
// walks the nonzero terms of U, which every channel shares.  Aggregations walk the CSR-by-destination rows (no atomics
// in the forward); the reverse scatters to sources with atomics.
#include "final_tail.cuh"
#include "mace_cg.cuh"
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
  constexpr int NP = mace_npaths(kL), NS = mace_nslots(kL), NSH = (kL + 1) * (kL + 1);
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
    const int np = mace_np_l(kL, l);
    float* blk = Am + (size_t)mace_slot_base(kL, l) * n_own * C;
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
  constexpr int NP = mace_npaths(kL), NS = mace_nslots(kL), NSH = (kL + 1) * (kL + 1);
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)n_own * C) return;  // n_own * C is a multiple of 32: whole warps leave together
  const int t = (int)(i / C), c = (int)(i % C), lane = threadIdx.x & 31;
  float ga[NS];
  {
    int s = 0;
#pragma unroll
    for (int l = 0; l <= kL; l++) {
      const int np = mace_np_l(kL, l);
      const float* blk = gAm + (size_t)mace_slot_base(kL, l) * n_own * C;
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

// out[i][m][:] (+)= in[i][m][:] @ W[type[i]][l(m)], m < ncomp (1 or 4), rows of pitch ldi / ldo: one block of C threads
// per row, each weight element read once per row and applied to the components of its l
__global__ void k_mace_elem_mix_rows(int n, int C, int ncomp, int ldi, int ldo, const int* __restrict__ type,
                                     const float* __restrict__ W, const float* __restrict__ in, float* __restrict__ out,
                                     int accum) {
  __shared__ float x[4][128];
  const int i = blockIdx.x, c2 = threadIdx.x;
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

// symmetric contraction with a 1o output: as k_mace_symc, with the term's output slot o (MaceTerm) selecting one of four
// accumulators (forward) or upstream adjoints (reverse); B / gB [4][n_own][C]
template <bool kBwd>
__global__ void __launch_bounds__(128) k_mace_symc_eq(int n_own, int C, int nsh, int Ktot, const int* __restrict__ type,
                                                      const float* __restrict__ A, const MaceTerm* __restrict__ terms,
                                                      int nterms, const float* __restrict__ w,
                                                      const float* __restrict__ gB, float* __restrict__ out) {
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
  float g[4] = {0.f, 0.f, 0.f, 0.f};
  if constexpr (kBwd) {
#pragma unroll
    for (int o = 0; o < 4; o++) g[o] = gB[o * plane + i];
  }
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int j = 0; j < nterms; j++) {
    const MaceTerm tm = terms[j];
    const int nu = (tm.idx >> 24) & 3, o = (tm.idx >> 28) & 3;
    const int i1 = tm.idx & 255, i2 = (tm.idx >> 8) & 255, i3 = (tm.idx >> 16) & 255;
    const float cw = tm.coef * wz[(size_t)tm.kg * C];
    const float a1 = a[i1][tid], a2 = nu >= 2 ? a[i2][tid] : 1.f, a3 = nu >= 3 ? a[i3][tid] : 1.f;
    if constexpr (!kBwd) {
      const float v = cw * (a1 * a2 * a3);  // the same o for the whole warp: the selects do not diverge
      acc[0] += o == 0 ? v : 0.f, acc[1] += o == 1 ? v : 0.f, acc[2] += o == 2 ? v : 0.f, acc[3] += o == 3 ? v : 0.f;
    } else {
      const float s = cw * (o == 0 ? g[0] : o == 1 ? g[1] : o == 2 ? g[2] : g[3]);
      ga[i1][tid] += s * a2 * a3;
      if (nu >= 2) ga[i2][tid] += s * a1 * a3;
      if (nu >= 3) ga[i3][tid] += s * a1 * a2;
    }
  }
  if constexpr (!kBwd) {
#pragma unroll
    for (int o = 0; o < 4; o++) out[o * plane + i] = acc[o];
  } else {
#pragma unroll
    for (int k = 0; k < kMaceMaxNsh; k++)
      if (k < nsh) out[k * plane + i] = ga[k][tid];
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
  B2M_REQUIRE(C <= 128 && (ncomp == 1 || ncomp == 4), B2M_ERR_INVALID, "mace elem mix: C <= 128, 1 or 4 components");
  launch(k_mace_elem_mix_rows, n, C, 0, st, n, C, ncomp, ldi, ldo, type, W, in, out, accum ? 1 : 0);
}
void launch_mace_symc_eq(cudaStream_t st, int n_own, int C, int nsh, int Ktot, const int* type, const float* A,
                         const MaceTerm* terms, int nterms, const float* w, float* B) {
  launch(k_mace_symc_eq<false>, cdiv((int64_t)n_own * C, 128), 128, 0, st, n_own, C, nsh, Ktot, type, A, terms, nterms,
         w, nullptr, B);
}
void launch_mace_symc_eq_bwd(cudaStream_t st, int n_own, int C, int nsh, int Ktot, const int* type, const float* A,
                             const MaceTerm* terms, int nterms, const float* w, const float* gB, float* gA) {
  launch(k_mace_symc_eq<true>, cdiv((int64_t)n_own * C, 128), 128, 0, st, n_own, C, nsh, Ktot, type, A, terms, nterms,
         w, gB, gA);
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
