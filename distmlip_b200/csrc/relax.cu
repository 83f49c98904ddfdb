// relax.cu -- batched FIRE relaxation with the Frechet cell filter (DESIGN.md §13), sm_90a.  The optimizer of ASE's
// FIRE + FrechetCellFilter, one independent copy per structure, all in f64: the per-structure kernel forms the
// generalised forces and FIRE's scalars from one reduction pass and takes the cell rows' step, the per-row kernel takes
// the atoms' step, the emit kernel writes the next graph build's input.
#include <math.h>

#include "relax.cuh"

namespace b2m {

constexpr int kRelaxThreads = 256;

// C = A B, M x M row-major
template <int M>
__device__ void mat_mul(const double* A, const double* B, double* C) {
  for (int i = 0; i < M; i++)
    for (int j = 0; j < M; j++) {
      double s = 0;
      for (int k = 0; k < M; k++) s += A[i * M + k] * B[k * M + j];
      C[i * M + j] = s;
    }
}

// expm(A), M x M: scaling to a 1-norm <= 1/8, a degree-16 Taylor polynomial (truncation < 1e-30 relative), squaring
template <int M>
__device__ void expm_dev(const double* A, double* E) {
  double nrm = 0;
  for (int j = 0; j < M; j++) {
    double c = 0;
    for (int i = 0; i < M; i++) c += fabs(A[i * M + j]);
    nrm = fmax(nrm, c);
  }
  int sq = 0;
  while (nrm > 0.125 && sq < 1000) nrm *= 0.5, sq++;
  const double sc = ldexp(1.0, -sq);
  double B[M * M], T[M * M];
  for (int i = 0; i < M * M; i++) B[i] = A[i] * sc, E[i] = (i % (M + 1) == 0) ? 1.0 : 0.0;
  for (int k = 16; k >= 1; k--) {  // Horner: E <- I + B E / k
    mat_mul<M>(B, E, T);
    for (int i = 0; i < M * M; i++) E[i] = T[i] / k + ((i % (M + 1) == 0) ? 1.0 : 0.0);
  }
  for (int q = 0; q < sq; q++) {
    mat_mul<M>(E, E, T);
    for (int i = 0; i < M * M; i++) E[i] = T[i];
  }
}

// lattice = cell0 F^T (rows r F^T like the positions)
__device__ void lattice_of(const RelaxStruct& r, double* lat) {
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++)
      lat[3 * i + j] = r.cell0[3 * i] * r.F[3 * j] + r.cell0[3 * i + 1] * r.F[3 * j + 1] + r.cell0[3 * i + 2] * r.F[3 * j + 2];
}

// g = f F (row vector times F)
__device__ __forceinline__ void gen_force(const double* F, double f0, double f1, double f2, double* g) {
  for (int j = 0; j < 3; j++) g[j] = f0 * F[j] + f1 * F[3 + j] + f2 * F[6 + j];
}

__global__ void k_relax_init(int S, const double* __restrict__ lat9, double dt0, double a0, RelaxStruct* __restrict__ rs,
                             double* __restrict__ stat) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  RelaxStruct r;
  for (int k = 0; k < 9; k++) {
    r.cell0[k] = lat9[9 * s + k];
    r.X[k] = r.vc[k] = r.Fold[k] = 0.0;
    r.F[k] = (k % 4 == 0) ? 1.0 : 0.0;
    stat[kRelaxStat * s + 3 + k] = r.cell0[k];
  }
  r.dt = dt0, r.a = a0, r.nsteps = 0;
  r.alpha = r.gamma = r.dtv = r.normdr = 0.0;
  r.move = r.scaled = 0;
  stat[kRelaxStat * s] = 0.0;
  stat[kRelaxStat * s + 1] = stat[kRelaxStat * s + 2] = 0.0;
  rs[s] = r;
}

__global__ void __launch_bounds__(kRelaxThreads) k_relax_emit(const int64_t* __restrict__ act,
                                                              const int64_t* __restrict__ in_off,
                                                              const int64_t* __restrict__ out_off,
                                                              const RelaxStruct* __restrict__ rs,
                                                              const double* __restrict__ r0,
                                                              const int* __restrict__ species_in,
                                                              double* __restrict__ cart_out, int* __restrict__ species_out) {
  const int64_t s = act[blockIdx.x], b = in_off[s], n = in_off[s + 1] - b, o = out_off[blockIdx.x];
  double F[9];
  for (int k = 0; k < 9; k++) F[k] = rs[s].F[k];
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const double* r = r0 + 3 * (b + i);
    for (int j = 0; j < 3; j++) cart_out[3 * (o + i) + j] = r[0] * F[3 * j] + r[1] * F[3 * j + 1] + r[2] * F[3 * j + 2];
    species_out[o + i] = species_in[b + i];
  }
}

// sums of the first three, max of the fourth, over the block; the result in thread 0
__device__ void block_reduce4(double* x) {
  __shared__ double sh[kRelaxThreads / 32][4];
  for (int o = 16; o > 0; o >>= 1) {
    for (int k = 0; k < 3; k++) x[k] += __shfl_down_sync(0xffffffffu, x[k], o);
    x[3] = fmax(x[3], __shfl_down_sync(0xffffffffu, x[3], o));
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0)
    for (int k = 0; k < 4; k++) sh[w][k] = x[k];
  __syncthreads();
  if (threadIdx.x == 0)
    for (int q = 1; q < kRelaxThreads / 32; q++) {
      for (int k = 0; k < 3; k++) x[k] += sh[q][k];
      x[3] = fmax(x[3], sh[q][3]);
    }
}

__device__ void take_step(const RelaxConst& c, int it, const double* acc, const double* gc, double cf, const double* F,
                          RelaxStruct& r, double* lat);

// block sl: structure s = act[sl], its rows b_off[sl] .. b_off[sl + 1] - 1 of the batch just evaluated
__global__ void __launch_bounds__(kRelaxThreads) k_relax_struct(int it, RelaxConst c, const int64_t* __restrict__ act,
                                                                const int64_t* __restrict__ in_off,
                                                                const int64_t* __restrict__ b_off,
                                                                const float* __restrict__ forces,
                                                                const double* __restrict__ bsum, double data_mean,
                                                                const double* __restrict__ v, RelaxStruct* __restrict__ rs,
                                                                double* __restrict__ stat, float* __restrict__ res_f,
                                                                double* __restrict__ res_e, double* __restrict__ res_s,
                                                                double* __restrict__ trace, int64_t trace_pitch) {
  const int sl = blockIdx.x;
  const int64_t s = act[sl], b = b_off[sl], n = b_off[sl + 1] - b, j0 = in_off[s];
  double F[9];
  for (int k = 0; k < 9; k++) F[k] = rs[s].F[k];
  // P = f.v, |f|^2, |v|^2, max row |f|^2 over the atom rows
  double acc[4] = {0, 0, 0, 0};
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const float* fi = forces + 3 * (b + i);
    const float f0 = fi[0], f1 = fi[1], f2 = fi[2];
    float* ro = res_f + 3 * (j0 + i);
    ro[0] = f0, ro[1] = f1, ro[2] = f2;
    double g[3];
    gen_force(F, f0, f1, f2, g);
    const double* vi = v + 3 * (j0 + i);
    const double g2 = g[0] * g[0] + g[1] * g[1] + g[2] * g[2];
    acc[0] += g[0] * vi[0] + g[1] * vi[1] + g[2] * vi[2];
    acc[1] += g2;
    acc[2] += vi[0] * vi[0] + vi[1] * vi[1] + vi[2] * vi[2];
    acc[3] = fmax(acc[3], g2);
  }
  block_reduce4(acc);
  if (threadIdx.x != 0) return;
  RelaxStruct& r = rs[s];
  const double* sum = bsum + 10 * sl;
  double lat[9];
  lattice_of(r, lat);
  const double V = fabs(lat[0] * (lat[4] * lat[8] - lat[5] * lat[7]) - lat[1] * (lat[3] * lat[8] - lat[5] * lat[6]) +
                        lat[2] * (lat[3] * lat[7] - lat[4] * lat[6]));
  const double energy = sum[0] + data_mean;
  res_e[s] = energy;
  for (int k = 0; k < 9; k++) res_s[9 * s + k] = sum[1 + k] / V * 160.21766208;
  if (trace) trace[trace_pitch * s + it] = energy;
  double gc[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};  // generalised force of the cell rows
  if (c.relax_cell) {
    const double cf = (double)n;
    // M = -(k sym(W) + p V I), G = M F^-T
    double M[9], Fi[9], G[9];
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++)
        M[3 * i + j] = -(c.k * 0.5 * (sum[1 + 3 * i + j] + sum[1 + 3 * j + i]) + (i == j ? c.p * V : 0.0));
    const double det = F[0] * (F[4] * F[8] - F[5] * F[7]) - F[1] * (F[3] * F[8] - F[5] * F[6]) +
                       F[2] * (F[3] * F[7] - F[4] * F[6]);
    Fi[0] = (F[4] * F[8] - F[5] * F[7]) / det, Fi[1] = (F[2] * F[7] - F[1] * F[8]) / det;
    Fi[2] = (F[1] * F[5] - F[2] * F[4]) / det, Fi[3] = (F[5] * F[6] - F[3] * F[8]) / det;
    Fi[4] = (F[0] * F[8] - F[2] * F[6]) / det, Fi[5] = (F[2] * F[3] - F[0] * F[5]) / det;
    Fi[6] = (F[3] * F[7] - F[4] * F[6]) / det, Fi[7] = (F[1] * F[6] - F[0] * F[7]) / det;
    Fi[8] = (F[0] * F[4] - F[1] * F[3]) / det;
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) G[3 * i + j] = M[3 * i] * Fi[3 * j] + M[3 * i + 1] * Fi[3 * j + 1] + M[3 * i + 2] * Fi[3 * j + 2];
    // (1/c) L_exp(A^T)[G], A = X / c: the upper-right block of expm([[A^T, G / gs], [0, A^T]]) times gs.  The block is
    // linear in G; scaling G to a max entry of 1 keeps it out of the norm that sets the number of squarings, whose
    // round-off would otherwise grow with |G| (virials of 1e2 - 1e3 eV)
    double gs = 0.0;
    for (int k = 0; k < 9; k++) gs = fmax(gs, fabs(G[k]));
    const double gi = gs > 0.0 ? 1.0 / gs : 0.0;
    double Y[36], E6[36];
    for (int i = 0; i < 36; i++) Y[i] = 0.0;
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) {
        Y[6 * i + j] = Y[6 * (i + 3) + j + 3] = r.X[3 * j + i] / cf;
        Y[6 * i + j + 3] = G[3 * i + j] * gi;
      }
    expm_dev<6>(Y, E6);
    for (int i = 0; i < 3; i++) {
      double g2 = 0;
      for (int j = 0; j < 3; j++) {
        const double g = E6[6 * i + j + 3] * gs / cf;
        gc[3 * i + j] = g;
        g2 += g * g;
        acc[0] += g * r.vc[3 * i + j];
        acc[2] += r.vc[3 * i + j] * r.vc[3 * i + j];
      }
      acc[1] += g2;
      acc[3] = fmax(acc[3], g2);
    }
  }
  double* so = stat + kRelaxStat * s;
  const int flag = acc[3] < c.fmax2 ? 1 : (it >= c.steps ? 2 : 0);
  so[0] = flag, so[1] = energy, so[2] = sqrt(acc[3]);
  r.move = flag == 0;
  if (r.move) take_step(c, it, acc, gc, (double)n, F, r, lat);
  for (int k = 0; k < 9; k++) so[3 + k] = lat[k];
}

// FIRE (ase.optimize.FIRE.step) of structure r from the reductions acc; the cell rows' step, and lat the next lattice
__device__ void take_step(const RelaxConst& c, int it, const double* acc, const double* gc, double cf, const double* F,
                          RelaxStruct& r, double* lat) {
  // the first step has v = 0 and skips the mixing
  double alpha = 0.0, gamma = 0.0;
  const double P = acc[0], ff = acc[1], vv = acc[2];
  if (it > 0) {
    if (P > 0.0) {
      alpha = 1.0 - r.a;
      gamma = r.a * sqrt(vv) / sqrt(ff);
      if (r.nsteps > c.Nmin) {
        r.dt = fmin(r.dt * c.finc, c.dtmax);
        r.a *= c.fa;
      }
      r.nsteps++;
    } else {
      r.a = c.astart;
      r.dt *= c.fdec;
      r.nsteps = 0;
    }
  }
  // |v_new|^2 for v_new = alpha v + (gamma + dt) f, from the three reductions
  const double beta = gamma + r.dt;
  const double vn2 = fmax(alpha * alpha * vv + 2.0 * alpha * beta * P + beta * beta * ff, 0.0);
  r.alpha = alpha, r.gamma = gamma, r.dtv = r.dt;
  r.normdr = r.dt * sqrt(vn2);
  r.scaled = r.normdr > c.maxstep;
  for (int k = 0; k < 9; k++) r.Fold[k] = F[k];
  if (c.relax_cell) {
    double Xc[9];
    for (int k = 0; k < 9; k++) {
      double vk = alpha * r.vc[k] + gamma * gc[k];
      vk += r.dt * gc[k];
      r.vc[k] = vk;
      double dr = r.dt * vk;
      if (r.scaled) dr = c.maxstep * dr / r.normdr;
      r.X[k] += dr;
      Xc[k] = r.X[k] / cf;
    }
    expm_dev<3>(Xc, r.F);
    lattice_of(r, lat);
  }
}

__global__ void k_relax_rows(int64_t N, double maxstep, const int64_t* __restrict__ act,
                             const int64_t* __restrict__ in_off, const int64_t* __restrict__ b_off,
                             const int* __restrict__ b_sid, const float* __restrict__ forces,
                             const RelaxStruct* __restrict__ rs, double* __restrict__ v, double* __restrict__ r0) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int sl = b_sid[i];
  const int64_t s = act[sl];
  const RelaxStruct& r = rs[s];
  if (!r.move) return;
  const int64_t j = in_off[s] + i - b_off[sl];
  double g[3];
  gen_force(r.Fold, forces[3 * i], forces[3 * i + 1], forces[3 * i + 2], g);
  for (int k = 0; k < 3; k++) {
    double vk = r.alpha * v[3 * j + k] + r.gamma * g[k];
    vk += r.dtv * g[k];
    v[3 * j + k] = vk;
    double dr = r.dtv * vk;
    if (r.scaled) dr = maxstep * dr / r.normdr;
    r0[3 * j + k] += dr;
  }
}

void launch_relax_init(cudaStream_t st, int S, const double* lat9, double dt0, double a0, RelaxStruct* rs,
                       double* stat) {
  launch(k_relax_init, cdiv(S, 128), 128, 0, st, S, lat9, dt0, a0, rs, stat);
}

void launch_relax_emit(cudaStream_t st, int Sa, const int64_t* act, const int64_t* in_off, const int64_t* out_off,
                       const RelaxStruct* rs, const double* r0, const int* species_in, double* cart_out,
                       int* species_out) {
  launch(k_relax_emit, Sa, kRelaxThreads, 0, st, act, in_off, out_off, rs, r0, species_in, cart_out, species_out);
}

void launch_relax_struct(cudaStream_t st, int Sa, int it, const RelaxConst& c, const int64_t* act,
                         const int64_t* in_off, const int64_t* b_off, const float* forces, const double* bsum,
                         double data_mean, const double* v, RelaxStruct* rs, double* stat, float* res_f,
                         double* res_e, double* res_s, double* trace, int64_t trace_pitch) {
  launch(k_relax_struct, Sa, kRelaxThreads, 0, st, it, c, act, in_off, b_off, forces, bsum, data_mean, v, rs, stat,
         res_f, res_e, res_s, trace, trace_pitch);
}

void launch_relax_rows(cudaStream_t st, int64_t N, const RelaxConst& c, const int64_t* act, const int64_t* in_off,
                       const int64_t* b_off, const int* b_sid, const float* forces, const RelaxStruct* rs, double* v,
                       double* r0) {
  launch(k_relax_rows, cdiv(N, 256), 256, 0, st, N, c.maxstep, act, in_off, b_off, b_sid, forces, rs, v, r0);
}

}  // namespace b2m
