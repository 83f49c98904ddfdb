// final_tail.cuh -- what the final kernels of every model share: the force and virial epilogue of the final geometry
// kernels (k_edge_final, k_halo_bond_final, k_tn_edge_final, k_mace_edge_final) and the energy tail of the CHGNet and
// TensorNet readouts (k_rowdot, k_tn_readout_final).  See DESIGN.md "Per-atom energies and virials".
//
// The per-atom virial array of a partition is [N][kVirPitch] f32 indexed by global atom id, beside `forces`: row i holds
// w_i = 1/2 sum_{e : i in e} v_e (x) g_e row-major in its first 9 floats; the pitch of 12 keeps rows 16-byte aligned so
// that one endpoint of an edge costs two red.global.add.v4.f32 and one scalar red.
#pragma once
#include "common.cuh"

namespace b2m {

constexpr int kVirPitch = 12;

__device__ __forceinline__ void red_add_f32x4(float* p, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// row `atom` of the per-atom virial array += w
__device__ __forceinline__ void red_add_virial(float* __restrict__ atom_vir, int atom, const float (&w)[9]) {
  float* p = atom_vir + (size_t)atom * kVirPitch;
  red_add_f32x4(p, w[0], w[1], w[2], w[3]);
  red_add_f32x4(p + 4, w[4], w[5], w[6], w[7]);
  atomicAdd(p + 8, w[8]);
}

// One edge per lane, edges of the warp in CSR order (equal destinations are adjacent).  w = 1/2 v (x) g goes to the
// source by one red per edge; the destination halves are summed over each run of equal destinations with a segmented
// inclusive scan (warp shuffles) and added once, by the run's last lane.  Every lane of the warp calls this; lanes
// without an edge pass gdst = -1.
__device__ __forceinline__ void red_add_edge_virial(float* __restrict__ atom_vir, int gsrc, int gdst, float (&w)[9]) {
  const int lane = threadIdx.x & 31;
  if (gdst >= 0) red_add_virial(atom_vir, gsrc, w);
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const bool take = __shfl_up_sync(0xffffffffu, gdst, o) == gdst && lane >= o;
#pragma unroll
    for (int k = 0; k < 9; k++) {
      const float x = __shfl_up_sync(0xffffffffu, w[k], o);
      if (take) w[k] += x;
    }
  }
  const int next = __shfl_down_sync(0xffffffffu, gdst, 1);
  if (gdst >= 0 && (lane == 31 || next != gdst)) red_add_virial(atom_vir, gdst, w);
}

// out[k] += the sum of v[k] over the block, k < K: warp sums in T, then the warps' sums in double by thread k, one
// atomic each.  Every thread of the block calls this; at most 256 threads.
template <class T, int K>
__device__ __forceinline__ void block_sum_add(const T (&v)[K], double* __restrict__ out) {
  __shared__ T red[K][8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; k++) {
    T x = v[k];
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if (lane == 0) red[k][warp] = x;
  }
  __syncthreads();
  if (threadIdx.x < K) {
    double s = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += (double)red[threadIdx.x][w];
    atomicAdd(&out[threadIdx.x], s);
  }
}

// g = dE/dv of an edge from dE/dd = gd and the adjoint h of the unit vector u = v / d (rd = 1 / d):
// g = gd u + (h - (h . u) u) / d
__device__ __forceinline__ float3 unit_vector_chain(float gd, float3 u, float rd, float3 h) {
  const float pr = h.x * u.x + h.y * u.y + h.z * u.z;
  return make_float3(gd * u.x + (h.x - pr * u.x) * rd, gd * u.y + (h.y - pr * u.y) * rd,
                     gd * u.z + (h.z - pr * u.z) * rd);
}

// vec = x_dst + off.L - x_src :  dE/dx_dst += g, dE/dx_src -= g ; F = -dE/dx   (pes.py:122-124)
// vir = v (x) g, the edge's part of strain_bar[a][b] = sum vec[a] g[b]   (pes.py:140-145)
__device__ __forceinline__ void scatter_edge(float* __restrict__ forces, int gsrc, int gdst, float4 v, float3 g,
                                             float (&vir)[9]) {
  atomicAdd(&forces[(size_t)gdst * 3], -g.x);
  atomicAdd(&forces[(size_t)gdst * 3 + 1], -g.y);
  atomicAdd(&forces[(size_t)gdst * 3 + 2], -g.z);
  atomicAdd(&forces[(size_t)gsrc * 3], g.x);
  atomicAdd(&forces[(size_t)gsrc * 3 + 1], g.y);
  atomicAdd(&forces[(size_t)gsrc * 3 + 2], g.z);
  vir[0] = v.x * g.x, vir[1] = v.x * g.y, vir[2] = v.x * g.z;
  vir[3] = v.y * g.x, vir[4] = v.y * g.y, vir[5] = v.y * g.z;
  vir[6] = v.z * g.x, vir[7] = v.z * g.y, vir[8] = v.z * g.z;
}

// End of a final kernel over the edges in CSR order, called by every thread: kAtomic, 1/2 vir into both endpoints'
// per-atom virial rows (adst = -1 for a thread without an edge); then the block's vir into virial[9].
template <bool kAtomic>
__device__ __forceinline__ void edge_virial_tail(float* __restrict__ atom_vir, int asrc, int adst,
                                                 const float (&vir)[9], double* __restrict__ virial) {
  if constexpr (kAtomic) {
    float w[9];
#pragma unroll
    for (int k = 0; k < 9; k++) w[k] = 0.5f * vir[k];
    red_add_edge_virial(atom_vir, asrc, adst, w);
  }
  block_sum_add(vir, virial);
}

// Energy of readout row `row` with output v: scale * v + eref[type[row]] (no eref: none).  kWeighted: times
// wgt[gid[row]] (heat flux: cell mask or position seed).  kAtomic: also the row's per-atom energy,
// atom_e[gid[row]] = that energy + mean_per_atom (weighted alike).
template <bool kAtomic, bool kWeighted>
__device__ __forceinline__ double readout_energy(int row, float v, float scale, const int* __restrict__ type,
                                                 const double* __restrict__ eref, const int* __restrict__ gid,
                                                 double* __restrict__ atom_e, double mean_per_atom,
                                                 const float* __restrict__ wgt) {
  double ev = (double)scale * (double)v;
  if (eref) ev += eref[type[row]];
  if constexpr (kWeighted) {
    const double wt = (double)wgt[gid[row]];
    ev *= wt;
    mean_per_atom *= wt;
  }
  if constexpr (kAtomic) atom_e[gid[row]] = ev + mean_per_atom;
  return ev;
}

}  // namespace b2m
