// atomic_virial.cuh -- per-atom virial accumulation of the final geometry kernels (k_edge_final, k_halo_bond_final,
// k_tn_edge_final, each in its kAtomic = true instantiation).  See DESIGN.md "Per-atom energies and virials".
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

}  // namespace b2m
