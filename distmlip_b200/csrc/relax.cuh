// relax.cuh -- batched FIRE relaxation with the Frechet cell filter (DESIGN.md §13): per-structure state and the
// launchers of csrc/relax.cu.  All state is f64; structures are indexed in the caller's order (s), the rows of a
// structure's atoms by in_off[s] .. in_off[s + 1] - 1, and the active subset of a step by its batch index (sl).
#pragma once
#include "common.cuh"

namespace b2m {

// the constants of one relaxation (b2m_relax_params, with fmax squared and stress_weight * 160.21766208 as k)
struct RelaxConst {
  double fmax2, maxstep, dtmax, Nmin, finc, fdec, astart, fa;
  double k, p;  // the strain derivative's weight in the cell force, scalar pressure (eV/A^3)
  int relax_cell, steps;
};

// one structure's optimizer state, and the step the per-structure kernel decided for the per-row kernel
struct RelaxStruct {
  double cell0[9];  // input lattice (rows)
  double X[9];      // c logm(F), c = natoms; F = expm(X / c) and the lattice is cell0 F^T
  double vc[9];     // FIRE velocity of the three cell rows
  double F[9];      // expm(X / c) of the current geometry
  double dt, a;
  int nsteps;       // FIRE's Nsteps (uphill resets it)
  // the step: v <- alpha v + gamma f; v <- v + dt f; dr = dt v, times maxstep / normdr when scaled
  double Fold[9];   // F the forces were generalised with
  double alpha, gamma, dtv, normdr;
  int move, scaled;
};

// per-structure status of a step, copied to the host: flag (0 running, 1 converged, 2 out of steps), energy (eV),
// max row force (eV/A, generalised), lattice [9] of the next geometry
constexpr int kRelaxStat = 12;

// state of every structure: cell0 from lat9 [S][9], X = vc = 0, F = I, dt / a from the parameters; stat's lattices
void launch_relax_init(cudaStream_t st, int S, const double* lat9, double dt0, double a0, RelaxStruct* rs,
                       double* stat);
// next build's input: positions r0 F^T and species of the active structures act[0..Sa-1], contiguous from out_off[sl]
void launch_relax_emit(cudaStream_t st, int Sa, const int64_t* act, const int64_t* in_off, const int64_t* out_off,
                       const RelaxStruct* rs, const double* r0, const int* species_in, double* cart_out,
                       int* species_out);
// evaluation `it` of the active structures: results (energy, forces f32, stress GPa) in input order, energy trace (if
// not null), generalised forces, convergence, FIRE scalars, the cell rows' step and stat; bsum [Sa][10] from
// k_batch_sums
void launch_relax_struct(cudaStream_t st, int Sa, int it, const RelaxConst& c, const int64_t* act,
                         const int64_t* in_off, const int64_t* b_off, const float* forces, const double* bsum,
                         double data_mean, const double* v, RelaxStruct* rs, double* stat, float* res_f,
                         double* res_e, double* res_s, double* trace, int64_t trace_pitch);
// the atoms' step: v and r0 of every row of a moving structure (b_sid: batch structure of each of the N rows)
void launch_relax_rows(cudaStream_t st, int64_t N, const RelaxConst& c, const int64_t* act, const int64_t* in_off,
                       const int64_t* b_off, const int* b_sid, const float* forces, const RelaxStruct* rs, double* v,
                       double* r0);

}  // namespace b2m
