/*
 * b200mlip.h -- C-ABI of libb200mlip.so: the H100-native (sm_90a) engine behind the
 * DistMLIP-compatible CHGNet hot path.  Plain C, no CPython / NumPy / torch types.
 *
 * What each entry point replaces in the reference (AegisIK/DistMLIP @ 9824cd4):
 *
 *   b2m_create / b2m_load_weights / b2m_finalize_weights
 *        CHGNet_Dist.from_existing + enable_distributed_mode, which deep-copy every sub-module
 *        onto every GPU (DistMLIP/implementations/matgl/models/chgnet.py:455-560).
 *   b2m_set_structure
 *        Distributed.create_distributed -> get_subgraphs_fast, the CPU neighbour list + slab
 *        partitioner + bond/line-graph builder run on every calculate()
 *        (DistMLIP/distributed/dist.py:158-275; subgraph_creation_fast.c:92-453; fpis.c:418-901;
 *        subgraph_creation_utils.c:26-931), plus the geometry block of potential_forward_dist
 *        (chgnet.py:33-197).
 *   b2m_compute
 *        CHGNet_Dist.dist_forward (chgnet.py:208-453) + Potential_Dist.forward's scaling,
 *        torch.autograd.backward, F = -grad, sigma = strain.grad / V * 160.21766208
 *        (DistMLIP/implementations/matgl/pes.py:50-146).
 *   b2m_create with ndev > 1, or b2m_comm_unique_id / b2m_comm_init
 *        the reference has no communicator: Distributed.transfer_nodes does cross-device
 *        slice copies from one thread (dist.py:323-358).  Here either one process drives every
 *        GPU (ndev > 1: peer-memory halo stores ordered by CUDA events, one host thread per
 *        partition) or one process per GPU with NCCL point-to-point halo exchange between slab
 *        neighbours.
 *   b2m_set_partition_policy
 *        no counterpart: the reference always places its slab walls equally spaced in fractional coordinate
 *        (subgraph_creation_utils.c:1370-1456); the balanced policy places them at the quantiles of the atoms' work.
 *   b2m_get_partition_info
 *        the 19-tuple returned by get_subgraphs_fast (subgraph_creation_fast.c:403-422), in
 *        canonical (set) form, for parity tests.
 *
 * Conventions: every call returns 0 on success, <0 on error (message via b2m_last_error);
 * the library never calls exit().  Caller owns all host buffers; the library owns all device
 * memory, streams and NCCL communicators.  A handle is single-caller (no internal locking) and
 * may be used with the GIL released.
 */
#ifndef B200MLIP_H
#define B200MLIP_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b2m_engine* b2m_handle;

/* error codes */
#define B2M_OK 0
#define B2M_ERR_INVALID (-1)     /* bad argument / unsupported model dimension          */
#define B2M_ERR_PARTITIONS (-2)  /* num_partitions < 1                                   */
#define B2M_ERR_SELF_EDGE (-3)   /* unused: periodic self images are never neighbours    */
#define B2M_ERR_SLAB_WIDTH (-4)  /* slab width <= 2 (r_cut [+ r_bond])  (ref: utils.c:1512-1529) */
#define B2M_ERR_CUDA (-5)        /* CUDA / NCCL runtime failure                          */
#define B2M_ERR_STATE (-6)       /* call order violation (e.g. compute before set_structure) */

typedef struct {
  int32_t n_elem;            /* rows of atom_embedding.weight                      */
  int32_t dim;               /* atom = bond = angle feature width (64 supported)   */
  int32_t max_n;             /* radial basis size (9 supported)                    */
  int32_t max_f;             /* Fourier order (4 supported -> 9 features)          */
  int32_t n_blocks;          /* number of atom-graph blocks (>= 2)                 */
  int32_t cutoff_exponent;   /* polynomial envelope exponent p                     */
  double cutoff;             /* r_cut  (Angstrom)                                  */
  double three_body_cutoff;  /* r_bond (Angstrom)                                  */
  double data_mean;          /* Potential: E = std * E + mean (pes.py:109)         */
  double data_std;
} b2m_model_desc;

/* devices: CUDA ordinals owned by this handle, one per partition (SURVEY 8b; the reference's
 * enable_distributed_mode(gpus), chgnet.py:455-549).
 *   ndev == 1: one partition, or one rank of a multi-process job (b2m_comm_init).
 *   ndev  > 1: a single-process group: partition p runs on devices[p] (ordinals may repeat, e.g.
 *              {0, 0} = two partitions on one GPU), one host thread + stream per partition inside
 *              b2m_set_structure / b2m_compute, halo rows exchanged as direct peer-memory stores
 *              ordered by CUDA events (no NCCL).  b2m_get_counts / b2m_get_partition_info describe
 *              the partition chosen with b2m_set_view (default 0), b2m_debug_tensor partition 0;
 *              energies, forces, stress and the site-wise readout are those of the whole structure. */
int b2m_create(const b2m_model_desc* desc, const int* devices, int ndev, b2m_handle* out);
int b2m_destroy(b2m_handle h);
const char* b2m_last_error(b2m_handle h);

/* TensorNet (SURVEY.md 8(f).2): the same handle type and every call below, for a model with matgl's TensorNet attribute
 * tree (DistMLIP/implementations/matgl/models/tensornet.py:163-204: bond_expansion, tensor_embedding, layers, out_norm,
 * linear, final_layer).  Supported: units = 64, Gaussian bond expansion (<= 64 centres), swish, O(3) or SO(3),
 * is_intensive = False, no state features.  No bond graph: use_bond_graph False, three_body_cutoff 0 (pes.py:79-80).
 * b2m_get_sitewise is an error on such a handle. */
typedef struct {
  int32_t n_elem;    /* len(element_types)                                            */
  int32_t units;     /* 64                                                            */
  int32_t num_rbf;   /* Gaussian centres (the centres themselves are a state_dict key) */
  int32_t n_blocks;  /* interaction layers                                            */
  int32_t so3;       /* equivariance_invariance_group: 0 = "O(3)", 1 = "SO(3)"       */
  int32_t reserved;
  double cutoff;     /* r_cut (Angstrom), also the cosine cutoff radius               */
  double rbf_width;  /* exp(-width (d - mu)^2)                                        */
  double data_mean;
  double data_std;
} b2m_tensornet_desc;
int b2m_create_tensornet(const b2m_tensornet_desc* desc, const int* devices, int ndev, b2m_handle* out);

/* MACE (DESIGN.md §11): the same handle type and calls, for a mace ScaleShiftMACE with hidden features C x 0e
 * (hidden_max_l = 0, MACE-MP-0 "small"), C x 0e + C x 1o (hidden_max_l = 1, MACE-MP-0 "medium"; then max_ell >= 1) or
 * C x 0e + C x 1o + C x 2e (hidden_max_l = 2, MACE-MP-0 "large"; then max_ell >= 2), loaded key by key from its
 * state_dict (arithmetic and conventions: oracle/mace_ref.py and, for 0e+1o and 0e+1o+2e, tests/mace_eq_ref.py and
 * tests/mace_l2_ref.py).  hidden_mul must be channels for every l <= hidden_max_l and 0 above (unequal multiplicities
 * are not supported); a contradiction fails b2m_create_mace with B2M_ERR_INVALID.
 * Supported: one head, C a multiple of 32 with C <= 128, max_ell <= 3, correlation <= 3, Bessel basis x polynomial cutoff,
 * an e3nn FullyConnectedNet radial MLP (hidden widths <= 64), RealAgnostic(Residual)InteractionBlock per layer, linear
 * readouts and a gated non-linear last readout; optionally mace's ZBL pair repulsion (keys pair_repulsion_fn.{c, a_exp,
 * a_prefactor, p, covalent_radii}) and Agnesi distance transform (radial_embedding.distance_transform.{q, p, a,
 * covalent_radii}), each turned on by loading its keys (DESIGN.md §11.2; this struct does not change).  A partial key set,
 * a wrong shape, an atomic number beyond a covalent_radii table or a non-integer ZBL p fails b2m_finalize_weights with
 * B2M_ERR_INVALID.  Edges are every periodic image closer than r_max (no bond graph).
 * Scale, shift and the atomic energies E0 come from the state_dict: b2m_set_scaling and b2m_set_element_refs return
 * B2M_ERR_INVALID on such a handle, as does b2m_get_sitewise.  b2m_set_atomic / b2m_get_atomic give
 * energies[i] = E0[z_i] + scale * e_i + shift and the per-atom virials; b2m_compute_heat_flux weights that whole energy
 * (its J_conv uses it, E0 and shift included). */
typedef struct {
  int32_t n_elem;                 /* len(atomic_numbers)                                                 */
  int32_t channels;               /* C of hidden_irreps = C x 0e (+ C x 1o (+ C x 2e))                   */
  int32_t max_ell;                /* edge spherical harmonics 0..max_ell                                 */
  int32_t correlation;            /* symmetric-contraction order                                         */
  int32_t num_interactions;       /* <= 8                                                                */
  int32_t num_bessel;             /* radial Bessel functions                                             */
  int32_t num_polynomial_cutoff;  /* PolynomialCutoff exponent p                                         */
  int32_t mlp_hidden;             /* width of the non-linear readout                                     */
  int32_t residual_mask;          /* bit t: interactions.t is a RealAgnosticResidualInteractionBlock     */
  int32_t hidden_max_l;           /* 0: C x 0e; 1: C x 0e + C x 1o; 2: + C x 2e (other values invalid)    */
  double r_max;                   /* cutoff (Angstrom)                                                   */
  double c_act;                   /* e3nn normalize2mom(SiLU) constant of the radial MLP and the readout */
  double avg_num_neighbors[8];    /* per interaction                                                     */
  int32_t hidden_mul[4];          /* multiplicity of each hidden l, as e3nn's Irreps has it              */
} b2m_mace_desc;
int b2m_create_mace(const b2m_mace_desc* desc, const int* devices, int ndev, b2m_handle* out);

/* One call per state_dict key of the matgl CHGNet attribute tree (SURVEY.md 8c), fp32 row-major. */
int b2m_load_weights(b2m_handle h, const char* name, const float* host_ptr, const int64_t* shape, int ndim);
/* Optional per-element energy offsets (Potential.element_refs), length n_elem. */
int b2m_set_element_refs(b2m_handle h, const double* offsets, int n);
/* Potential scaling E = std * E + mean (pes.py:109); may be changed between computes. */
int b2m_set_scaling(b2m_handle h, double data_mean, double data_std);
/* Composes derived matrices, uploads everything. Fails if a required key is missing. */
int b2m_finalize_weights(b2m_handle h);

/* Multi-process graph parallelism: rank 0 makes an id, every rank calls b2m_comm_init with it. */
int b2m_comm_unique_id(char* out128);
int b2m_comm_init(b2m_handle h, const char* id128, int rank, int world);
/* Graph-only view of partition `rank` of `world` without a communicator (parity tests of the
 * partitioner on one GPU).  b2m_compute refuses to run in this state when world > 1. */
int b2m_set_partition(b2m_handle h, int rank, int world);

/* Where the world - 1 slab walls go (DESIGN.md §4, §4.1).  Axis: the longest Cartesian extent of the wrapped
 * coordinates, for both policies.
 *   B2M_PARTITION_EQUAL (default): the reference's walls, equally spaced in fractional coordinate between the lowest and
 *     highest atom; fails with B2M_ERR_SLAB_WIDTH when the first slab is not wider than 2 (r_cut + r_bond) along the
 *     lattice column of the axis.
 *   B2M_PARTITION_BALANCED: every slab owns about the same work w_i = deg_i + nb_i (nb_i - 1) (deg_i: edges into atom
 *     i, nb_i: bonds into it; the second term is 0 without a bond graph).  Wall k goes half-way between the two
 *     distinct coordinates where the prefix of the work, atoms sorted along the axis, first reaches k W / world; then
 *     every slab is widened to at least 2 (r_cut + r_bond) across the walls (the cell's height, not the lattice column),
 *     or the build fails with B2M_ERR_SLAB_WIDTH naming the slab.  Every partition and every rank computes the same
 *     walls from the same coordinates: nothing is exchanged.
 * The policy holds for every partition of a single-process group and takes effect at the next b2m_set_structure (the
 * unfolded heat-flux cell included).  Any other value: B2M_ERR_INVALID. */
#define B2M_PARTITION_EQUAL 0
#define B2M_PARTITION_BALANCED 1
int b2m_set_partition_policy(b2m_handle h, int policy);

/* Graph build (neighbour list, slab partition, halo sections, bond graph, angles) on the GPU.
 * cart: [natoms,3] f64 Cartesian (unwrapped ok); lattice9: row vectors; species: index into
 * element_types; pbc3: 0/1 flags.  tol as in the reference (1e-8 on d^2). */
int b2m_set_structure(b2m_handle h, int64_t natoms, const double* cart, const double* lattice9,
                      const int32_t* species, const int* pbc3, double tol);

/* Energy (+forces [natoms,3] eV/A, +stress [9] GPa).  forces/stress9 may be NULL.
 * With world > 1 every rank receives the full (all-reduced) result. */
int b2m_compute(b2m_handle h, int want_forces, int want_stress, double* energy, float* forces, float* stress9);
/* Same arithmetic, graph already resident; runs `reps` passes and returns device time (ms) of
 * the last one measured with CUDA events on the compute stream. Used by bench.py `value`. */
int b2m_compute_resident(b2m_handle h, int want_forces, int want_stress, int reps, double* energy, float* ms);
/* Results of the last evaluation (b2m_compute or b2m_compute_resident) without running another one: energy,
 * forces [natoms][3] and stress [3][3] (GPa), as b2m_compute returns them; any pointer may be NULL. */
int b2m_get_results(b2m_handle h, double* energy, float* forces, float* stress9);

/* Batched evaluation (DESIGN.md §12): many independent structures in one graph build and one model pass, for relaxing
 * or screening many small cells, phonon displacements, strain sets, NEB images or a dataset.  nstruct structures, atoms
 * concatenated in structure order (structure s owns the atoms off_s .. off_s + natoms[s] - 1, off_s the sum of the
 * natoms before it): cart [sum natoms][3], lattice9 [nstruct][9] row vectors, species [sum natoms], pbc3 [nstruct][3],
 * tol as in b2m_set_structure.  The graph is the disjoint union of the structures' graphs: no edge crosses from one
 * structure to another, each has its own lattice, periodicity and cell grid, and the graph build costs the same number
 * of launches and host synchronisations whatever nstruct is.
 * Refused with B2M_ERR_INVALID and a message (nothing of the handle changes but the resident structure, which is gone):
 * a single-process group (ndev > 1) or a rank of a multi-process job (a batch runs on one partition), nstruct < 1, and,
 * naming the structure's index, a structure with no atoms, pbc flags other than 0 / 1, a singular lattice, a cell far too
 * small for the cutoff, or no edge at all (isolated atoms are not supported).  B2M_ERR_STATE while a heat-flux reach is
 * set.
 * While a batch is resident, b2m_compute, b2m_compute_resident, b2m_get_results and b2m_compute_heat_flux return
 * B2M_ERR_STATE (their one energy and one stress do not describe a batch); b2m_get_atomic, b2m_get_sitewise,
 * b2m_get_counts, b2m_get_partition_info, b2m_last_timings and b2m_release_workspace work, with the atoms numbered in
 * batch order.  The next b2m_set_structure drops the batch. */
int b2m_set_structures(b2m_handle h, int32_t nstruct, const int64_t* natoms, const double* cart,
                       const double* lattice9, const int32_t* species, const int* pbc3, double tol);
/* Evaluates the resident batch: energies [nstruct] (eV), forces [sum natoms][3] (eV/A), stress9 [nstruct][9] (GPa), each
 * what b2m_compute returns for that structure alone (the stress from the sum of the structure's per-atom virials over
 * its own volume).  forces / stress9 may be NULL.  Per-atom energies and virials are always computed for a batch, so
 * b2m_get_atomic returns them afterwards whatever b2m_set_atomic says (energies[i] with data_mean / natoms[s] of its
 * structure s). */
int b2m_compute_batch(b2m_handle h, int want_forces, int want_stress, double* energies, float* forces, float* stress9);

/* Batched relaxation (DESIGN.md §13): ASE's FIRE, optionally with its FrechetCellFilter, run independently on each
 * structure of a batch, with the whole loop on the device.  fmax (eV/A; 0 never converges), steps (optimizer steps at
 * most: a structure is evaluated at most steps + 1 times), relax_cell (the Frechet cell filter, exp_cell_factor = natoms,
 * with scalar_pressure in eV/A^3; the cell force weighs the strain derivative by stress_weight * 160.21766208), and the
 * nine constants of ase.optimize.FIRE (ASE's defaults: dt 0.1, maxstep 0.2, dtmax 1.0, Nmin 5, finc 1.1, fdec 0.5,
 * astart 0.1, fa 0.99, a 0.1). */
typedef struct {
  double fmax;
  int32_t steps;
  int32_t relax_cell;
  double scalar_pressure;
  double stress_weight;
  double dt, maxstep, dtmax, Nmin, finc, fdec, astart, fa, a;
} b2m_relax_params;
/* Relaxes nstruct structures, laid out as in b2m_set_structures.  Each step builds the graph of the structures still
 * running, evaluates it, takes one FIRE step per structure on the device and copies one small status block to the
 * host; a structure leaves the batch when max_row |f_row| < fmax (cell rows included) or after `steps` steps.  On
 * return cart_inout [sum natoms][3] and lattice9_inout [nstruct][9] hold the final geometries, and, each at that
 * geometry (its last evaluation): energies [nstruct] (eV), forces [sum natoms][3] (eV/A), stress9 [nstruct][9] (GPa),
 * steps_taken [nstruct], converged [nstruct] (1 / 0).  energy_trace [nstruct][steps + 1], if not NULL, gets the energy
 * of every evaluation, NaN after the structure stopped.  Every output but energy_trace is required.
 * Refused before anything runs, with B2M_ERR_INVALID: a single-process group or a rank of a multi-process job,
 * nstruct < 1, a structure with no atoms, relax_cell with a non-periodic axis, steps < 0, non-finite FIRE constants,
 * fmax or pressure, fmax < 0, dt, maxstep or dtmax <= 0, a NULL output other than energy_trace (whose [nstruct][steps + 1]
 * buffer is only allocated when it is given); B2M_ERR_STATE while a heat-flux reach is set or before
 * b2m_finalize_weights.  What b2m_set_structures
 * refuses in the graph build (a singular lattice, a structure without edges, ...) fails the step it happens in, with
 * the same code and a message naming the step and the structure by its input index, for example a structure whose
 * atoms lose every edge; the handle stays usable.  Afterwards the batch of the
 * last step is resident, as after b2m_compute_batch, and b2m_get_counts' launch count is that of the last step. */
int b2m_relax_batch(b2m_handle h, int32_t nstruct, const int64_t* natoms, double* cart_inout, double* lattice9_inout,
                    const int32_t* species, const int* pbc3, double tol, const b2m_relax_params* params,
                    double* energies, float* forces, float* stress9, int32_t* steps_taken, int32_t* converged,
                    double* energy_trace);

/* Per-atom energies and virials (DESIGN.md "Per-atom energies and virials"), off by default.  With on != 0 the
 * following evaluations (b2m_compute, b2m_compute_resident) also produce, for every atom i,
 *   energies[i] = data_std * e_i + element_ref[Z_i] + data_mean / natoms   (eV; sums to the energy)
 *   virials[i]  = 1/2 sum over the edges e with endpoint i of v_e (x) dE/dv_e   (eV, 3x3 row-major, not symmetrised;
 *                 sums to the strain derivative of the energy, i.e. stress * volume / 160.21766208)
 * With the flag off no buffer is allocated and no extra kernel or collective runs. */
int b2m_set_atomic(b2m_handle h, int on);
/* Per-atom results of the last evaluation (energies [natoms] or NULL, virials [natoms][9] or NULL), every partition
 * layout, both model families.  B2M_ERR_STATE if that evaluation ran with the flag off, or if virials are asked for
 * after an evaluation without a backward (want_forces = want_stress = 0). */
int b2m_get_atomic(b2m_handle h, double* energies, float* virials);

/* Heat flux of the model (DESIGN.md "Heat flux"), off by default (reach = 0).  With reach > 0 (Angstrom, at least the
 * model's receptive field: n_blocks * r_cut for CHGNet, (n_blocks + 1) * r_cut for TensorNet, num_interactions * r_max
 * for MACE) the following
 * b2m_set_structure calls build the unfolded cell: the natoms cell atoms, then every periodic image within `reach` of
 * them along the periodic axes, evaluated without periodicity with the energy U = sum of the cell atoms' energies.
 * On such a handle b2m_compute (and b2m_compute_resident, b2m_get_results) returns the periodic energy, forces [natoms][3]
 * (the forces of an atom's images summed onto it) and stress, and b2m_get_atomic the cell atoms' values: an MD loop pays
 * for the flux only on the steps that call b2m_compute_heat_flux.  reach = 0 switches back at the next
 * b2m_set_structure. */
int b2m_set_heat_flux(b2m_handle h, double reach);
/* One masked and three position-seeded evaluations of the unfolded cell.  vel: [natoms][3] Angstrom / (unit time), f64.
 * energy / forces / stress9 as b2m_compute (any may be NULL).  flux6 (f64):
 *   flux6[0..2] = J_pot  = sum_{i<n} sum_j r_ij (dU_i/dr_j . v_j),  r_ij = r_i - r_j, j over every unfolded atom
 *   flux6[3..5] = J_conv = sum_{i<n} e_i v_i  (e_i: the per-atom energies of b2m_set_atomic)
 * in eV * (velocity unit), not divided by the volume (LAMMPS compute heat/flux); the kinetic part sum 1/2 m v^2 v is the
 * caller's.  Afterwards b2m_get_atomic returns the per-atom energies and virials of the masked evaluation.
 * B2M_ERR_STATE when the reach is 0 or the resident structure was set before it. */
int b2m_compute_heat_flux(b2m_handle h, const double* vel, double* energy, float* forces, float* stress9,
                          double* flux6);

/* site-wise readout (magmom) for all atoms, [natoms] */
int b2m_get_sitewise(b2m_handle h, float* out);

/* Single-process groups: which partition b2m_get_counts / b2m_get_partition_info describe (default 0).  The reference's
 * Distributed keeps every partition's arrays on the host (dist.py:39-99) and its counters take a `partition` argument
 * (dist.py:462-551); this is the equivalent view. */
int b2m_set_view(b2m_handle h, int part);

/* counts: [0]=n_own [1]=n_halo [2]=n_edges [3]=n_bond_own [4]=n_bond_halo [5]=n_angles
 *         [6]=partition axis [7]=rank [8]=world [9]=kernel launches in last compute */
int b2m_get_counts(b2m_handle h, int64_t* out, int n);

/* Partition info export (int64, canonical content; see DESIGN.md "partition export"):
 *   which = 0: owned atom gids                 [n_own]
 *           1: halo atom gids                  [n_halo]   (grouped by owner, gid ascending)
 *           2: halo owner partition            [n_halo]
 *           3: edges (src gid, dst gid, ox,oy,oz)        [n_edges,5]
 *           4: bonds (src gid, dst gid, ox,oy,oz), owned first then halo  [n_bond,5]
 *           5: angles (in-bond id, out-bond id, centre gid)               [n_angles,3]
 *           6: to-lists (q, gid) pairs          [n_to,2]
 *           7: walls as IEEE-754 bit patterns   [world-1]
 * Returns number of int64 written, or <0. cap = capacity of out in int64 elements. */
int64_t b2m_get_partition_info(b2m_handle h, int which, int64_t* out, int64_t cap);

/* Debug taps (tests only): copies a named device tensor to host (fp32). rows/cols returned. */
int b2m_debug_tensor(b2m_handle h, const char* name, float* out, int64_t cap, int64_t* rows, int64_t* cols);

/* Frees the resident graph and every per-structure device buffer (weights, streams and communicators stay); the next
 * b2m_set_structure allocates again.  For callers that want the memory back between structures of very different size. */
int b2m_release_workspace(b2m_handle h);

/* Per-phase device timings (ms) of the last b2m_compute: [0]=graph build [1]=forward [2]=backward
 * [3]=edge-gather (atom conv fwd) kernel average [4]=total */
int b2m_last_timings(b2m_handle h, double* out, int n);

#ifdef __cplusplus
}
#endif
#endif
