// graph.cuh -- GPU-resident partitioned atom graph + bond graph + angle list.
//
// Replaces, per rank, what the reference builds on the CPU for *all* partitions on every call:
//   fpis.c:418-901 (neighbour list), subgraph_creation_utils.c:26-931 (slab partition, halo
//   sections, bond/line graph).  Layout is CSR-by-destination with int32 indices (the reference
//   emits COO int64, SURVEY.md 3.3) so that every scatter-add of the model is a segmented sum.
#pragma once
#include "common.cuh"

namespace b2m {

// cell grid of one structure, and its lattice (rows), inverse and periodicity
struct GridParams {
  double lat[9];
  double inv[9];
  int nc[3], reach[3], pbc[3];
  double fmin[3], fscale[3];
};

// How a build kernel finds the grid of an atom's structure (DESIGN.md §12).  Each build kernel is one template over
// these two; a single-structure build runs the OneGrid instantiations, a batch the GridTable ones.
// OneGrid: one structure, its grid in the kernel parameters, cell ids from 0.
struct OneGrid {
  GridParams gp;
  static constexpr bool kPartitioned = true;  // atoms may be owned by other partitions: owners and halo masks
  __device__ __forceinline__ int structure(int64_t) const { return 0; }
  __device__ __forceinline__ const GridParams& grid(int) const { return gp; }
  __device__ __forceinline__ int first_cell(int) const { return 0; }
};
// GridTable: structure s = sid[gid] of a batch, its grid gp[s] and its first global cell id cell_off[s]; one partition.
struct GridTable {
  const GridParams* gp;  // [S]
  const int* cell_off;   // [S]
  const int* sid;        // [N]
  static constexpr bool kPartitioned = false;  // every atom owned by partition 0
  __device__ __forceinline__ int structure(int64_t g) const { return sid[g]; }
  __device__ __forceinline__ const GridParams& grid(int s) const { return gp[s]; }
  __device__ __forceinline__ int first_cell(int s) const { return cell_off[s]; }
};

struct Graph {
  // ---- problem ----
  int64_t N = 0;
  int rank = 0, world = 1;
  int axis = 0;              // partition axis (longest Cartesian extent of wrapped coords)
  double walls[MAXP] = {0};  // world-1 walls in wrapped fractional coordinate
  double r_cut = 0, r_bond = 0, tol = 1e-8;
  // ---- sizes ----
  int n_own = 0, n_halo = 0, n_loc = 0;
  int64_t E = 0;
  int B_own = 0, B_halo = 0, B_loc = 0;
  int64_t A = 0;
  // ---- per global atom ----
  DBuf<double> cart;      // [N,3] input
  DBuf<double> fracw;     // [N,3] wrapped fractional
  DBuf<double> wc;        // [N,3] wrapped Cartesian
  DBuf<int> corr;         // [N,3] integer unwrap correction (frac = fracw + corr)
  DBuf<int> species;      // [N]
  DBuf<unsigned char> owner;  // [N]
  DBuf<int> g2l;          // [N] global -> local (-1 if not local)
  DBuf<int> cell_of;      // [N]
  DBuf<int> s_gid;        // [N] atoms sorted by cell
  DBuf<double> s_wc;      // [N,3] wrapped Cartesian in sorted order
  DBuf<int> sidx_of_gid;  // [N]
  DBuf<int> cell_start;   // [ncell+1]
  // ---- local atoms: [owned (cell order) | halo (owner, gid order)] ----
  DBuf<int> gid;       // [n_loc]
  DBuf<int> type;      // [n_loc]
  DBuf<int> loc_sidx;  // [n_loc] sorted index of each local atom
  DBuf<unsigned> to_mask;  // [n_own] bit q set: has a neighbour owned by q
  int n_from[MAXP] = {0}, from_off[MAXP + 1] = {0};  // halo sections by owner
  int n_to[MAXP] = {0}, to_off[MAXP + 1] = {0};
  DBuf<int> to_list;  // [sum n_to] local ids (gid ascending within q)
  // ---- edges: CSR by owned dst ----
  DBuf<int> row_ptr;   // [n_own+1]
  DBuf<int> e_src;     // [E] local src (may be halo)
  DBuf<int> e_dst;     // [E] local dst
  DBuf<int> e_img;     // [E] packed image of src as seen from dst (wrapped frame)
  DBuf<int> e_bond;    // [E] owned bond id or -1
  DBuf<float4> e_vec;  // [E] (vx,vy,vz,d), vec = x_dst + off.L - x_src  (chgnet.py:96-99)
  // ---- bonds: [owned (row order) | halo (halo-atom order)] ----
  DBuf<int> brow_ptr;   // [n_loc+1] in-bonds by dst local atom
  DBuf<int> b_src_gid;  // [B_loc]
  DBuf<int> b_src;      // [B_loc] local src (-1 if src atom not local; halo bonds only)
  DBuf<int> b_dst;      // [B_loc] local dst
  DBuf<int> b_img;      // [B_loc]
  DBuf<int> b_edge;     // [B_own]
  DBuf<float4> b_vec;   // [B_loc]
  int nb_from[MAXP] = {0}, bfrom_off[MAXP + 1] = {0};
  int nb_to[MAXP] = {0}, bto_off[MAXP + 1] = {0};
  DBuf<int> bto_list;   // [sum nb_to] owned bond ids to send to q
  // ---- angles grouped by centre: (a = s->c) -> (b = c->x), x != s ----
  DBuf<int> out_ptr, out_list;   // owned bonds by src local atom
  DBuf<int> a_in, a_out, a_ctr;  // [A]
  // ---- scratch ----
  DBuf<int> tmp_i0, tmp_i1, tmp_i2, tmp_i3;
  DBuf<unsigned char> tmp_flag;
  DBuf<char> cub_tmp;
  DBuf<double> red_tmp;
  DBuf<int> e_src_gid;
  DBuf<unsigned char> keys_out;  // persistent scratch: no cudaMalloc/cudaFree on the per-step path
  DBuf<int> sel_out, nsel;
  // unfolded (heat-flux) structures: slab walls are measured from the lowest fractional coordinate, not from 0, because
  // the periodic images put atoms below 0 along the partition axis
  bool walls_from_min = false;
  // partition policy (b2m_set_partition_policy): false = the reference's equally spaced walls, true = walls at the
  // quantiles of the atoms' work (edges + angles), so that every slab holds about the same share of it (DESIGN.md §4.1)
  bool balanced = false;
  DBuf<double> bal_x;     // [2N] coordinates along the axis, then sorted
  DBuf<long long> bal_w;  // [2N] work per atom, then sorted; its inclusive prefix overwrites the first half
  // ---- structures: the graph is the disjoint union of S structures (S = 1 unless a batch), structure s owning the
  // gids b_off[s] .. b_off[s + 1] - 1 ----
  int S = 0;
  bool batch = false;            // built as a batch (DESIGN.md §12): one partition, the GridTable kernels, b_sid filled
  std::vector<int64_t> b_off;    // [S + 1]
  std::vector<double> volume;    // [S]
  std::vector<GridParams> grids; // [S] each structure's own cell grid
  DBuf<GridParams> b_gp;         // [S] grids on the device (batch)
  DBuf<int> b_cell_off;          // [S] first global cell id of each structure (batch)
  DBuf<int> b_sid;               // [N] structure of each atom (batch)
  DBuf<int64_t> b_doff;          // [S + 1] b_off on the device
  std::vector<int64_t> b_name;   // the caller's index of each structure, for error messages; empty: the batch index

  // nstruct structures, atoms concatenated in structure order (natoms[s] each), lattices [S][9] (rows), pbc flags
  // [S][3].  Inside a structure the rows, edges, bonds and angles come in the order a build of that structure alone
  // gives, with every atom index offset by b_off[s].  A batch (as_batch) needs world = 1 and names the structure in
  // its errors; otherwise nstruct = 1 and the atoms are split into world slabs, this rank holding slab `rank`.
  void build(cudaStream_t st, int nstruct, const int64_t* natoms, const double* h_cart, const double* h_lat,
             const int32_t* h_species, const int* h_pbc, double rcut, double rbond, double tol_, int rank_, int world_,
             bool as_batch);
  int64_t export_info(cudaStream_t st, int which, int64_t* out, int64_t cap);
  std::string structure_name(int s) const {  // "structure <caller's index>"
    return "structure " + std::to_string(s < (int)b_name.size() ? b_name[s] : (int64_t)s);
  }

 private:
  void upload(cudaStream_t st, const double* h_cart, const int32_t* h_species);
  void sort_by_cell(cudaStream_t st, int ncell);
  void build_rows(cudaStream_t st);
  // f(grid) with the grid object of this build: GridTable for a batch, else OneGrid of the one structure
  template <class F>
  void with_grid(F&& f) const {
    if (batch) f(GridTable{b_gp.p, b_cell_off.p, b_sid.p});
    else f(OneGrid{grids[0]});
  }
};

// Unfolded cell of the heat flux (DESIGN.md §10): the n cell atoms at their given positions, followed by every periodic
// image j + s.L (s integer, nonzero, zero along non-periodic axes) whose fractional coordinates lie in the cell atoms'
// fractional bounding box widened by reach / h_k along each periodic axis k (h_k: the cell's height across lattice
// plane k).  Every atom within `reach` Angstrom of a cell atom is inside that box.  Built on the GPU as count / scan /
// fill; the result stays on the device and is the input of a non-periodic Graph::build.
struct Unfold {
  int64_t n = 0, N = 0;   // cell atoms, cell atoms + images
  DBuf<double> cart;      // [N,3]
  DBuf<int> species;      // [N]
  DBuf<int> image_of;     // [N] cell atom of every unfolded atom (image_of[i] = i for i < n)
  DBuf<double> cart0, frac0, red_tmp;
  DBuf<int64_t> dseg;  // [2] the atoms 0 .. n - 1 as one segment of the bounds reduction
  DBuf<int> species0, cnt, off;
  DBuf<char> cub_tmp;
  void build(cudaStream_t st, int64_t natoms, const double* h_cart, const int32_t* h_species, const double* h_lat,
             const int* h_pbc, double reach);
};

}  // namespace b2m
