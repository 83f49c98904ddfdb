// graph.cu -- GPU graph build: wrap, slab partition, global cell list, CSR neighbour list,
// halo sections, bond graph, centre-grouped angle list.  Integer/f64 work, HBM-bound.
//
// Reference behaviour reproduced (file:line in the reference's DistMLIP/distributed):
//   * wrap to the cell, unwrap correction ....................... fpis.c:492-506
//   * edge rule  tol < d^2 < r^2 + tol, i != j (no self images) . fpis.c:760, 827
//   * bond rule  d^2 < r_bond^2 + tol ........................... fpis.c:763, 844
//   * partition axis = longest Cartesian extent, walls equally spaced in fractional
//     coordinate + EPSILON, collision nudge ..................... subgraph_creation_utils.c:1370-1456
//   * owner = number of walls <= coordinate ..................... :1312-1322
//   * slab width check .......................................... :1512-1529
//   * edge owned by the partition of its dst .................... :178-250
//   * halo ("from") atoms = src atoms of owned edges living elsewhere; "to q" = owned atoms
//     with an edge into q ........................................ :1189-1306
//   * bond nodes: owned = bonds whose dst is owned; halo = every bond whose dst is a halo atom
//     ............................................................. :497-653
//   * line graph (s->d) -> (d->x), x != s by atom index, centre d . :703-751
// Not in the reference: the balanced partition policy (Graph::balanced, DESIGN.md §4.1) places the walls at the
// quantiles of the atoms' edge + angle work, slabs at least 2 (r_cut + r_bond) wide across the walls.
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <cstring>

#include "graph.cuh"

namespace b2m {

static constexpr double kEpsilon = 1e-10;  // subgraph_creation_utils.c:9

// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void wrap_atom(int64_t i, const double* __restrict__ cart, const GridParams& gp,
                                          double* __restrict__ fracw, double* __restrict__ wc, int* __restrict__ corr) {
  double x = cart[3 * i], y = cart[3 * i + 1], z = cart[3 * i + 2];
  double f[3];
  // frac = cart @ inv  (fpis.c:198-207, plain triple loop: no FMA contraction)
  for (int j = 0; j < 3; j++) {
    double s = 0.0;
    s = __dadd_rn(s, __dmul_rn(x, gp.inv[0 * 3 + j]));
    s = __dadd_rn(s, __dmul_rn(y, gp.inv[1 * 3 + j]));
    s = __dadd_rn(s, __dmul_rn(z, gp.inv[2 * 3 + j]));
    f[j] = s;
  }
  double w[3];
  for (int j = 0; j < 3; j++) {
    if (gp.pbc[j]) {
      double t = fmod(f[j], 1.0);
      if (t < 0) t += 1.0;
      w[j] = t;
      corr[3 * i + j] = (int)llrint(f[j] - t);
    } else {
      w[j] = f[j];
      corr[3 * i + j] = 0;
    }
    fracw[3 * i + j] = w[j];
  }
  for (int m = 0; m < 3; m++) {
    double s = 0.0;
    s = __dadd_rn(s, __dmul_rn(w[0], gp.lat[0 * 3 + m]));
    s = __dadd_rn(s, __dmul_rn(w[1], gp.lat[1 * 3 + m]));
    s = __dadd_rn(s, __dmul_rn(w[2], gp.lat[2 * 3 + m]));
    wc[3 * i + m] = s;
  }
}

template <class G>
__global__ void k_wrap(int64_t n, const double* __restrict__ cart, G grid, double* __restrict__ fracw,
                       double* __restrict__ wc, int* __restrict__ corr) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  wrap_atom(i, cart, grid.grid(grid.structure(i)), fracw, wc, corr);
}

// min/max of wc[.,0..2] and fracw[.,0..2] over the atoms off[s] .. off[s + 1] - 1 of structure s = blockIdx.x, split
// over gridDim.y blocks; out[s][blockIdx.y][12]
__global__ void k_minmax(const int64_t* __restrict__ off, const double* __restrict__ wc,
                         const double* __restrict__ fracw, double* __restrict__ out) {
  __shared__ double smin[6][256], smax[6][256];
  double mn[6], mx[6];
  for (int k = 0; k < 6; k++) {
    mn[k] = 1e300;
    mx[k] = -1e300;
  }
  for (int64_t i = off[blockIdx.x] + blockIdx.y * (int64_t)blockDim.x + threadIdx.x; i < off[blockIdx.x + 1];
       i += (int64_t)gridDim.y * blockDim.x) {
    for (int k = 0; k < 3; k++) {
      double a = wc[3 * i + k], b = fracw[3 * i + k];
      mn[k] = fmin(mn[k], a);
      mx[k] = fmax(mx[k], a);
      mn[3 + k] = fmin(mn[3 + k], b);
      mx[3 + k] = fmax(mx[3 + k], b);
    }
  }
  for (int k = 0; k < 6; k++) {
    smin[k][threadIdx.x] = mn[k];
    smax[k][threadIdx.x] = mx[k];
  }
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) {
      for (int k = 0; k < 6; k++) {
        smin[k][threadIdx.x] = fmin(smin[k][threadIdx.x], smin[k][threadIdx.x + s]);
        smax[k][threadIdx.x] = fmax(smax[k][threadIdx.x], smax[k][threadIdx.x + s]);
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    double* o = out + ((int64_t)blockIdx.x * gridDim.y + blockIdx.y) * 12;
    for (int k = 0; k < 6; k++) {
      o[k] = smin[k][0];
      o[6 + k] = smax[k][0];
    }
  }
}

struct Walls {
  double w[MAXP];
  int nw;
  int axis;
};

// counts atoms sitting exactly on a wall (subgraph_creation_utils.c:1436-1453)
__global__ void k_wall_collisions(int64_t n, const double* __restrict__ fracw, Walls wl, int* __restrict__ hits) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  double f = fracw[3 * i + wl.axis];
  for (int k = 0; k < wl.nw; k++)
    if (f == wl.w[k]) atomicAdd(&hits[k], 1);
}

__device__ __forceinline__ int cell_coord(double f, int k, const GridParams& gp) {
  int c;
  if (gp.pbc[k]) {
    c = (int)floor(f * gp.nc[k]);
  } else {
    c = (int)floor((f - gp.fmin[k]) * gp.fscale[k]);
  }
  if (c < 0) c = 0;
  if (c > gp.nc[k] - 1) c = gp.nc[k] - 1;
  return c;
}

// owner = number of walls <= the coordinate along the axis (0 without walls or partitions); cell id = the structure's first cell + its
// cell in the structure's grid
template <class G>
__global__ void k_owner_cell(int64_t n, const double* __restrict__ fracw, Walls wl, G grid,
                             unsigned char* __restrict__ owner, int* __restrict__ cell_of, int* __restrict__ iota) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int o = 0;
  if (G::kPartitioned) {
    double f = fracw[3 * i + wl.axis];
    for (int k = 0; k < wl.nw; k++)
      if (!(f < wl.w[k])) o = k + 1;  // first wall strictly greater wins (:1312-1322)
  }
  // walls ascending: o = number of walls <= f
  owner[i] = (unsigned char)o;
  const int s = grid.structure(i);
  const GridParams& gp = grid.grid(s);
  int cx = cell_coord(fracw[3 * i + 0], 0, gp);
  int cy = cell_coord(fracw[3 * i + 1], 1, gp);
  int cz = cell_coord(fracw[3 * i + 2], 2, gp);
  cell_of[i] = grid.first_cell(s) + (cx * gp.nc[1] + cy) * gp.nc[2] + cz;
  iota[i] = (int)i;
}

// balanced partition: work of the atom at sorted (cell-order) index i, keyed by its wrapped fractional coordinate along
// the partition axis.  w = incoming edges + angles centred on the atom (nb (nb - 1) bond pairs; 0 without a bond graph)
__global__ void k_work_keys(int64_t n, const int* __restrict__ s_gid, const double* __restrict__ fracw, int axis,
                            const int* __restrict__ cnt_e, const int* __restrict__ cnt_b, double* __restrict__ key,
                            long long* __restrict__ w) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long nb = cnt_b[i];
  key[i] = fracw[3 * (int64_t)s_gid[i] + axis];
  w[i] = (long long)cnt_e[i] + nb * (nb - 1);
}

// balanced partition, wall k + 1 of `world`: the atoms sorted by coordinate x[] with the inclusive prefix S[] of their
// work; i = first atom with S[i] * world >= (k + 1) * S[n-1].  gap[2k], gap[2k+1] = x[i] and the next larger coordinate
// (the wall goes half-way); when x[i] is the largest coordinate, the gap below it.
__global__ void k_balanced_gaps(int nw, int64_t n, int world, const double* __restrict__ x,
                                const long long* __restrict__ S, double* __restrict__ gap) {
  const int k = threadIdx.x;
  if (k >= nw) return;
  const long long target = (long long)(k + 1) * S[n - 1];
  int64_t lo = 0, hi = n - 1;  // S[n-1] * world >= target always
  while (lo < hi) {
    const int64_t m = (lo + hi) / 2;
    if (S[m] * world >= target) hi = m;
    else lo = m + 1;
  }
  const double xi = x[lo];
  int64_t a = lo, b = n;  // first index with x > xi
  while (a < b) {
    const int64_t m = (a + b) / 2;
    if (x[m] > xi) b = m;
    else a = m + 1;
  }
  if (a < n) {
    gap[2 * k] = xi, gap[2 * k + 1] = x[a];
    return;
  }
  a = 0, b = lo;  // first index with x >= xi
  while (a < b) {
    const int64_t m = (a + b) / 2;
    if (x[m] < xi) a = m + 1;
    else b = m;
  }
  gap[2 * k] = a > 0 ? x[a - 1] : xi, gap[2 * k + 1] = xi;
}

__global__ void k_cell_hist(int64_t n, const int* __restrict__ cell_sorted, int* __restrict__ cnt) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  atomicAdd(&cnt[cell_sorted[i]], 1);
}

// after sort: gather wrapped coords, inverse permutation, owned flags
__global__ void k_post_sort(int64_t n, const int* __restrict__ s_gid, const double* __restrict__ wc,
                            const unsigned char* __restrict__ owner, int rank, double* __restrict__ s_wc,
                            int* __restrict__ sidx_of_gid, int* __restrict__ own_flag) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int g = s_gid[i];
  s_wc[3 * i] = wc[3 * g];
  s_wc[3 * i + 1] = wc[3 * g + 1];
  s_wc[3 * i + 2] = wc[3 * g + 2];
  sidx_of_gid[g] = (int)i;
  own_flag[i] = owner[g] == rank ? 1 : 0;
}

// local ids for owned atoms (cell order)
__global__ void k_assign_owned(int64_t n, const int* __restrict__ s_gid, const int* __restrict__ own_flag,
                               const int* __restrict__ own_scan, const int* __restrict__ species,
                               int* __restrict__ gid, int* __restrict__ type, int* __restrict__ loc_sidx,
                               int* __restrict__ g2l) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int g = s_gid[i];
  if (own_flag[i]) {
    int l = own_scan[i];
    gid[l] = g;
    type[l] = species[g];
    loc_sidx[l] = (int)i;
    g2l[g] = l;
  } else {
    g2l[g] = -1;
  }
}

__device__ __forceinline__ int floordiv(int a, int b) {
  int q = a / b;
  if ((a % b != 0) && ((a < 0) != (b < 0))) q--;
  return q;
}

__device__ __forceinline__ int pack_img(int ix, int iy, int iz) {
  return ((ix + 128) & 255) | (((iy + 128) & 255) << 8) | (((iz + 128) & 255) << 16);
}
__host__ __device__ __forceinline__ void unpack_img(int p, int& ix, int& iy, int& iz) {
  ix = (p & 255) - 128;
  iy = ((p >> 8) & 255) - 128;
  iz = ((p >> 16) & 255) - 128;
}

// Visit every (neighbour j, image) of the centre at sorted index ci with tol < d2 < r2 + tol,
// gid_j != gid_centre, in a fixed global traversal order (identical on every rank).
template <class F>
__device__ __forceinline__ void traverse(int ci, const GridParams& gp, const int* __restrict__ s_gid,
                                         const double* __restrict__ s_wc, const int* __restrict__ cell_start,
                                         const double* __restrict__ fracw, double r2, double tol, F&& f) {
  const int gc = s_gid[ci];
  const double tx = s_wc[3 * ci], ty = s_wc[3 * ci + 1], tz = s_wc[3 * ci + 2];
  const int c0 = cell_coord(fracw[3 * gc + 0], 0, gp);
  const int c1 = cell_coord(fracw[3 * gc + 1], 1, gp);
  const int c2 = cell_coord(fracw[3 * gc + 2], 2, gp);
  for (int dx = -gp.reach[0]; dx <= gp.reach[0]; dx++) {
    int cx = c0 + dx, ix = 0;
    if (gp.pbc[0]) {
      ix = floordiv(cx, gp.nc[0]);
      cx -= ix * gp.nc[0];
    } else if (cx < 0 || cx >= gp.nc[0])
      continue;
    for (int dy = -gp.reach[1]; dy <= gp.reach[1]; dy++) {
      int cy = c1 + dy, iy = 0;
      if (gp.pbc[1]) {
        iy = floordiv(cy, gp.nc[1]);
        cy -= iy * gp.nc[1];
      } else if (cy < 0 || cy >= gp.nc[1])
        continue;
      for (int dz = -gp.reach[2]; dz <= gp.reach[2]; dz++) {
        int cz = c2 + dz, iz = 0;
        if (gp.pbc[2]) {
          iz = floordiv(cz, gp.nc[2]);
          cz -= iz * gp.nc[2];
        } else if (cz < 0 || cz >= gp.nc[2])
          continue;
        // image shift, summed like fpis.c:537-540 (no FMA contraction)
        double sh[3];
        for (int m = 0; m < 3; m++)
          sh[m] = __dadd_rn(__dadd_rn(__dmul_rn((double)ix, gp.lat[m]), __dmul_rn((double)iy, gp.lat[3 + m])),
                            __dmul_rn((double)iz, gp.lat[6 + m]));
        const int cell = (cx * gp.nc[1] + cy) * gp.nc[2] + cz;
        const int b = cell_start[cell], e = cell_start[cell + 1];
        for (int j = b; j < e; j++) {
          const int gj = s_gid[j];
          if (gj == gc) continue;
          const double ex = __dadd_rn(sh[0], s_wc[3 * j]);
          const double ey = __dadd_rn(sh[1], s_wc[3 * j + 1]);
          const double ez = __dadd_rn(sh[2], s_wc[3 * j + 2]);
          const double ddx = ex - tx, ddy = ey - ty, ddz = ez - tz;
          double d2 = 0.0;
          d2 = __dadd_rn(d2, __dmul_rn(ddx, ddx));
          d2 = __dadd_rn(d2, __dmul_rn(ddy, ddy));
          d2 = __dadd_rn(d2, __dmul_rn(ddz, ddz));
          if (d2 < r2 + tol && d2 > tol) f(j, gj, ddx, ddy, ddz, d2, ix, iy, iz);
        }
      }
    }
  }
}

// count edges / bonds per centre; centres given by sorted index list.  The traversal's cell ids are those of the centre's
// structure, so cell_start is offset by its first cell
template <class G>
__global__ void k_count(int ncent, const int* __restrict__ cent_sidx, G grid, const int* __restrict__ s_gid,
                        const double* __restrict__ s_wc, const int* __restrict__ cell_start,
                        const double* __restrict__ fracw, const unsigned char* __restrict__ owner, int rank, double r2,
                        double rb2, double tol, int* __restrict__ cnt_e, int* __restrict__ cnt_b,
                        unsigned* __restrict__ to_mask) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= ncent) return;
  const int ci = cent_sidx[t], s = grid.structure(s_gid[ci]);
  int ne = 0, nb = 0;
  unsigned mask = 0;
  traverse(ci, grid.grid(s), s_gid, s_wc, cell_start + grid.first_cell(s), fracw, r2, tol,
           [&](int, int gj, double, double, double, double d2, int, int, int) {
             ne++;
             if (d2 < rb2 + tol) nb++;
             if (G::kPartitioned) {
               int o = owner[gj];
               if (o != rank) mask |= 1u << o;
             }
           });
  if (cnt_e) cnt_e[t] = ne;
  cnt_b[t] = nb;
  if (G::kPartitioned && to_mask) to_mask[t] = mask;
}

// fill owned rows
template <class G>
__global__ void k_fill_owned(int n_own, const int* __restrict__ cent_sidx, G grid, const int* __restrict__ s_gid,
                             const double* __restrict__ s_wc, const int* __restrict__ cell_start,
                             const double* __restrict__ fracw, const unsigned char* __restrict__ owner, int rank,
                             double r2, double rb2, double tol, const int* __restrict__ row_ptr,
                             const int* __restrict__ brow_ptr, int* __restrict__ e_src_gid, int* __restrict__ e_dst,
                             int* __restrict__ e_img, int* __restrict__ e_bond, float4* __restrict__ e_vec,
                             int* __restrict__ b_src_gid, int* __restrict__ b_dst, int* __restrict__ b_img,
                             int* __restrict__ b_edge, float4* __restrict__ b_vec, unsigned char* __restrict__ halo_flag) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_own) return;
  const int ci = cent_sidx[t], s = grid.structure(s_gid[ci]);
  int e = row_ptr[t], b = brow_ptr[t];
  traverse(ci, grid.grid(s), s_gid, s_wc, cell_start + grid.first_cell(s), fracw, r2, tol,
           [&](int, int gj, double dx, double dy, double dz, double d2, int ix, int iy, int iz) {
             // (dx,dy,dz) = x_src_image - x_dst ; reference bond_vec = x_dst + off.L - x_src = -(dx,dy,dz)
             float4 v = make_float4((float)(-dx), (float)(-dy), (float)(-dz), (float)sqrt(d2));
             int img = pack_img(ix, iy, iz);
             e_src_gid[e] = gj;
             e_dst[e] = t;
             e_img[e] = img;
             e_vec[e] = v;
             if (owner[gj] != rank) halo_flag[gj] = 1;
             if (d2 < rb2 + tol) {
               e_bond[e] = b;
               b_src_gid[b] = gj;
               b_dst[b] = t;
               b_img[b] = img;
               b_edge[b] = e;
               b_vec[b] = v;
               b++;
             } else {
               e_bond[e] = -1;
             }
             e++;
           });
}

// batch: out[s] = ptr[off[s]] (edges before the first row of each structure)
__global__ void k_gather_at(int n, const int64_t* __restrict__ off, const int* __restrict__ ptr, int* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = ptr[off[i]];
}

// fill halo bond rows (every bond whose dst is a halo atom)
__global__ void k_fill_halo_bonds(int n_halo, int n_own, const int* __restrict__ cent_sidx, GridParams gp,
                                  const int* __restrict__ s_gid, const double* __restrict__ s_wc,
                                  const int* __restrict__ cell_start, const double* __restrict__ fracw,
                                  double rb2, double tol, const int* __restrict__ brow_ptr,
                                  int* __restrict__ b_src_gid, int* __restrict__ b_dst, int* __restrict__ b_img,
                                  float4* __restrict__ b_vec) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_halo) return;
  int b = brow_ptr[n_own + t];
  traverse(cent_sidx[t], gp, s_gid, s_wc, cell_start, fracw, rb2, tol,
           [&](int, int gj, double dx, double dy, double dz, double d2, int ix, int iy, int iz) {
             b_src_gid[b] = gj;
             b_dst[b] = n_own + t;
             b_img[b] = pack_img(ix, iy, iz);
             b_vec[b] = make_float4((float)(-dx), (float)(-dy), (float)(-dz), (float)sqrt(d2));
             b++;
           });
}

__global__ void k_halo_keys(int64_t n, const unsigned char* __restrict__ halo_flag,
                            const unsigned char* __restrict__ owner, int world, unsigned char* __restrict__ key,
                            int* __restrict__ iota) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  key[i] = halo_flag[i] ? owner[i] : (unsigned char)world;
  iota[i] = (int)i;
}

__global__ void k_assign_halo(int n_halo, int n_own, const int* __restrict__ halo_gid_sorted,
                              const int* __restrict__ species, const int* __restrict__ sidx_of_gid,
                              int* __restrict__ gid, int* __restrict__ type, int* __restrict__ loc_sidx,
                              int* __restrict__ g2l) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_halo) return;
  int g = halo_gid_sorted[i];
  gid[n_own + i] = g;
  type[n_own + i] = species[g];
  loc_sidx[n_own + i] = sidx_of_gid[g];
  g2l[g] = n_own + i;
}

__global__ void k_relabel(int64_t n, const int* __restrict__ src_gid, const int* __restrict__ g2l,
                          int* __restrict__ out) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[i] = g2l[src_gid[i]];
}

// flags over all gids: owned by me and exported to q
__global__ void k_to_flags(int64_t n, const unsigned char* __restrict__ owner, int rank, int q,
                           const int* __restrict__ g2l, const unsigned* __restrict__ to_mask,
                           unsigned char* __restrict__ flag) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned char f = 0;
  if (owner[i] == rank) {
    int l = g2l[i];
    f = (to_mask[l] >> q) & 1u;
  }
  flag[i] = f;
}

__global__ void k_map_g2l(int n, const int* __restrict__ in_gid, const int* __restrict__ g2l, int* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[i] = g2l[in_gid[i]];
}

__global__ void k_row_sizes(int n, const int* __restrict__ rows, const int* __restrict__ ptr, int* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int r = rows[i];
  out[i] = ptr[r + 1] - ptr[r];
}

__global__ void k_expand_rows(int n, const int* __restrict__ rows, const int* __restrict__ ptr,
                              const int* __restrict__ scan, int* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int r = rows[i];
  int o = scan[i];
  for (int k = ptr[r]; k < ptr[r + 1]; k++) out[o++] = k;
}

// out-bond histogram by src local atom (owned bonds only)
__global__ void k_out_hist(int nb, const int* __restrict__ b_src, int* __restrict__ cnt) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nb) return;
  atomicAdd(&cnt[b_src[i]], 1);
}
__global__ void k_out_fill(int nb, const int* __restrict__ b_src, const int* __restrict__ out_ptr,
                           int* __restrict__ cursor, int* __restrict__ out_list) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nb) return;
  int s = b_src[i];
  int k = atomicAdd(&cursor[s], 1);
  out_list[out_ptr[s] + k] = i;
}
// deterministic order inside each out row (ascending bond id)
__global__ void k_out_sort(int n_loc, const int* __restrict__ out_ptr, int* __restrict__ out_list) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_loc) return;
  int b = out_ptr[c], e = out_ptr[c + 1];
  for (int i = b + 1; i < e; i++) {
    int v = out_list[i], j = i - 1;
    while (j >= b && out_list[j] > v) {
      out_list[j + 1] = out_list[j];
      j--;
    }
    out_list[j + 1] = v;
  }
}

// angles per centre: sum over out-bonds b=(c->x) of #in-bonds a=(s->c) with s != x (atom index)
__global__ void k_angle_count(int n_loc, const int* __restrict__ out_ptr, const int* __restrict__ out_list,
                              const int* __restrict__ brow_ptr, const int* __restrict__ b_src_gid,
                              const int* __restrict__ b_dst, const int* __restrict__ gid, int* __restrict__ cnt) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_loc) return;
  int n = 0;
  for (int o = out_ptr[c]; o < out_ptr[c + 1]; o++) {
    int b = out_list[o];
    int xg = gid[b_dst[b]];
    for (int a = brow_ptr[c]; a < brow_ptr[c + 1]; a++)
      if (b_src_gid[a] != xg) n++;
  }
  cnt[c] = n;
}
__global__ void k_angle_fill(int n_loc, const int* __restrict__ out_ptr, const int* __restrict__ out_list,
                             const int* __restrict__ brow_ptr, const int* __restrict__ b_src_gid,
                             const int* __restrict__ b_dst, const int* __restrict__ gid,
                             const int* __restrict__ ang_ptr, int* __restrict__ a_in, int* __restrict__ a_out,
                             int* __restrict__ a_ctr) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_loc) return;
  int k = ang_ptr[c];
  for (int o = out_ptr[c]; o < out_ptr[c + 1]; o++) {
    int b = out_list[o];
    int xg = gid[b_dst[b]];
    for (int a = brow_ptr[c]; a < brow_ptr[c + 1]; a++)
      if (b_src_gid[a] != xg) {
        a_in[k] = a;
        a_out[k] = b;
        a_ctr[k] = c;
        k++;
      }
  }
}

__global__ void k_key_hist(int64_t n, const unsigned char* k, int* c) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  atomicAdd(&c[k[i]], 1);
}
__global__ void k_add_offset(int n, const int* in, int off, int* out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = in[i] + off;
}

__global__ void k_fill_i(int64_t n, int* p, int v) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// ---------------------------------------------------------------------------------------------
// unfolded cell (heat flux)
struct UnfoldBox {
  double lat[9], inv[9];
  double lo[3], hi[3];  // admitted fractional range per axis
  int smin[3], smax[3];  // image shifts to try (0, 0 along non-periodic axes)
};

__global__ void k_unfold_frac(int64_t n, const double* __restrict__ cart, UnfoldBox b, double* __restrict__ frac) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int j = 0; j < 3; j++)
    frac[3 * i + j] = cart[3 * i] * b.inv[j] + cart[3 * i + 1] * b.inv[3 + j] + cart[3 * i + 2] * b.inv[6 + j];
}

__device__ __forceinline__ bool unfold_admits(const UnfoldBox& b, int k, double f, int s) {
  if (b.smin[k] == 0 && b.smax[k] == 0) return s == 0;  // non-periodic axis (or no room for an image)
  const double g = f + s;
  return g >= b.lo[k] && g <= b.hi[k];
}

// cnt[i] = number of images of atom i (shift s != 0 with every coordinate admitted)
__global__ void k_unfold_count(int64_t n, const double* __restrict__ frac, UnfoldBox b, int* __restrict__ cnt) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int c[3];
  for (int k = 0; k < 3; k++) {
    c[k] = 0;
    for (int s = b.smin[k]; s <= b.smax[k]; s++) c[k] += unfold_admits(b, k, frac[3 * i + k], s) ? 1 : 0;
  }
  cnt[i] = c[0] * c[1] * c[2] - 1;  // the atom itself (s = 0) is always admitted
}

// the cell atom at row i, its images at rows n + off[i] + (0, 1, ...) in (s0, s1, s2) lexicographic order
__global__ void k_unfold_fill(int64_t n, const double* __restrict__ cart0, const int* __restrict__ spec0,
                              const double* __restrict__ frac, const int* __restrict__ off, UnfoldBox b,
                              double* __restrict__ cart, int* __restrict__ spec, int* __restrict__ image_of) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double x = cart0[3 * i], y = cart0[3 * i + 1], z = cart0[3 * i + 2];
  const int sp = spec0[i];
  cart[3 * i] = x, cart[3 * i + 1] = y, cart[3 * i + 2] = z;
  spec[i] = sp, image_of[i] = (int)i;
  int64_t o = n + off[i];
  for (int s0 = b.smin[0]; s0 <= b.smax[0]; s0++) {
    if (!unfold_admits(b, 0, frac[3 * i], s0)) continue;
    for (int s1 = b.smin[1]; s1 <= b.smax[1]; s1++) {
      if (!unfold_admits(b, 1, frac[3 * i + 1], s1)) continue;
      for (int s2 = b.smin[2]; s2 <= b.smax[2]; s2++) {
        if (!unfold_admits(b, 2, frac[3 * i + 2], s2) || (s0 == 0 && s1 == 0 && s2 == 0)) continue;
        for (int m = 0; m < 3; m++)
          cart[3 * o + m] = (m == 0 ? x : m == 1 ? y : z) + s0 * b.lat[m] + s1 * b.lat[3 + m] + s2 * b.lat[6 + m];
        spec[o] = sp, image_of[o] = (int)i;
        o++;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
static void inv3(const double* m, double* o, double& det) {
  det = m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
  double id = 1.0 / det;
  o[0] = (m[4] * m[8] - m[5] * m[7]) * id;
  o[1] = (m[2] * m[7] - m[1] * m[8]) * id;
  o[2] = (m[1] * m[5] - m[2] * m[4]) * id;
  o[3] = (m[5] * m[6] - m[3] * m[8]) * id;
  o[4] = (m[0] * m[8] - m[2] * m[6]) * id;
  o[5] = (m[2] * m[3] - m[0] * m[5]) * id;
  o[6] = (m[3] * m[7] - m[4] * m[6]) * id;
  o[7] = (m[1] * m[6] - m[0] * m[7]) * id;
  o[8] = (m[0] * m[4] - m[1] * m[3]) * id;
}

template <class T>
static void excl_scan(DBuf<char>& tmp, const T* in, T* out, int64_t n, cudaStream_t st) {
  size_t bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, (int)n, st);
  tmp.ensure(bytes + 16);
  B2M_CK(cub::DeviceScan::ExclusiveSum(tmp.p, bytes, in, out, (int)n, st));
}

static int read_int(const int* dptr, cudaStream_t st) {
  int v;
  B2M_CK(cudaMemcpyAsync(&v, dptr, sizeof(int), cudaMemcpyDeviceToHost, st));
  B2M_CK(cudaStreamSynchronize(st));
  return v;
}

// Cell grid of one structure (cell edge >= r_cut where the cell allows it, at most 2^27 cells) from its inverse lattice,
// periodicity and, for the non-periodic axes, the fractional bounds fmn / fmx [3] of its wrapped atoms.  A structure gets
// the same grid alone and in a batch.
static void cell_grid(const double* inv, const int* pbc, const double* fmn, const double* fmx, double rcut,
                      GridParams& gp) {
  // perpendicular height along lattice vector k = 1 / |column k of inv|
  for (int k = 0; k < 3; k++) {
    double cn = sqrt(inv[k] * inv[k] + inv[3 + k] * inv[3 + k] + inv[6 + k] * inv[6 + k]);
    double height = 1.0 / cn;
    double reff = rcut + 1e-6;
    if (pbc[k]) {
      int n = (int)floor(height / reff);
      if (n < 1) n = 1;
      if (n > 1024) n = 1024;
      gp.nc[k] = n;
      double width = height / n;
      gp.reach[k] = (int)ceil(reff / width);
      if (gp.reach[k] < 1) gp.reach[k] = 1;
      B2M_REQUIRE(gp.reach[k] < 120, B2M_ERR_INVALID, "cell far too small for the cutoff");
    } else {
      double ext = (fmx[k] - fmn[k]);
      double extc = ext * height;
      int n = (int)floor(extc / reff);
      if (n < 1) n = 1;
      if (n > 1024) n = 1024;
      gp.nc[k] = n;
      gp.fmin[k] = fmn[k];
      gp.fscale[k] = ext > 0 ? n / ext : 0.0;
      gp.reach[k] = 1;
    }
  }
  while ((int64_t)gp.nc[0] * gp.nc[1] * gp.nc[2] > (1LL << 27)) {
    int kmax = 0;
    for (int k = 1; k < 3; k++)
      if (gp.nc[k] > gp.nc[kmax]) kmax = k;
    gp.nc[kmax] = (gp.nc[kmax] + 1) / 2;
    gp.reach[kmax] = 2 * gp.reach[kmax];  // conservative
  }
}

// Bounds of each structure s of the device offsets doff [S + 1]: lo / hi [S][6], the min / max of wc (k = 0..2) and of
// fracw (k = 3..5), from k_minmax over nb blocks per structure
static void bounds(cudaStream_t st, int S, int nb, const int64_t* doff, const double* wc, const double* fracw,
                   DBuf<double>& tmp, std::vector<double>& lo, std::vector<double>& hi) {
  tmp.ensure((size_t)S * nb * 12);
  launch(k_minmax, dim3(S, nb), 256, 0, st, doff, wc, fracw, tmp.p);
  std::vector<double> h((size_t)S * nb * 12);
  B2M_CK(cudaMemcpyAsync(h.data(), tmp.p, h.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2M_CK(cudaStreamSynchronize(st));
  lo.assign(6 * (size_t)S, 1e300);
  hi.assign(6 * (size_t)S, -1e300);
  for (size_t s = 0; s < (size_t)S; s++)
    for (size_t b = 0; b < (size_t)nb; b++)
      for (int k = 0; k < 6; k++) {
        lo[6 * s + k] = std::min(lo[6 * s + k], h[(s * nb + b) * 12 + k]);
        hi[6 * s + k] = std::max(hi[6 * s + k], h[(s * nb + b) * 12 + 6 + k]);
      }
}

// per-atom arrays for N atoms, positions and species uploaded (host staging, or the device arrays of an Unfold)
void Graph::upload(cudaStream_t st, const double* h_cart, const int32_t* h_species) {
  cart.ensure(3 * N);
  fracw.ensure(3 * N);
  wc.ensure(3 * N);
  corr.ensure(3 * N);
  species.ensure(N);
  owner.ensure(N);
  g2l.ensure(N);
  cell_of.ensure(N);
  s_gid.ensure(N);
  s_wc.ensure(3 * N);
  sidx_of_gid.ensure(N);
  tmp_i0.ensure(N + 1);
  tmp_i1.ensure(N + 1);
  tmp_i2.ensure(N + 1);
  tmp_i3.ensure(N + 1);
  tmp_flag.ensure(2 * N + 16);
  B2M_CK(cudaMemcpyAsync(cart.p, h_cart, 3 * N * sizeof(double), cudaMemcpyDefault, st));
  B2M_CK(cudaMemcpyAsync(species.p, h_species, N * sizeof(int), cudaMemcpyDefault, st));
}

// atoms sorted by cell (s_gid), cell_start; cell_of and the iota in tmp_i0 from k_owner_cell
void Graph::sort_by_cell(cudaStream_t st, int ncell) {
  cell_start.ensure(ncell + 2);
  tmp_i2.ensure(std::max<int64_t>(N + 1, ncell + 2));
  size_t bytes = 0;
  int bits = 1;
  while ((1 << bits) < ncell + 1) bits++;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, cell_of.p, tmp_i1.p, tmp_i0.p, s_gid.p, (int)N, 0, bits, st);
  cub_tmp.ensure(bytes + 16);
  B2M_CK(cub::DeviceRadixSort::SortPairs(cub_tmp.p, bytes, cell_of.p, tmp_i1.p, tmp_i0.p, s_gid.p, (int)N, 0,
                                         bits, st));
  // tmp_i1 = sorted cell ids
  B2M_CK(cudaMemsetAsync(tmp_i2.p, 0, (ncell + 1) * sizeof(int), st));
  launch(k_cell_hist, cdiv(N, 256), 256, 0, st, N, tmp_i1.p, tmp_i2.p);
  excl_scan(cub_tmp, tmp_i2.p, cell_start.p, ncell + 1, st);
}

// Every build (DESIGN.md §12): each structure wrapped in its own lattice and given its own cell grid by cell_grid(); cell
// ids are the structure's first cell + its local cell, so the radix sort groups the atoms by structure, then by cell,
// and inside a structure reproduces the order of its build alone.  Launches and host synchronisations do not depend on
// the number of structures.
void Graph::build(cudaStream_t st, int nstruct, const int64_t* natoms, const double* h_cart, const double* h_lat,
                  const int32_t* h_species, const int* h_pbc, double rcut, double rbond, double tol_, int rank_,
                  int world_, bool as_batch) {
  B2M_REQUIRE(nstruct >= 1 && (as_batch || nstruct == 1), B2M_ERR_INVALID, "a batch needs at least one structure");
  B2M_REQUIRE(world_ >= 1 && world_ <= MAXP, B2M_ERR_PARTITIONS, "num_partitions must be in [1,16]");
  B2M_REQUIRE(!as_batch || world_ == 1, B2M_ERR_PARTITIONS, "a batch runs on one partition");
  B2M_REQUIRE(rbond <= rcut, B2M_ERR_INVALID, "bond_r cannot be greater than regular cutoff");
  auto named = [&](int s, const std::string& what) { return as_batch ? structure_name(s) + ": " + what : what; };
  std::vector<int64_t> off(nstruct + 1, 0);
  std::vector<GridParams> gps(nstruct);
  std::vector<double> vol(nstruct);
  for (int s = 0; s < nstruct; s++) {
    B2M_REQUIRE(natoms[s] > 0, B2M_ERR_INVALID, as_batch ? named(s, "no atoms") : "natoms out of range");
    off[s + 1] = off[s] + natoms[s];
    B2M_REQUIRE(off[s + 1] < (1LL << 31) / 4, B2M_ERR_INVALID,
                as_batch ? "batch has too many atoms" : "natoms out of range");
    GridParams& gp = gps[s];
    for (int k = 0; k < 3; k++) {
      const int f = h_pbc[3 * s + k];
      B2M_REQUIRE(!as_batch || f == 0 || f == 1, B2M_ERR_INVALID, named(s, "pbc flags must be 0 or 1"));
      gp.pbc[k] = f ? 1 : 0, gp.nc[k] = 1, gp.reach[k] = 1, gp.fmin[k] = 0, gp.fscale[k] = 0;
    }
    memcpy(gp.lat, h_lat + 9 * s, sizeof gp.lat);
    double det;
    inv3(gp.lat, gp.inv, det);
    B2M_REQUIRE(fabs(det) > 1e-12, B2M_ERR_INVALID, named(s, "singular lattice"));
    vol[s] = fabs(det);
  }
  S = nstruct;
  batch = as_batch;
  N = off[S];
  rank = rank_;
  world = world_;
  r_cut = rcut;
  r_bond = rbond;
  tol = tol_;
  b_off = off;
  volume = vol;
  grids = gps;

  // ---- upload + wrap: the lattices of the grids now, the cell grids after the bounds ----
  b_doff.ensure(S + 1);
  B2M_CK(cudaMemcpyAsync(b_doff.p, off.data(), (S + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  upload(st, h_cart, h_species);
  if (batch) {
    std::vector<int> sid(N);
    for (int s = 0; s < S; s++) std::fill(sid.begin() + off[s], sid.begin() + off[s + 1], s);
    b_gp.ensure(S);
    b_cell_off.ensure(S);
    b_sid.ensure(N);
    B2M_CK(cudaMemcpyAsync(b_sid.p, sid.data(), N * sizeof(int), cudaMemcpyHostToDevice, st));
    B2M_CK(cudaMemcpyAsync(b_gp.p, grids.data(), S * sizeof(GridParams), cudaMemcpyHostToDevice, st));
  }
  with_grid([&](auto grid) {
    launch(k_wrap<decltype(grid)>, cdiv(N, 256), 256, 0, st, N, cart.p, grid, fracw.p, wc.p, corr.p);
  });

  // ---- bounds of every structure (partition axis, walls, non-periodic cell grid): 256 blocks for one structure, one
  // block each in a batch ----
  std::vector<double> mn, mx;
  bounds(st, S, batch ? 1 : 256, b_doff.p, wc.p, fracw.p, red_tmp, mn, mx);

  // ---- cell grids and the first cell of every structure; they do not depend on the walls ----
  std::vector<int> coff(S);
  int64_t ncell = 0;
  for (int s = 0; s < S; s++) {
    try {
      cell_grid(grids[s].inv, grids[s].pbc, &mn[6 * s + 3], &mx[6 * s + 3], rcut, grids[s]);
    } catch (const Error& ex) {
      throw Error(ex.code, named(s, ex.what()));
    }
    coff[s] = (int)ncell;
    ncell += (int64_t)grids[s].nc[0] * grids[s].nc[1] * grids[s].nc[2];
    B2M_REQUIRE(ncell <= (1LL << 27), B2M_ERR_INVALID, "batch needs more than 2^27 cells; split it");
  }
  if (batch) {
    B2M_CK(cudaMemcpyAsync(b_gp.p, grids.data(), S * sizeof(GridParams), cudaMemcpyHostToDevice, st));
    B2M_CK(cudaMemcpyAsync(b_cell_off.p, coff.data(), S * sizeof(int), cudaMemcpyHostToDevice, st));
  }
  const double r2 = rcut * rcut, rb2 = rbond * rbond;

  Walls wl;
  wl.nw = world - 1;
  wl.axis = 0;
  if (world > 1) {  // one structure
    const GridParams& gp = grids[0];
    // create_partition (:1370-1456)
    double diffs[3] = {mx[0] - mn[0], mx[1] - mn[1], mx[2] - mn[2]};
    int longest = 0;
    for (int i = 1; i < 3; i++)
      if (diffs[i] > diffs[longest]) longest = i;
    double fmn = mn[3 + longest], fmx = mx[3 + longest];
    double flen = fmx - fmn;
    wl.axis = longest;
    if (!balanced) {
      for (int i = 1; i < world; i++) wl.w[i - 1] = (i * (flen / world)) + kEpsilon + fmn;
    } else {
      // balanced (DESIGN.md §4.1): the work of every atom from a count pass over all of them (cell ids do not depend
      // on the walls, so the cell list is built first), then walls at the work quantiles
      Walls none = wl;
      none.nw = 0;
      launch(k_owner_cell<OneGrid>, cdiv(N, 256), 256, 0, st, N, fracw.p, none, OneGrid{gp}, owner.p, cell_of.p,
             tmp_i0.p);
      sort_by_cell(st, (int)ncell);
      tmp_i3.ensure(N + 1);
      launch(k_post_sort, cdiv(N, 256), 256, 0, st, N, s_gid.p, wc.p, owner.p, rank, s_wc.p, sidx_of_gid.p, tmp_i3.p);
      // tmp_i0 still holds the iota: every sorted index is a centre
      launch(k_count<OneGrid>, cdiv(N, 256), 256, 0, st, (int)N, tmp_i0.p, OneGrid{gp}, s_gid.p, s_wc.p, cell_start.p,
             fracw.p, owner.p, rank, r2, rb2, tol, tmp_i1.p, tmp_i2.p, (unsigned*)nullptr);
      bal_x.ensure(2 * N);
      bal_w.ensure(2 * N);
      double *x_in = bal_x.p, *x_s = bal_x.p + N;
      long long *w_in = bal_w.p, *w_s = bal_w.p + N;
      launch(k_work_keys, cdiv(N, 256), 256, 0, st, N, s_gid.p, fracw.p, longest, tmp_i1.p, tmp_i2.p, x_in, w_in);
      size_t bytes = 0;
      cub::DeviceRadixSort::SortPairs(nullptr, bytes, x_in, x_s, w_in, w_s, (int)N, 0, 64, st);
      cub_tmp.ensure(bytes + 16);
      B2M_CK(cub::DeviceRadixSort::SortPairs(cub_tmp.p, bytes, x_in, x_s, w_in, w_s, (int)N, 0, 64, st));
      bytes = 0;
      cub::DeviceScan::InclusiveSum(nullptr, bytes, w_s, w_in, (int)N, st);
      cub_tmp.ensure(bytes + 16);
      B2M_CK(cub::DeviceScan::InclusiveSum(cub_tmp.p, bytes, w_s, w_in, (int)N, st));
      launch(k_balanced_gaps, 1, 32, 0, st, wl.nw, N, world, x_s, w_in, red_tmp.p);
      double gap[2 * MAXP];
      B2M_CK(cudaMemcpyAsync(gap, red_tmp.p, 2 * wl.nw * sizeof(double), cudaMemcpyDeviceToHost, st));
      B2M_CK(cudaStreamSynchronize(st));
      for (int k = 0; k < wl.nw; k++) wl.w[k] = 0.5 * (gap[2 * k] + gap[2 * k + 1]);
      // minimum slab width delta = need / h, h the cell's height across the partition axis (stricter than the lattice
      // column for a tilted cell); forward then backward pass against the end bounds
      const double need = 2 * (rcut + rbond);
      const double h = 1.0 / sqrt(gp.inv[longest] * gp.inv[longest] + gp.inv[3 + longest] * gp.inv[3 + longest] +
                                  gp.inv[6 + longest] * gp.inv[6 + longest]);
      const double delta = need / h;
      const bool from_min = walls_from_min || !gp.pbc[longest];
      const double lo = from_min ? fmn : 0.0, hi = from_min ? fmx : 1.0;
      for (int k = 0; k < wl.nw; k++) wl.w[k] = std::max(wl.w[k], (k ? wl.w[k - 1] : lo) + delta);
      for (int k = wl.nw - 1; k >= 0; k--) wl.w[k] = std::min(wl.w[k], (k + 1 < wl.nw ? wl.w[k + 1] : hi) - delta);
      for (int k = 0; k <= wl.nw; k++) {
        const double width = (k < wl.nw ? wl.w[k] : hi) - (k ? wl.w[k - 1] : lo);
        if (width < delta * (1 - 1e-12)) {  // slack for the rounding of the two passes
          char buf[256];
          snprintf(buf, sizeof buf,
                   "Balanced partition: slab %d is %.4f A wide across the walls < 2*(atom_cutoff+bond_cutoff) = %.4f; "
                   "reduce the number of partitions",
                   k, width * h, need);
          throw Error(B2M_ERR_SLAB_WIDTH, buf);
        }
      }
    }
    // collision nudge
    for (int iter = 0; iter < 64; iter++) {
      B2M_CK(cudaMemsetAsync(tmp_i0.p, 0, MAXP * sizeof(int), st));
      launch(k_wall_collisions, cdiv(N, 256), 256, 0, st, N, fracw.p, wl, tmp_i0.p);
      int hits[MAXP];
      B2M_CK(cudaMemcpyAsync(hits, tmp_i0.p, MAXP * sizeof(int), cudaMemcpyDeviceToHost, st));
      B2M_CK(cudaStreamSynchronize(st));
      bool any = false;
      for (int k = 0; k < wl.nw; k++)
        if (hits[k]) {
          wl.w[k] += kEpsilon;
          any = true;
        }
      if (!any) break;
    }
    if (!balanced) {
      // check_partition_size (:1512-1529): lattice *column* of the axis, width = walls[0] * |col|
      double col[3] = {gp.lat[longest], gp.lat[longest + 3], gp.lat[longest + 6]};
      double width = (wl.w[0] - (walls_from_min ? fmn : 0.0)) * sqrt(col[0] * col[0] + col[1] * col[1] + col[2] * col[2]);
      double need = 2 * (rcut + rbond);
      if (width <= need) {
        char buf[256];
        snprintf(buf, sizeof buf,
                 "Partition walls are too close together: slab width %.4f <= 2*(atom_cutoff+bond_cutoff) = %.4f; "
                 "reduce the number of partitions",
                 width, need);
        throw Error(B2M_ERR_SLAB_WIDTH, buf);
      }
    }
  }
  axis = wl.axis;
  for (int k = 0; k < MAXP; k++) walls[k] = k < wl.nw ? wl.w[k] : 0.0;

  // ---- owner + cell id, sort by cell (a balanced partition sorted the atoms by cell before placing its walls) ----
  with_grid([&](auto grid) {
    launch(k_owner_cell<decltype(grid)>, cdiv(N, 256), 256, 0, st, N, fracw.p, wl, grid, owner.p, cell_of.p, tmp_i0.p);
  });
  if (!(balanced && world > 1)) sort_by_cell(st, (int)ncell);
  build_rows(st);
}

// Local atoms, edges, halo sections, bonds and angles of the atoms sorted by cell (every build ends here)
void Graph::build_rows(cudaStream_t st) {
  const double r2 = r_cut * r_cut, rb2 = r_bond * r_bond;
  // own flags, scan -> local ids
  launch(k_post_sort, cdiv(N, 256), 256, 0, st, N, s_gid.p, wc.p, owner.p, rank, s_wc.p, sidx_of_gid.p, tmp_i0.p);
  tmp_i3.ensure(N + 1);
  B2M_CK(cudaMemsetAsync(tmp_i0.p + N, 0, sizeof(int), st));
  excl_scan(cub_tmp, tmp_i0.p, tmp_i3.p, N + 1, st);
  n_own = read_int(tmp_i3.p + N, st);
  B2M_REQUIRE(n_own > 0, B2M_ERR_INVALID, "a partition owns no atoms");

  // local arrays sized for the worst case n_loc <= N (halo count known later); use N bound lazily
  gid.ensure(N);
  type.ensure(N);
  loc_sidx.ensure(N);
  to_mask.ensure(n_own);
  launch(k_assign_owned, cdiv(N, 256), 256, 0, st, N, s_gid.p, tmp_i0.p, tmp_i3.p, species.p, gid.p, type.p, loc_sidx.p,
         g2l.p);

  // ---- count pass over owned rows ----
  row_ptr.ensure(n_own + 2);
  DBuf<int>& cnt_e = tmp_i0;
  DBuf<int>& cnt_b = tmp_i1;
  with_grid([&](auto grid) {
    launch(k_count<decltype(grid)>, cdiv(n_own, 256), 256, 0, st, n_own, loc_sidx.p, grid, s_gid.p, s_wc.p,
           cell_start.p, fracw.p, owner.p, rank, r2, rb2, tol, cnt_e.p, cnt_b.p, to_mask.p);
  });
  B2M_CK(cudaMemsetAsync(cnt_e.p + n_own, 0, sizeof(int), st));
  B2M_CK(cudaMemsetAsync(cnt_b.p + n_own, 0, sizeof(int), st));
  excl_scan(cub_tmp, cnt_e.p, row_ptr.p, n_own + 1, st);
  // owned part of brow_ptr (halo part appended later); brow_ptr sized for n_loc+1 <= N+1
  brow_ptr.ensure(N + 2);
  excl_scan(cub_tmp, cnt_b.p, brow_ptr.p, n_own + 1, st);
  // batch: the rows of structure s are b_off[s] .. b_off[s + 1] - 1 (every atom owned, cell ids grouped by structure)
  std::vector<int> e_at(S + 1);
  if (batch) {
    sel_out.ensure(S + 1);
    launch(k_gather_at, cdiv(S + 1, 256), 256, 0, st, S + 1, b_doff.p, row_ptr.p, sel_out.p);
    B2M_CK(cudaMemcpyAsync(e_at.data(), sel_out.p, (S + 1) * sizeof(int), cudaMemcpyDeviceToHost, st));
  }
  E = read_int(row_ptr.p + n_own, st);
  B_own = read_int(brow_ptr.p + n_own, st);
  B2M_REQUIRE(E > 0, B2M_ERR_INVALID, "No neighbors were found!");
  for (int s = 0; batch && s < S; s++)
    B2M_REQUIRE(e_at[s + 1] > e_at[s], B2M_ERR_INVALID,
                structure_name(s) + " has no edges (No neighbors were found!)");

  e_src.ensure(E);
  e_dst.ensure(E);
  e_img.ensure(E);
  e_bond.ensure(E);
  e_vec.ensure(E);
  e_src_gid.ensure(E);
  // bond arrays: owned now, grown (copy-preserving) when the halo count is known
  const int bond_cap_guess = B_own + B_own / 2 + 1024;
  b_src_gid.ensure(bond_cap_guess);
  b_src.ensure(bond_cap_guess);
  b_dst.ensure(bond_cap_guess);
  b_img.ensure(bond_cap_guess);
  b_vec.ensure(bond_cap_guess);
  b_edge.ensure(B_own + 1);
  unsigned char* halo_flag = tmp_flag.p;
  B2M_CK(cudaMemsetAsync(halo_flag, 0, N, st));
  with_grid([&](auto grid) {
    launch(k_fill_owned<decltype(grid)>, cdiv(n_own, 256), 256, 0, st, n_own, loc_sidx.p, grid, s_gid.p, s_wc.p,
           cell_start.p, fracw.p, owner.p, rank, r2, rb2, tol, row_ptr.p, brow_ptr.p, e_src_gid.p, e_dst.p, e_img.p,
           e_bond.p, e_vec.p, b_src_gid.p, b_dst.p, b_img.p, b_edge.p, b_vec.p, halo_flag);
  });

  // ---- halo atoms: grouped by owner, gid ascending ----
  n_halo = 0;
  for (int q = 0; q <= MAXP; q++) from_off[q] = 0;
  for (int q = 0; q < MAXP; q++) n_from[q] = n_to[q] = nb_from[q] = nb_to[q] = 0;
  if (world > 1) {
    unsigned char* keys = tmp_flag.p + N;
    launch(k_halo_keys, cdiv(N, 256), 256, 0, st, N, halo_flag, owner.p, world, keys, tmp_i0.p);
    // sort (key, gid): stable radix sort keeps gid ascending inside each key
    keys_out.ensure(N);
    size_t bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, bytes, keys, keys_out.p, tmp_i0.p, tmp_i1.p, (int)N, 0, 8, st);
    cub_tmp.ensure(bytes + 16);
    B2M_CK(cub::DeviceRadixSort::SortPairs(cub_tmp.p, bytes, keys, keys_out.p, tmp_i0.p, tmp_i1.p, (int)N, 0, 8, st));
    // section sizes: histogram of the sorted keys
    B2M_CK(cudaMemsetAsync(tmp_i2.p, 0, (MAXP + 2) * sizeof(int), st));
    launch(k_key_hist, cdiv(N, 256), 256, 0, st, N, keys_out.p, tmp_i2.p);
    int hc[MAXP + 2];
    B2M_CK(cudaMemcpyAsync(hc, tmp_i2.p, (MAXP + 2) * sizeof(int), cudaMemcpyDeviceToHost, st));
    B2M_CK(cudaStreamSynchronize(st));
    int off = 0;
    for (int q = 0; q < world; q++) {
      n_from[q] = hc[q];
      from_off[q] = off;
      off += hc[q];
    }
    for (int q = world; q <= MAXP; q++) from_off[q] = off;
    n_halo = off;
    launch(k_assign_halo, cdiv(n_halo, 256), 256, 0, st, n_halo, n_own, tmp_i1.p, species.p, sidx_of_gid.p, gid.p,
           type.p, loc_sidx.p, g2l.p);
  }
  n_loc = n_own + n_halo;
  launch(k_relabel, cdiv(E, 256), 256, 0, st, E, e_src_gid.p, g2l.p, e_src.p);

  // ---- halo bonds ----
  B_halo = 0;
  if (n_halo > 0) {
    DBuf<int>& hb_cnt = tmp_i0;
    launch(k_count<OneGrid>, cdiv(n_halo, 256), 256, 0, st, n_halo, loc_sidx.p + n_own, OneGrid{grids[0]}, s_gid.p,
           s_wc.p, cell_start.p, fracw.p, owner.p, rank, rb2, rb2, tol, (int*)nullptr, hb_cnt.p, (unsigned*)nullptr);
    B2M_CK(cudaMemsetAsync(hb_cnt.p + n_halo, 0, sizeof(int), st));
    excl_scan(cub_tmp, hb_cnt.p, tmp_i1.p, n_halo + 1, st);
    B_halo = read_int(tmp_i1.p + n_halo, st);
    // brow_ptr[n_own + h] = B_own + scan[h]
    launch(k_add_offset, cdiv(n_halo + 1, 256), 256, 0, st, n_halo + 1, tmp_i1.p, B_own, brow_ptr.p + n_own);
  }
  B_loc = B_own + B_halo;
  if ((size_t)B_loc > b_src_gid.cap) {
    // grow preserving the owned part
    auto grow_i = [&](DBuf<int>& b) {
      DBuf<int> nb;
      nb.ensure(B_loc);
      B2M_CK(cudaMemcpyAsync(nb.p, b.p, B_own * sizeof(int), cudaMemcpyDeviceToDevice, st));
      B2M_CK(cudaStreamSynchronize(st));
      std::swap(nb.p, b.p);
      std::swap(nb.cap, b.cap);
    };
    grow_i(b_src_gid);
    grow_i(b_src);
    grow_i(b_dst);
    grow_i(b_img);
    DBuf<float4> nv;
    nv.ensure(B_loc);
    B2M_CK(cudaMemcpyAsync(nv.p, b_vec.p, B_own * sizeof(float4), cudaMemcpyDeviceToDevice, st));
    B2M_CK(cudaStreamSynchronize(st));
    std::swap(nv.p, b_vec.p);
    std::swap(nv.cap, b_vec.cap);
  }
  if (n_halo > 0)
    launch(k_fill_halo_bonds, cdiv(n_halo, 256), 256, 0, st, n_halo, n_own, loc_sidx.p + n_own, grids[0], s_gid.p,
           s_wc.p, cell_start.p, fracw.p, rb2, tol, brow_ptr.p, b_src_gid.p, b_dst.p, b_img.p, b_vec.p);
  launch(k_relabel, cdiv(B_loc, 256), 256, 0, st, (int64_t)B_loc, b_src_gid.p, g2l.p, b_src.p);
  for (int q = 0; q <= MAXP; q++) bfrom_off[q] = 0;
  if (n_halo > 0) {
    // bond halo sections follow the atom halo sections
    std::vector<int> hptr(world + 1);
    for (int q = 0; q <= world; q++) {
      int idx = n_own + (q < world ? from_off[q] : n_halo);
      B2M_CK(cudaMemcpyAsync(&hptr[q], brow_ptr.p + idx, sizeof(int), cudaMemcpyDeviceToHost, st));
    }
    B2M_CK(cudaStreamSynchronize(st));
    for (int q = 0; q < world; q++) {
      bfrom_off[q] = hptr[q] - B_own;
      nb_from[q] = hptr[q + 1] - hptr[q];
    }
    for (int q = world; q <= MAXP; q++) bfrom_off[q] = B_halo;
  }

  // ---- to-lists (atoms, then their bond rows) ----
  for (int q = 0; q <= MAXP; q++) to_off[q] = bto_off[q] = 0;
  if (world > 1) {
    to_list.ensure(n_own + 1);
    int off = 0;
    sel_out.ensure(N);
    nsel.ensure(4);
    for (int q = 0; q < world; q++) {
      to_off[q] = off;
      if (q == rank) continue;
      unsigned char* flag = tmp_flag.p;  // halo_flag no longer needed
      launch(k_to_flags, cdiv(N, 256), 256, 0, st, N, owner.p, rank, q, g2l.p, to_mask.p, flag);
      size_t bytes = 0;
      cub::CountingInputIterator<int> it(0);
      cub::DeviceSelect::Flagged(nullptr, bytes, it, flag, sel_out.p, nsel.p, (int)N, st);
      cub_tmp.ensure(bytes + 16);
      B2M_CK(cub::DeviceSelect::Flagged(cub_tmp.p, bytes, it, flag, sel_out.p, nsel.p, (int)N, st));
      int cnt = read_int(nsel.p, st);
      n_to[q] = cnt;
      if (cnt > 0) launch(k_map_g2l, cdiv(cnt, 256), 256, 0, st, cnt, sel_out.p, g2l.p, to_list.p + off);
      off += cnt;
    }
    for (int q = world; q <= MAXP; q++) to_off[q] = off;
    // bond to-lists: bond rows of the to atoms
    int boff = 0;
    bto_list.ensure(B_own + 1);
    for (int q = 0; q < world; q++) {
      bto_off[q] = boff;
      int cnt = n_to[q];
      if (cnt == 0) continue;
      launch(k_row_sizes, cdiv(cnt, 256), 256, 0, st, cnt, to_list.p + to_off[q], brow_ptr.p, tmp_i0.p);
      B2M_CK(cudaMemsetAsync(tmp_i0.p + cnt, 0, sizeof(int), st));
      excl_scan(cub_tmp, tmp_i0.p, tmp_i1.p, cnt + 1, st);
      int tot = read_int(tmp_i1.p + cnt, st);
      nb_to[q] = tot;
      launch(k_expand_rows, cdiv(cnt, 256), 256, 0, st, cnt, to_list.p + to_off[q], brow_ptr.p, tmp_i1.p,
             bto_list.p + boff);
      boff += tot;
    }
    for (int q = world; q <= MAXP; q++) bto_off[q] = boff;
  }

  // ---- out-bonds by src, angles grouped by centre ----
  out_ptr.ensure(n_loc + 2);
  out_list.ensure(B_own + 1);
  {
    DBuf<int>& ocnt = tmp_i0;
    B2M_CK(cudaMemsetAsync(ocnt.p, 0, (n_loc + 1) * sizeof(int), st));
    launch(k_out_hist, cdiv(B_own, 256), 256, 0, st, B_own, b_src.p, ocnt.p);
    excl_scan(cub_tmp, ocnt.p, out_ptr.p, n_loc + 1, st);
    B2M_CK(cudaMemsetAsync(tmp_i1.p, 0, (n_loc + 1) * sizeof(int), st));
    launch(k_out_fill, cdiv(B_own, 256), 256, 0, st, B_own, b_src.p, out_ptr.p, tmp_i1.p, out_list.p);
    launch(k_out_sort, cdiv(n_loc, 256), 256, 0, st, n_loc, out_ptr.p, out_list.p);
    DBuf<int>& acnt = tmp_i2;
    acnt.ensure(n_loc + 2);
    launch(k_angle_count, cdiv(n_loc, 256), 256, 0, st, n_loc, out_ptr.p, out_list.p, brow_ptr.p, b_src_gid.p, b_dst.p,
           gid.p, acnt.p);
    B2M_CK(cudaMemsetAsync(acnt.p + n_loc, 0, sizeof(int), st));
    tmp_i3.ensure(n_loc + 2);
    excl_scan(cub_tmp, acnt.p, tmp_i3.p, n_loc + 1, st);
    A = read_int(tmp_i3.p + n_loc, st);
    a_in.ensure(A + 1);
    a_out.ensure(A + 1);
    a_ctr.ensure(A + 1);
    launch(k_angle_fill, cdiv(n_loc, 256), 256, 0, st, n_loc, out_ptr.p, out_list.p, brow_ptr.p, b_src_gid.p, b_dst.p,
           gid.p, tmp_i3.p, a_in.p, a_out.p, a_ctr.p);
  }
  B2M_CK(cudaStreamSynchronize(st));
}

// ---------------------------------------------------------------------------------------------
template <class T>
static std::vector<T> d2h(const T* p, size_t n, cudaStream_t st) {
  std::vector<T> v(n);
  if (n) B2M_CK(cudaMemcpyAsync(v.data(), p, n * sizeof(T), cudaMemcpyDeviceToHost, st));
  B2M_CK(cudaStreamSynchronize(st));
  return v;
}

int64_t Graph::export_info(cudaStream_t st, int which, int64_t* out, int64_t cap) {
  auto need = [&](int64_t n) { B2M_REQUIRE(n <= cap, B2M_ERR_INVALID, "export buffer too small"); };
  std::vector<int> hgid = d2h(gid.p, n_loc, st);
  std::vector<int> hcorr;
  auto off_of = [&](int img, int src_g, int dst_g, int64_t* o) {
    // reference offset (unwrapped frame): off = -img - corr[dst] + corr[src]   (see DESIGN.md)
    int ix, iy, iz;
    unpack_img(img, ix, iy, iz);
    o[0] = -ix - hcorr[3 * dst_g] + hcorr[3 * src_g];
    o[1] = -iy - hcorr[3 * dst_g + 1] + hcorr[3 * src_g + 1];
    o[2] = -iz - hcorr[3 * dst_g + 2] + hcorr[3 * src_g + 2];
  };
  switch (which) {
    case 0:
      need(n_own);
      for (int i = 0; i < n_own; i++) out[i] = hgid[i];
      return n_own;
    case 1:
      need(n_halo);
      for (int i = 0; i < n_halo; i++) out[i] = hgid[n_own + i];
      return n_halo;
    case 2: {
      need(n_halo);
      for (int q = 0; q < world; q++)
        for (int i = 0; i < n_from[q]; i++) out[from_off[q] + i] = q;
      return n_halo;
    }
    case 3: {
      need(E * 5);
      hcorr = d2h(corr.p, 3 * N, st);
      auto s = d2h(e_src.p, E, st);
      auto d = d2h(e_dst.p, E, st);
      auto im = d2h(e_img.p, E, st);
      for (int64_t e = 0; e < E; e++) {
        int sg = hgid[s[e]], dg = hgid[d[e]];
        out[5 * e] = sg;
        out[5 * e + 1] = dg;
        off_of(im[e], sg, dg, out + 5 * e + 2);
      }
      return E * 5;
    }
    case 4: {
      need((int64_t)B_loc * 5);
      hcorr = d2h(corr.p, 3 * N, st);
      auto s = d2h(b_src_gid.p, B_loc, st);
      auto d = d2h(b_dst.p, B_loc, st);
      auto im = d2h(b_img.p, B_loc, st);
      for (int b = 0; b < B_loc; b++) {
        int sg = s[b], dg = hgid[d[b]];
        out[5 * b] = sg;
        out[5 * b + 1] = dg;
        off_of(im[b], sg, dg, out + 5 * b + 2);
      }
      return (int64_t)B_loc * 5;
    }
    case 5: {
      need(A * 3);
      auto ai = d2h(a_in.p, A, st);
      auto ao = d2h(a_out.p, A, st);
      auto ac = d2h(a_ctr.p, A, st);
      for (int64_t a = 0; a < A; a++) {
        out[3 * a] = ai[a];
        out[3 * a + 1] = ao[a];
        out[3 * a + 2] = hgid[ac[a]];
      }
      return A * 3;
    }
    case 6: {
      int tot = to_off[world];
      need(2 * (int64_t)tot);
      auto tl = d2h(to_list.p, tot, st);
      int k = 0;
      for (int q = 0; q < world; q++)
        for (int i = 0; i < n_to[q]; i++) {
          out[2 * k] = q;
          out[2 * k + 1] = hgid[tl[to_off[q] + i]];
          k++;
        }
      return 2 * (int64_t)tot;
    }
    case 7: {
      need(world - 1);
      for (int k = 0; k < world - 1; k++) memcpy(&out[k], &walls[k], 8);
      return world - 1;
    }
    default:
      throw Error(B2M_ERR_INVALID, "unknown partition-info selector");
  }
}

void Unfold::build(cudaStream_t st, int64_t natoms, const double* h_cart, const int32_t* h_species,
                   const double* h_lat, const int* h_pbc, double reach) {
  B2M_REQUIRE(natoms > 0 && natoms < (1LL << 31) / 4, B2M_ERR_INVALID, "natoms out of range");
  B2M_REQUIRE(reach > 0, B2M_ERR_INVALID, "heat-flux reach must be > 0");
  n = natoms;
  UnfoldBox b;
  double det;
  memcpy(b.lat, h_lat, sizeof b.lat);
  inv3(b.lat, b.inv, det);
  B2M_REQUIRE(fabs(det) > 1e-12, B2M_ERR_INVALID, "singular lattice");
  cart0.ensure(3 * n);
  frac0.ensure(3 * n);
  species0.ensure(n);
  cnt.ensure(n + 1);
  off.ensure(n + 1);
  dseg.ensure(2);
  B2M_CK(cudaMemcpyAsync(cart0.p, h_cart, 3 * n * sizeof(double), cudaMemcpyDefault, st));
  B2M_CK(cudaMemcpyAsync(species0.p, h_species, n * sizeof(int), cudaMemcpyDefault, st));
  launch(k_unfold_frac, cdiv(n, 256), 256, 0, st, n, cart0.p, b, frac0.p);
  // fractional bounding box of the cell atoms (the Cartesian half of the bounds reads the positions and is not used)
  const int64_t seg[2] = {0, n};
  B2M_CK(cudaMemcpyAsync(dseg.p, seg, sizeof seg, cudaMemcpyHostToDevice, st));
  std::vector<double> mn, mx;
  bounds(st, 1, 256, dseg.p, cart0.p, frac0.p, red_tmp, mn, mx);
  for (int k = 0; k < 3; k++) {
    const double fmn = mn[3 + k], fmx = mx[3 + k];
    b.smin[k] = b.smax[k] = 0;
    b.lo[k] = fmn, b.hi[k] = fmx;
    if (h_pbc[k]) {
      // reach / h_k in fractional units: |column k of inv| = 1 / h_k
      const double pad = reach * sqrt(b.inv[k] * b.inv[k] + b.inv[3 + k] * b.inv[3 + k] + b.inv[6 + k] * b.inv[6 + k]);
      b.lo[k] = fmn - pad, b.hi[k] = fmx + pad;
      b.smin[k] = (int)ceil(b.lo[k] - fmx), b.smax[k] = (int)floor(b.hi[k] - fmn);
      B2M_REQUIRE(b.smax[k] - b.smin[k] < 4096, B2M_ERR_INVALID, "heat-flux reach far larger than the cell");
    }
  }
  launch(k_unfold_count, cdiv(n, 256), 256, 0, st, n, frac0.p, b, cnt.p);
  B2M_CK(cudaMemsetAsync(cnt.p + n, 0, sizeof(int), st));
  excl_scan(cub_tmp, cnt.p, off.p, n + 1, st);
  const int64_t n_img = read_int(off.p + n, st);
  N = n + n_img;
  B2M_REQUIRE(N < (1LL << 31) / 4, B2M_ERR_INVALID, "unfolded cell too large");
  cart.ensure(3 * N);
  species.ensure(N);
  image_of.ensure(N);
  launch(k_unfold_fill, cdiv(n, 256), 256, 0, st, n, cart0.p, species0.p, frac0.p, off.p, b, cart.p, species.p,
         image_of.p);
}

}  // namespace b2m
