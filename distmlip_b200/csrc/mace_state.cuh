// mace_state.cuh -- kernels (kernels_mace.cu), weights and workspace of the MACE path (engine_mace.inl).
// Layouts: node features h [n][C], or [n][4][C] (0e, then 1o m = 0..2) for 0e+1o layers, so that a halo row is one
// contiguous span; the l-resolved atom basis A [nsh][n_own][C] (lm-major, so that the rows of one l form one contiguous
// [(2l+1) n_own][C] block for the per-l channel mixes); edge quantities [E][...].
#pragma once
#include <array>
#include <vector>

#include "kernels.cuh"

namespace b2m {

constexpr int kMaceMaxLayers = 8;
constexpr int kMaceMaxNsh = 16;  // max_ell <= 3

struct MaceRadial {
  int nb;       // Bessel functions in use
  int nbp;      // row pitch of the basis buffers (64, padding columns zero)
  int p;        // polynomial cutoff exponent
  float r_max;
  float pref;   // sqrt(2 / r_max)
  float w[64];  // Bessel frequencies
};

// ZBL pair repulsion (mace's ZBLBasis) and the Agnesi distance transform (AgnesiTransform), tests/mace_zbl_ref.py; each
// is on when its state_dict keys are loaded (DESIGN §11.2)
struct MaceCore {
  const float4* elem = nullptr;  // [n_elem]: (Z, Z^a_exp, ZBL covalent radius, Agnesi covalent radius)
  int zbl = 0, agnesi = 0;
  int zp = 6;                    // ZBL envelope exponent
  float za = 0.f;                // a_prefactor * 0.529
  float zc[4] = {0.f, 0.f, 0.f, 0.f};
  float zscale = 0.f;            // the model's scale: dE/dd of an edge gains scale * dV/dd
  float aq = 0.f, ap = 0.f, aa = 0.f;  // Agnesi q, p, a
};

// one term coef * A[i1] A[i2] A[i3] (first nu factors) of the symmetric contraction, weighted by w[z][kg][c], added to
// output slot o (0: the 0e output; 1 + m: component m of the 1o output; always 0 on layers with scalar output)
struct MaceTerm {
  int idx;  // i1 | i2 << 8 | i3 << 16 | nu << 24 | o << 28
  int kg;   // row of the element-channel weight table (all nu concatenated)
  float coef;
};

// conv_tp with 0e+1o node features (tests/mace_eq_ref.py conv_paths): paths per output l, all paths, and the message
// accumulators, ordered (l_out, m_out, j) with j the path's place among those of its l_out.  The message buffer Am of a
// 0e+1o layer holds, per l_out, a [(2 l_out + 1)][n_own][np(l_out) C] block (slot_base(l_out) n_own C floats in)
__host__ __device__ constexpr int mace_np_l(int max_ell, int l) { return l == 0 ? 2 : (l < max_ell ? 3 : 2); }
__host__ __device__ constexpr int mace_slot_base(int max_ell, int l) {
  return l == 0 ? 0 : mace_slot_base(max_ell, l - 1) + (2 * l - 1) * mace_np_l(max_ell, l - 1);
}
__host__ __device__ constexpr int mace_npaths(int max_ell) { return 3 * max_ell + 1; }
__host__ __device__ constexpr int mace_nslots(int max_ell) { return mace_slot_base(max_ell, max_ell + 1); }
constexpr int kMaceMaxSlots = mace_nslots(3);  // 40

// host side of the weight packing (engine_mace.inl).  The conv_tp paths (l_in, l_sh, l_out) for node features 0e (+ 1o
// when hidden_l = 1), in the order of tests/mace_eq_ref.py conv_paths (the radial MLP's output blocks)
std::vector<std::array<int, 3>> mace_conv_paths(int max_ell, int hidden_l);
// the terms of one U tensor of the symmetric contraction: U [ncomp][nsh]^nu [K] (ncomp 1: contractions.0, output slot 0;
// 3: contractions.1, slot 1 + m), summed over the permutations of each sorted index tuple, entries <= 1e-6 max |U|
// dropped, weight rows kg0 + k
std::vector<MaceTerm> mace_sym_terms(const float* U, int nsh, int nu, int ncomp, int K, int kg0);

// Y, eb; with the Agnesi transform on, the Bessel argument is x(d, Z_src, Z_dst) (endpoint species type[e_src / e_dst])
void launch_mace_edge_geom(cudaStream_t st, int64_t E, const float4* e_vec, const MaceRadial& rp, int nsh, float* Y,
                           float* eb, const int* e_src, const int* e_dst, const int* type, const MaceCore& core);
// e_lin[i] += sum of the ZBL energies V_e of the edges e -> i, in CSR row order (no atomics)
void launch_mace_zbl(cudaStream_t st, int n_own, const int* row_ptr, const int* e_src, const float4* e_vec,
                     const int* type, const MaceCore& core, float* e_lin);
void launch_mace_embed(cudaStream_t st, int n, int C, const int* type, const float* W, float* h0);
void launch_mace_msg(cudaStream_t st, int n_own, int C, int L1, const int* row_ptr, const int* e_src, const float* R,
                     const float* Y, const float* u, float* A);
void launch_mace_msg_bwd(cudaStream_t st, int n_own, int C, int L1, const int* row_ptr, const int* e_src, const float* R,
                         const float* Y, const float* u, const float* gA, float* gR, float* gY, float* gu);
// 0e+1o node features: Am (layout above) from u [n][4][C], R [E][npaths C], Y
void launch_mace_msg_eq(cudaStream_t st, int max_ell, int n_own, int C, const int* row_ptr, const int* e_src,
                        const float* R, const float* Y, const float* u, float* Am);
// its reverse: R is overwritten with gR (each (atom, channel) thread owns its edges' entries); gY, gu [n][4][C] accumulate
void launch_mace_msg_eq_bwd(cudaStream_t st, int max_ell, int n_own, int C, const int* row_ptr, const int* e_src,
                            float* R, const float* Y, const float* u, const float* gAm, float* gY, float* gu);
// out[i][m][:] (+)= in[i][m][:] @ W[type[i]][l(m)] for the first ncomp (1 or 4) components of rows of pitch ldi / ldo
// (the node-feature layout; W [n_elem][1 or 2][C][C])
void launch_mace_elem_mix_rows(cudaStream_t st, int n, int C, int ncomp, int ldi, int ldo, const int* type,
                               const float* W, const float* in, float* out, bool accum);
// symmetric contraction with a 1o output: B [4][n_own][C] (slot 0: 0e, 1..3: 1o) and its reverse (gB in the same layout)
void launch_mace_symc_eq(cudaStream_t st, int n_own, int C, int nsh, int Ktot, const int* type, const float* A,
                         const MaceTerm* terms, int nterms, const float* w, float* B);
void launch_mace_symc_eq_bwd(cudaStream_t st, int n_own, int C, int nsh, int Ktot, const int* type, const float* A,
                             const MaceTerm* terms, int nterms, const float* w, const float* gB, float* gA);
// out[lm][i][:] (+)= in[lm][i][:] @ W[type[i]][l(lm)]  (W [n_elem][L1][C][C]); nsh = 1 for a plain [n][C] row block
void launch_mace_elem_mix(cudaStream_t st, int n, int C, int L1, int nsh, const int* type, const float* W,
                          const float* in, float* out, bool accum);
void launch_mace_symc(cudaStream_t st, int n_own, int C, int nsh, int Ktot, const int* type, const float* A, const MaceTerm* terms,
                      int nterms, const float* w, float* B);
void launch_mace_symc_bwd(cudaStream_t st, int n_own, int C, int nsh, int Ktot, const int* type, const float* A,
                          const MaceTerm* terms, int nterms, const float* w, const float* gB, float* gA);
// e_lin[i] += h[i][0:C] . w   (linear readouts; w carries 1 / sqrt(C); rows of pitch ld)
void launch_mace_readout_lin(cudaStream_t st, int n_own, int C, int ld, const float* h, const float* w, float* e_lin);
// eps_i = E0[z] + scale * (e_lin + act(h W1) . w2) + shift; pre [n][H] kept for the reverse; energy += sum eps
// atom_e != nullptr: atom_e[gid[i]] = eps_i.  wgt != nullptr (heat flux, DESIGN.md §10): eps_i times wgt[gid[i]]
void launch_mace_readout_final(cudaStream_t st, int n_own, int C, int H, const float* h, const float* W1, const float* w2,
                               const float* e_lin, const int* type, const double* E0, double scale, double shift,
                               float* pre, double* energy, const int* gid, double* atom_e, const float* wgt);
// gh[i][c] = scale * sum_j W1[c][j] w2[j] SiLU'(pre[i][j])   (wgt != nullptr: times wgt[gid[i]])
void launch_mace_readout_seed(cudaStream_t st, int n_own, int C, int H, const float* pre, const float* W1,
                              const float* w2, float scale, float* gh, const int* gid, const float* wgt);
// gh[i][c] += scale * w[c]  (c < C, rows of pitch ld; wgt != nullptr: times wgt[gid[i]])
void launch_mace_add_row(cudaStream_t st, int n_own, int C, int ld, const float* w, float scale, float* gh,
                         const int* gid, const float* wgt);
// wgt != nullptr: the ZBL term of edge e times wgt[gid[dst(e)]]
void launch_mace_edge_final(cudaStream_t st, int64_t E, int nsh, const int* e_src, const int* e_dst, const float4* e_vec,
                            const int* gid, const int* type, const MaceRadial& rp, const MaceCore& core,
                            const float* g_eb, const float* gY, float* forces, double* virial, float* atom_vir,
                            const float* wgt);

struct MaceLayerW {
  bool residual = true;
  int Lin = 0, Lout = 0;      // node features 0e (0) or 0e+1o (1) in and out
  int NP = 0;                 // conv_tp paths (max_ell + 1 for 0e input)
  TcW Wup, WupT;              // [C][C] / sqrt(C) and its transpose
  TcW Wup1, Wup1T, Wprod1, Wprod1T;  // the 1o blocks of linear_up (Lin) and of the product linear (Lout)
  std::vector<TcW> mlp, mlpT;  // radial MLP layers (scaled, c_act folded, padded to multiples of 64) and transposes
  TcW Wlin[4], WlinT[4];       // per l [np(l) C][C] / (avg_num_neighbors sqrt(np(l) C)), np(l) = 1 for 0e input
  const float *Wskip = nullptr, *WskipT = nullptr;  // [n_elem][L1, 1 or 2][C][C] / sqrt(C n_elem)
  int Lskip = 1;                                    // l blocks of a residual skip
  TcW Wprod, WprodT;          // [C][C] / sqrt(C)
  const float* wsym = nullptr;                              // [n_elem][Ktot][C] (contractions.0, then .1)
  const MaceTerm* terms = nullptr;
  int nterms = 0, Ktot = 0;
  const float* wread = nullptr;                             // linear readout [C] / sqrt(C) (all layers but the last)
};

// workspace of the resident structure (b2m_release_workspace replaces it with an empty one)
struct MaceWork {
  DBuf<float> Y, eb, R, e_lin, pre_out, B, Am, sc;
  std::vector<DBuf<float>> h, u, A, pre;  // h: T + 1, u / A: T, pre: radial MLP hidden layers
  DBuf<float> act[2];
  // reverse
  DBuf<float> gY, g_eb, gR, gB, gA, gAm, gh, ghn, gu, gact[2];
};

struct MaceState : MaceWork {
  // C: row pitch of every per-atom array, the model's channel count Cr rounded up to a multiple of 64 (the wgmma GEMM
  // shapes); the padding channels carry zero weights and stay zero
  int C = 128, Cr = 128, L1 = 4, nsh = 16, T = 2, correlation = 3, H = 16;
  int hidden_max_l = 0;   // 1: hidden features 0e+1o (layers 0 < t and t < T - 1 carry 1o)
  std::vector<int> hw;    // row pitch of h[t], t = 0..T: C or 4 C
  double c_act = 1.0, scale = 1.0, shift = 0.0;
  MaceRadial rp{};
  MaceCore core{};
  std::vector<int> hid;   // radial MLP hidden widths, padded to 64
  int interaction_residual[kMaceMaxLayers] = {0};
  double avg_nb[kMaceMaxLayers] = {0};
  // weights
  const float* Wemb = nullptr;  // [n_elem][C] / sqrt(n_elem)
  std::vector<MaceLayerW> L;
  const float *W1 = nullptr, *w2 = nullptr;  // non-linear readout: [C][H] / sqrt(C), [H] c_act / sqrt(H)
  const double* E0 = nullptr;
  DBuf<double> e0buf;
};

}  // namespace b2m
