// kernels.cuh -- launch-side declarations of the CHGNet hot-path kernels (sm_90a).
//
// Formulation (verified against autograd in oracle/manual_ref.py):
//   first layer of every GatedMLP is split by input block, so the per-edge / per-angle work is
//     pre = gather(node projections) + (rank-9 radial term | dense 64->128 on the row's own feature)
//   followed by the 64x64 second layers, the gate product and a segmented sum.
// Reference arithmetic being replaced: SURVEY.md 8 rows a6-a15 (DistMLIP chgnet.py:208-453,
// chgnet_layers.py:16-119; matgl layer internals restated in SURVEY.md 9).
#pragma once
#include "common.cuh"

namespace b2m {

constexpr int TM = 128;   // rows (edges / angles) per tile
constexpr int LDA = 68;   // smem row pitch of a [TM][64] tile
constexpr int NT = 256;   // threads per block for the fused tile kernels

struct RadialParams {
  float freq[NR];
  float rc;
  float norm;  // sqrt(2/rc)
  int p;
};

// -------- elementwise / init --------
void launch_embed(cudaStream_t st, int n, const int* type, const float* emb, float* x0);
void launch_bond_init(cudaStream_t st, int nb, const float4* b_vec, RadialParams rp, const float* W /*[64][9]*/,
                      float* out /*[nb,64]*/);
void launch_angle_init(cudaStream_t st, int64_t na, const int* a_in, const int* a_out, const float4* b_vec,
                       const float* fa /*[5]*/, const float* Wae /*[64][9]*/, float* ang0 /*[A,64]*/);
void launch_silu(cudaStream_t st, int64_t n, const float* pre, float* out);
void launch_dsilu_mul(cudaStream_t st, int64_t n, const float* pre, float* g);  // g *= dsilu(pre)
void launch_zero_rows(cudaStream_t st, float* p, int64_t nfloats);

// -------- atom conv (the edge-gather kernel of the headline metric) --------
constexpr int ATOM_RAD_M = 0, ATOM_RAD_WAB = 2048, ATOM_RAD_M8 = 3072, ATOM_RAD_WAB8 = 3200, ATOM_RAD = 3264;
struct AtomConvArgs {
  int64_t E;
  const int* e_src;
  const int* e_dst;
  const int* e_bond;
  const float4* e_vec;
  const float* Aproj;  // [n_loc,128]  x @ W1s^T
  const float* Cproj;  // [n_own,128]  x @ W1t^T + b1
  const float* Qproj;  // [B_own,128]  h @ W1e^T   (nullptr for layer 0)
  // the rank-9 radial products be . M^T (M = W1e @ W_be, [128][9]) and be . W_ab^T (W_ab [64][9]) as one block of
  // ATOM_RAD floats (engine.cu radial_can): k = 0..7 as k-permuted wgmma B images of one k8 block, tf32 hi plane then
  // lo plane (M branch 0 at 0, M branch 1 at 1024, W_ab at 2048; each [64 n][8 k]), then column k = 8: M[.][8] at
  // 3072, W_ab[.][8] at 3200
  const float* radial;
  // second layers (L then G) as wgmma B operands: per branch the canonical K-major core-matrix image of a [64 n][64 k]
  // matrix, tf32 hi plane then lo plane (8192 floats per branch; engine.cu canon_split)
  const float* W2can;   // B[n][k] = W2[n][k]   (forward: hid . W2^T)
  const float* W2Tcan;  // B[n][k] = W2[k][n]   (backward: g . W2)
  const float* b2;     // [128]
  RadialParams rp;
  // forward
  float* agg;  // [n_own,64] (+=)
  // backward
  const float* gagg;  // [n_own,64]
  float* gA;          // [n_loc,128] (+=, atomics)   nullptr -> skip (layer 0)
  float* gC;          // [n_own,128] (+=)
  float* gQ;          // [B_own,128] (=)
  float* gd;          // [E] (+=)
};
// persistent: min(tiles, num_sms) CTAs loop over the 128-edge tiles
void launch_atomconv_fwd(cudaStream_t st, const AtomConvArgs& a, int num_sms);
void launch_atomconv_bwd(cudaStream_t st, const AtomConvArgs& a, int num_sms);

// -------- bond conv ("node" phase, HIDDEN) and angle update ("edge" phase, !HIDDEN) --------
struct LineArgs {
  int64_t A;
  const int* a_in;
  const int* a_out;
  const int* a_ctr;
  const float* ang;   // [A,64] input angle features
  const float* Ha;    // [B_loc,128]
  const float* Hb;    // [B_own,128] (+bias folded)
  const float* Xc;    // [n_loc,128]
  // wgmma B operands (canonical core-matrix images, tf32 hi plane then lo plane, k permuted inside every 8-wide k block;
  // engine.cu second_layer_can / line_reverse_can)
  const float* Wgcan;   // per branch [64 n][64 k]: B[n][k] = Wg[br*64 + n][k]  (angle block of the first layer)
  const float* WgTcan;  // [64 n][128 k]: B[n][k] = Wg[k][n]                     (backward: gang += gpre . Wg)
  const float* W2can;   // hidden only, as AtomConvArgs
  const float* W2Tcan;
  const float* b2;
  // forward outputs
  float* aggB;     // HIDDEN: [B_own,64] (+=)
  float* ang_out;  // !HIDDEN: [A,64]
  // backward
  const float* gaggB;  // HIDDEN: [B_own,64]
  float* gang;         // [A,64]: !HIDDEN reads it as upstream grad; both accumulate into it
  float* gHa;          // [B_loc,128] (+=)
  float* gHb;          // [B_own,128] (+=)
  float* gXc;          // [n_loc,128] (+=)
};
// persistent: min(tiles, num_sms) CTAs loop over the 128-angle tiles
void launch_line_fwd(cudaStream_t st, const LineArgs& a, bool hidden, int num_sms);
void launch_line_bwd(cudaStream_t st, const LineArgs& a, bool hidden, int num_sms);

// -------- host-side weight images of the fused kernels (engine.cu) --------
// raw [N][K] row-major -> canonical no-swizzle core-matrix layout, tf32 hi plane then lo plane (Kpad >= K: zero pad)
std::vector<float> canon_split(const std::vector<float>& raw, int N, int K, int Kpad);
// raw [N][K] with k permuted inside every 8-wide k block (slot q <- column 2q, slot q + 4 <- column 2q + 1)
std::vector<float> permute_k8(const std::vector<float>& raw, int N, int K);
// a stacked [128][64] block as the two k-permuted branch images of W2can / Wgcan (transposed: W2Tcan)
std::vector<float> second_layer_can(const std::vector<float>& raw128x64, bool transposed);
// a [128][64] first-layer block W as the k-permuted [64 n][128 k] image of gpre . W (WgTcan)
std::vector<float> line_reverse_can(const std::vector<float>& raw128x64);
// M [128][9] and W_ab [64][9] as AtomConvArgs::radial (ATOM_RAD floats)
std::vector<float> radial_can(const std::vector<float>& M, const std::vector<float>& Wab);

// -------- bond update: h' = h + upd * w3b(d_b) --------
void launch_bond_update_fwd(cudaStream_t st, int nb, const float4* b_vec, RadialParams rp3, const float* W3bw,
                            const float* h, const float* upd, float* hout);
// gupd = gh * w3b ; gdb += sum_k (sum_c gh*upd*W3bw[c][k]) * dtbe_k
void launch_bond_update_bwd(cudaStream_t st, int nb, const float4* b_vec, RadialParams rp3, const float* W3bw,
                            const float* gh, const float* upd, float* gupd, float* gdb);
// gdb += sum_k (sum_c gh0[b][c] Wbe[c][k]) dbe_k(d_b)
void launch_h0_bwd(cudaStream_t st, int nb, const float4* b_vec, RadialParams rp, const float* Wbe, const float* gh0,
                   float* gdb);
// theta / Fourier backward: gbvec[a], gbvec[b] += ...
void launch_angle_init_bwd(cudaStream_t st, int64_t na, const int* a_in, const int* a_out, const float4* b_vec,
                           const float* fa, const float* Wae, const float* gang0, float* gbvec);

// -------- readout --------
// e_atom = y2 @ F2 + c2 (+elem ref); energy (double) += sum; site = x @ Ws + bs
// atom_e != nullptr: also atom_e[gid[row]] = scale * e_atom + elem ref + mean_per_atom (per-atom energies, double)
void launch_rowdot(cudaStream_t st, int n, const float* X, const float* w, float bias, float* out, double* sum,
                   const int* type, const double* elem_ref, float scale, const int* gid = nullptr,
                   double* atom_e = nullptr, double mean_per_atom = 0.0, const float* wgt = nullptr);
// g[r][c] = scale * w[c] * dsilu(pre[r][c])   (wgt != nullptr: times wgt[gid[r]])
void launch_readout_seed(cudaStream_t st, int n, const float* pre, const float* w, float scale, float* g,
                         const int* gid = nullptr, const float* wgt = nullptr);

// -------- final geometry backward --------
// atom_vir != nullptr: also the per-atom virials, [N][12] f32 by global id (atomic_virial.cuh)
void launch_edge_final(cudaStream_t st, int64_t E, const int* e_src, const int* e_dst, const int* e_bond,
                       const float4* e_vec, const int* gid, const float* gd, const float* gdb, const float* gbvec,
                       float* forces /*[N,3]*/, double* virial /*[9]*/, float* atom_vir = nullptr);
void launch_halo_bond_final(cudaStream_t st, int b0, int b1, const int* b_src_gid, const int* b_dst,
                            const float4* b_vec, const int* gid, const float* gdb, const float* gbvec, float* forces,
                            double* virial, float* atom_vir = nullptr);

// -------- halo pack / unpack --------
void launch_gather_rows(cudaStream_t st, int n, int width, const int* idx, const float* src, float* dst);
void launch_scatter_add_rows(cudaStream_t st, int n, int width, const int* idx, const float* src, float* dst);

}  // namespace b2m

// ---------------------------------------------------------------------------------------------
// Row GEMMs on the Hopper tensor cores (kernels_wg.cu, wgmma).  3xTF32 split (hi*hi + lo*hi + hi*lo, fp32 accumulate)
// keeps fp32-level accuracy.  Weights are pre-formatted on the host into the canonical K-major / no-swizzle
// core-matrix layout (8 rows x 16 B), hi and lo planes (see engine.cu: canon_split()).
// ---------------------------------------------------------------------------------------------
namespace b2m {
// C[M,N] = (R | accum C | 0) + A[M,K] @ B + bias, B given as canonical hi/lo planes of its [N][K] view, then the
// epilogue: epi 1 keeps the value in Cpre (pitch ldc) and writes SiLU(value) to C; epi 2 multiplies the (accumulated)
// value by SiLU'(Pre[row][col]) (pitch ldp); epi 0 = plain.  (K,N) in {(64,128), (64,64), (128,64)}.
// The engine calls it only through tc_mm (engine.cu), which splits a larger product into these blocks.
void launch_gemm_wg(cudaStream_t st, const float* A, int lda, const float* Bcan, float* C, int ldc, int M, int N, int K,
                    const float* bias, const float* R, int ldr, bool accum, int epi, float* Cpre, const float* Pre,
                    int ldp, int num_sms);
// A [K][N] weight (y = x W) as B operands of launch_gemm_wg: the blocks tc_mm launches, in launch order (engine.cu
// pack_tc), each the canonical hi/lo image of its [nc][kc] view stored at float offset `off` of the engine's weight buffer
struct TcW {
  struct Blk {
    int k0, kc, n0, nc;
    size_t off;
  };
  int K = 0, N = 0;
  std::vector<Blk> blk;
};
}  // namespace b2m

// ---------------------------------------------------------------------------------------------
// TensorNet path (kernels_tn.cu).  Per-atom tensors in decomposed form [n][10][64] (I | a_xyz | S_xx xy xz yy yz zz).
// ---------------------------------------------------------------------------------------------
namespace b2m {
struct TnRadial {
  int nr;       // Gaussian centres in use
  int nrp;      // row pitch of the rbf / g_rbf buffers (multiple of 64, padding columns zero)
  float width;  // exp(-width (d - mu_k)^2)
  float rc;     // cosine cutoff radius
  float mu[64];
};
// C[z][M,N] = epi(A[z][M,K] @ B[K,N] + bias); z-batched over the 10 rows of a decomposed tensor when nz = 10
// (A + z*zA, C + z*zC, B = bsel ? (z==0 ? B0 : z<4 ? B1 : B2) : B0).  B is [K][N] row-major.  K % 32 == 0, N % 64 == 0.
// epi 0: store | 1: Cpre = value, C = SiLU(value) | 2: value *= SiLU'(Pre[m][n]) ; accum adds the old C afterwards.
struct TnGemm {
  const float* A = nullptr;
  int lda = 0;
  int64_t zA = 0;
  const float *B0 = nullptr, *B1 = nullptr, *B2 = nullptr;
  int bsel = 0;
  float* C = nullptr;
  int ldc = 0;
  int64_t zC = 0;
  float* Cpre = nullptr;
  const float* Pre = nullptr;
  int ldp = 0;
  const float* bias = nullptr;
  int M = 0, N = 0, K = 0, accum = 0, epi = 0;
};
void launch_tn_gemm(cudaStream_t st, const TnGemm& g, int nz);
void launch_tn_edge_geom(cudaStream_t st, int64_t E, const float4* e_vec, const TnRadial& rp, float* rbf, float* cut);
void launch_tn_embed_agg(cudaStream_t st, int n_own, const int* row_ptr, const int* e_src, const int* type,
                         const float* U, const float* V, const float* P, const float* cut, const float4* e_vec,
                         float* T0, float* nr0);
void launch_tn_layernorm(cudaStream_t st, int rows, int W, const float* x, const float* gamma, const float* beta,
                         float* y, float* stats);
void launch_tn_layernorm_bwd(cudaStream_t st, int rows, int W, const float* x, const float* stats, const float* gamma,
                             const float* gy, float* gx);
void launch_tn_embed_out(cudaStream_t st, int n, const float* T0m, const float* s2p, float* X0);
void launch_tn_embed_out_bwd(cudaStream_t st, int n, const float* T0m, const float* s2p, const float* gX0, float* gT0m,
                             float* gs2p);
void launch_tn_norm_bwd_add(cudaStream_t st, int n, const float* T0, const float* gnr0, float* gT0);
void launch_tn_embed_agg_bwd(cudaStream_t st, int64_t E, const int* e_src, const int* e_dst, const int* type,
                             const float* U, const float* V, const float* P, const float* cut, const float4* e_vec,
                             const float* gT0, float* gP, float* gC, float* gvh);
void launch_tn_scale(cudaStream_t st, int n, const float* X, float* Xh, float* q);
void launch_tn_scale_bwd(cudaStream_t st, int n, const float* X, const float* q, float* g);
void launch_tn_msg(cudaStream_t st, int n_own, const int* row_ptr, const int* e_src, const float* f3p, const float* cut,
                   const float* Y, float* msg);
void launch_tn_msg_bwd(cudaStream_t st, int n_own, const int* row_ptr, const int* e_src, const float* f3p,
                       const float* cut, const float* Y, const float* gmsg, float* g3, float* gC, float* gY);
void launch_tn_prod(cudaStream_t st, int n, const float* msg, const float* Y, int so3, float* Pn);
void launch_tn_prod_bwd(cudaStream_t st, int n, const float* msg, const float* Y, int so3, const float* gPn,
                        float* gmsg, float* gY);
void launch_tn_update(cudaStream_t st, int n, const float* Xh, const float* dX, float* Xn);
void launch_tn_update_bwd(cudaStream_t st, int n, const float* dX, const float* gXn, float* gdX);
void launch_tn_invariants(cudaStream_t st, int n, const float* X, float* inv);
void launch_tn_invariants_bwd(cudaStream_t st, int n, const float* X, const float* ginv, float* gX);
void launch_tn_readout_final(cudaStream_t st, int n, int W, const float* hL, const float* wL, float bL, const float* hG,
                             const float* wG, float bG, const int* type, const double* eref, float scale, float* lout,
                             float* gout, float* e_atom, double* energy, const int* gid = nullptr,
                             double* atom_e = nullptr, double mean_per_atom = 0.0, const float* wgt = nullptr);
void launch_tn_readout_seed(cudaStream_t st, int n, int W, const float* lout, const float* gout, float scale,
                            const float* wL, const float* wG, const float* preL, const float* preG, float* gL,
                            float* gG, const int* gid = nullptr, const float* wgt = nullptr);
void launch_tn_edge_final(cudaStream_t st, int64_t E, const int* e_src, const int* e_dst, const float4* e_vec,
                          const int* gid, const TnRadial& rp, const float* g_rbf, const float* gC, const float* gvh,
                          float* gd, float* forces, double* virial, float* atom_vir = nullptr);
}  // namespace b2m
