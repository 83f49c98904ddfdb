// engine.cu -- host orchestration behind the C-ABI (include/b200mlip.h):
// weight composition, GPU-resident workspace, forward + hand-derived backward schedule, halo exchange
// between slab neighbours (NCCL point-to-point between processes, peer-memory stores inside a
// single-process group), and the extern "C" entry points.
//
// Schedule mirrors (and is verified stage-by-stage against) oracle/manual_ref.py; the reference
// control flow it replaces is DistMLIP/implementations/matgl/models/chgnet.py:208-453 (forward)
// and pes.py:109-145 (scaling, autograd backward, forces, stress).
#include <dlfcn.h>
#include <nccl.h>

#include <cmath>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <cstring>
#include <map>
#include <new>
#include <set>
#include <string>
#include <vector>

#include <algorithm>
#include <array>

#include "atomic_virial.cuh"
#include "graph.cuh"
#include "kernels.cuh"
#include "mace_state.cuh"
#include "tn_state.cuh"

namespace b2m {

// ------------------------------------------------------------------------------------------
// NCCL through dlopen: if torch already loaded its bundled libnccl.so.2 we reuse that copy.
// ------------------------------------------------------------------------------------------
struct Nccl {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  void load() {
    if (lib) return;
    lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);
    if (!lib) lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    B2M_REQUIRE(lib != nullptr, B2M_ERR_CUDA, "cannot dlopen libnccl.so.2 (needed for world > 1)");
#define L(name, sym)                                              \
  *(void**)(&name) = dlsym(lib, sym);                             \
  B2M_REQUIRE(name != nullptr, B2M_ERR_CUDA, "NCCL symbol missing: " sym)
    L(GetUniqueId, "ncclGetUniqueId");
    L(CommInitRank, "ncclCommInitRank");
    L(CommDestroy, "ncclCommDestroy");
    L(Send, "ncclSend");
    L(Recv, "ncclRecv");
    L(AllReduce, "ncclAllReduce");
    L(GroupStart, "ncclGroupStart");
    L(GroupEnd, "ncclGroupEnd");
    L(GetErrorString, "ncclGetErrorString");
#undef L
  }
};
static Nccl g_nccl;
#define NCCL_CK(call)                                                                              \
  do {                                                                                             \
    ncclResult_t r__ = (call);                                                                     \
    if (r__ != ncclSuccess)                                                                        \
      throw b2m::Error(B2M_ERR_CUDA, std::string("NCCL error: ") + g_nccl.GetErrorString(r__));   \
  } while (0)

// ------------------------------------------------------------------------------------------
// row-GEMM weights as TcW pairs (the projection, then its transpose for the reverse pass); the fused-kernel images and
// the biases as device pointers
struct AtomLayerW {
  TcW W1s, W1sT, W1e, W1eT, W1t, W1tT, Wout, WoutT;
  float *b1, *radial, *W2can, *W2Tcan, *b2;
};
struct BondLayerW {
  TcW W1a, W1aT, W1b, W1bT, W1c, W1cT, Wout, WoutT, WAa, WAaT, WAb, WAbT, WAc, WAcT;
  float *Wgcan, *WgTcan, *b1, *W2can, *W2Tcan, *b2, *WAgcan, *WAgTcan, *bA;
};

}  // namespace b2m

using namespace b2m;

// Host-side rendezvous of the partition threads of a single-process group (b2m_create with ndev > 1).  abort() releases
// every waiter so that an exception in one partition cannot dead-lock the others.
struct GroupSync {
  std::mutex m;
  std::condition_variable cv;
  int n = 1, waiting = 0;
  long long gen = 0;
  bool aborted = false;
  void reset(int n_) { n = n_, waiting = 0, aborted = false; }
  void arrive_and_wait() {
    std::unique_lock<std::mutex> lk(m);
    if (aborted) throw b2m::Error(B2M_ERR_STATE, "a partition of the group failed");
    const long long my = gen;
    if (++waiting == n) {
      waiting = 0, gen++;
      cv.notify_all();
      return;
    }
    cv.wait(lk, [&] { return gen != my || aborted; });
    if (aborted && gen == my) throw b2m::Error(B2M_ERR_STATE, "a partition of the group failed");
  }
  void abort() {
    std::lock_guard<std::mutex> lk(m);
    aborted = true;
    cv.notify_all();
  }
};

struct b2m_engine {
  b2m_model_desc desc;
  int kind = 0;                   // 0: CHGNet (b2m_create), 1: TensorNet (b2m_create_tensornet), 2: MACE (b2m_create_mace)
  b2m::TnState* tn = nullptr;     // TensorNet weights and workspace (kind 1)
  b2m::MaceState* mace = nullptr;  // MACE weights and workspace (kind 2)
  int device = 0;
  cudaStream_t st = nullptr;
  cudaStream_t cst = nullptr;            // halo traffic of the forward pass (overlaps the projections that do not need it)
  cudaEvent_t ev_prod = nullptr, ev_halo = nullptr;
  std::string err;
  // weights
  std::map<std::string, std::vector<float>> host_w;
  std::map<std::string, std::vector<int64_t>> host_shape;
  std::set<std::string> consumed;  // state_dict keys finalize_weights actually used
  std::vector<double> elem_refs;
  DBuf<double> erefbuf;
  bool finalized = false;
  DBuf<float> wbuf;
  std::vector<AtomLayerW> aw;
  std::vector<BondLayerW> bw;
  float *d_emb = nullptr, *d_Wbe = nullptr, *d_Wae = nullptr, *d_W3bw = nullptr, *d_fa = nullptr;
  TcW F0, F0T, F1, F1T;  // final MLP 64 -> 64 -> 64 and transposes
  float *d_c0 = nullptr, *d_c1 = nullptr, *d_F2 = nullptr, *d_Ws = nullptr;
  const double* d_eref = nullptr;  // per-element energy offsets, double like the energy accumulator
  float c2 = 0.f, bs = 0.f;
  RadialParams rp2, rp3;
  // comm
  int rank = 0, world = 1;
  ncclComm_t comm = nullptr;
  // single-process group (ndev > 1): the handle returned by b2m_create is parts[0]; every partition is a full engine on
  // its own device (ordinals may repeat) and stream, driven by its own host thread inside b2m_set_structure /
  // b2m_compute; halo rows travel as direct peer-memory stores / copies ordered by CUDA events (no NCCL)
  std::vector<b2m_engine*> parts;  // leader only: all partitions, parts[0] == this
  b2m_engine* leader = nullptr;    // members: the leader (for the peer table and the rendezvous)
  GroupSync gsync;                 // leader only
  std::vector<cudaEvent_t> hev;    // one event per halo-exchange point of a run
  int hpoint = 0;
  DBuf<float> precv[2];            // adjoint rows pushed by my neighbours (backward), double-buffered by point parity
  DBuf<float> ftmp;                // leader: staging of a peer's force array
  DBuf<float> fsum;                // leader: the group's summed forces (the partitions' own arrays stay untouched)
  int view = 0;                    // leader: partition addressed by the inspection calls (b2m_set_view)
  // page-locked staging owned by the library: host arrays go through it with a few copy threads (a single-threaded
  // memcpy of 24 MB of positions was the largest host item of an end-to-end step at 1 M atoms)
  void* pin_in = nullptr;   // [N,3] f64 positions followed by [N] i32 species
  size_t pin_in_cap = 0;
  void* pin_out = nullptr;  // [N,3] f32 forces
  size_t pin_out_cap = 0;
  // graph + workspace
  Graph g;
  bool have_graph = false;
  std::vector<DBuf<float>> x, h, ang, upd;
  bool want_grads = true;
  // first-layer projections of every atom-conv layer (A = x W1s^T, C = x W1t^T + b1, Q = h W1e^T), one buffer per
  // layer: the backward gathers the rows the forward wrote instead of re-running three GEMMs per layer
  // (about 1.1 GB per 100k atoms for the four layers)
  std::vector<DBuf<float>> ApL, CpL, QpL;
  static int proj_slot(int l) { return l; }
  DBuf<float> Ha, Hb, Xc, agg, aggB, y1p, y1, y2p, y2, e_atom, site;
  DBuf<float> gx, gh, gang, gA, gC, gQ, gHa, gHb, gXc, gagg, gupd, gaggB, gd, gdb, gbvec, gy1, gy2;
  DBuf<float> forces, sendbuf, recvbuf, site_full;
  DBuf<double> scal;  // [0]=energy, [1..9]=virial
  // per-atom energies and virials (b2m_set_atomic; DESIGN.md "Per-atom energies and virials"): allocated on the first
  // evaluation with the flag on, indexed by global atom id like `forces`
  bool atomic = false;
  int atomic_last = 0;      // what the last evaluation left in them: 0 nothing, 1 energies, 2 energies and virials
  DBuf<double> atom_e;      // [N]
  DBuf<float> atom_vir;     // [N][kVirPitch]
  DBuf<double> aesum, aetmp;  // leader of a group: the summed energies / staging of a peer's array
  DBuf<float> avsum, avtmp;   // same for the virials
  // heat flux (b2m_set_heat_flux; DESIGN.md §10): with hf_reach > 0 b2m_set_structure builds the unfolded cell (`uf`) and
  // the graph of it without periodicity; every readout then weights atom j's energy by hf_w[j]
  double hf_reach = 0;
  Unfold uf;
  int64_t hf_n = 0;       // cell atoms of the resident unfolded graph; 0: the graph is the structure itself
  int hf_seed = -1;       // weight of the next evaluation: -1 the cell mask (1 / 0), 0..2 the seed (r_j - c)_alpha
  double hf_c[3] = {0, 0, 0};  // cell centre
  DBuf<float> hf_w;       // [N] readout weight of every unfolded atom
  DBuf<float> hf_G;       // leader: [3][N][3] forces of the three seeded passes
  DBuf<float> hf_fold;    // leader: folded forces [n][3] or virials [n][kVirPitch]
  DBuf<double> hf_vel, hf_out;
  // timings
  cudaEvent_t ev[8] = {nullptr};
  double t_graph = 0, t_fwd = 0, t_bwd = 0, t_gather = 0, t_total = 0;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> gather_ev;
  long long launches_last = 0;
  double last_energy = 0;
  int num_sms = 132;
  bool debug_no_halo = false;  // B2M_DEBUG_NO_HALO=1: a b2m_set_partition view may run with its exchanges skipped (wrong
                               // numbers, right amount of per-partition work: timing one slab of an N-way split on one GPU)
};

namespace b2m {

// atoms of the structure the caller passed: the graph's atoms, or the cell atoms of an unfolded graph
static int64_t cell_atoms(const b2m_engine* e) { return e->hf_n ? e->hf_n : e->g.N; }

static const std::vector<float>& W(b2m_engine* e, const std::string& k, std::vector<int64_t> shape) {
  auto it = e->host_w.find(k);
  B2M_REQUIRE(it != e->host_w.end(), B2M_ERR_INVALID, "missing weight: " + k);
  e->consumed.insert(k);
  const auto& sh = e->host_shape[k];
  size_t n = 1;
  for (auto s : shape) n *= (size_t)s;
  B2M_REQUIRE(it->second.size() == n && sh == shape, B2M_ERR_INVALID,
              "weight '" + k + "' has an unsupported shape (engine supports dim=64, max_n=9, max_f=4)");
  return it->second;
}

struct Packer {
  std::vector<float> host;
  size_t add(const std::vector<float>& v) {
    size_t off = (host.size() + 63) / 64 * 64;  // 256 B alignment
    host.resize(off + v.size());
    memcpy(host.data() + off, v.data(), v.size() * sizeof(float));
    return off;
  }
};

// slice columns [c0, c0+64) of a row-major [rows][ncol] matrix -> [rows][64]
static std::vector<float> cols(const std::vector<float>& m, int rows, int ncol, int c0) {
  std::vector<float> o((size_t)rows * 64);
  for (int r = 0; r < rows; r++)
    for (int c = 0; c < 64; c++) o[(size_t)r * 64 + c] = m[(size_t)r * ncol + c0 + c];
  return o;
}
static std::vector<float> transpose(const std::vector<float>& m, int rows, int ncol) {
  std::vector<float> o(m.size());
  for (int r = 0; r < rows; r++)
    for (int c = 0; c < ncol; c++) o[(size_t)c * rows + r] = m[(size_t)r * ncol + c];
  return o;
}
static std::vector<float> vcat(const std::vector<float>& a, const std::vector<float>& b) {
  std::vector<float> o(a);
  o.insert(o.end(), b.begin(), b.end());
  return o;
}
// tf32 "hi" part: round-to-nearest (ties away) on the 13 dropped mantissa bits == cvt.rna.tf32.f32
static float tf32_hi_host(float x) {
  uint32_t u;
  memcpy(&u, &x, 4);
  u += 0x1000u;
  u &= 0xFFFFE000u;
  float r;
  memcpy(&r, &u, 4);
  return r;
}
// raw [N][K] row-major (K contiguous == K-major operand) -> canonical no-swizzle core-matrix layout
// (8 rows x 16 B per core matrix; K-chunk-major then row-group), hi plane followed by lo plane.
// element (n, k) at ((k/4) * (N/8) + n/8) * 32 + (n%8)*4 + k%4 ;  Kpad >= K pads with zeros.
std::vector<float> canon_split(const std::vector<float>& raw, int N, int K, int Kpad) {
  std::vector<float> o((size_t)2 * N * Kpad, 0.f);
  for (int n = 0; n < N; n++)
    for (int k = 0; k < K; k++) {
      const size_t off = ((size_t)(k / 4) * (N / 8) + n / 8) * 32 + (n % 8) * 4 + (k % 4);
      const float x = raw[(size_t)n * K + k];
      const float h = tf32_hi_host(x);
      o[off] = h;
      o[(size_t)N * Kpad + off] = x - h;
    }
  return o;
}

// raw [N][K] with k permuted inside every 8-wide k block: slot q holds column 2q and slot q + 4 column 2q + 1.  The
// fused kernels pass A as float2 pairs (columns 2 (l%4), 2 (l%4) + 1 of a block), from their wgmma accumulator
// fragments or from a shared-memory tile, as the register A fragment (k slots l%4, l%4 + 4) of the product
// (kernels.cu: wg_mm64_acc, wg_mm64), so every fused-kernel B image is formatted this way.
std::vector<float> permute_k8(const std::vector<float>& raw, int N, int K) {
  std::vector<float> o(raw.size());
  for (int n = 0; n < N; n++)
    for (int k = 0; k < K; k++) {
      const int q = k % 8;
      o[(size_t)n * K + k] = raw[(size_t)n * K + (k - q) + (q < 4 ? 2 * q : 2 * (q - 4) + 1)];
    }
  return o;
}

// both 64-row branches (L then G) of a stacked [128][64] block as k-permuted wgmma B operands of the fused kernels:
// per branch canon_split of B[n][k] = raw[br*64 + n][k] (transposed = false) or raw[br*64 + k][n] (true)
std::vector<float> second_layer_can(const std::vector<float>& raw128x64, bool transposed) {
  std::vector<float> out;
  for (int br = 0; br < 2; br++) {
    std::vector<float> blk(raw128x64.begin() + (size_t)br * 4096, raw128x64.begin() + (size_t)(br + 1) * 4096);
    if (transposed) blk = transpose(blk, 64, 64);
    const auto c = canon_split(permute_k8(blk, 64, 64), 64, 64, 64);
    out.insert(out.end(), c.begin(), c.end());
  }
  return out;
}
// the [128][64] first-layer block W as the k-permuted B operand of gpre . W (K = 128): B[n][k] = W[k][n]
std::vector<float> line_reverse_can(const std::vector<float>& raw128x64) {
  return canon_split(permute_k8(transpose(raw128x64, 128, 64), 64, 128), 64, 128, 128);
}
// the atom conv's radial weights M [128][9] and W_ab [64][9] in the layout of AtomConvArgs::radial: columns 0..7 of each
// 64-row block as a k-permuted [64 n][8 k] wgmma B image (one k8 block on the tensor cores), column 8 as a side table
std::vector<float> radial_can(const std::vector<float>& M, const std::vector<float>& Wab) {
  auto k8 = [](const std::vector<float>& w, int row0) {
    std::vector<float> o(64 * 8);
    for (int n = 0; n < 64; n++)
      for (int k = 0; k < 8; k++) o[(size_t)n * 8 + k] = w[(size_t)(row0 + n) * NR + k];
    return canon_split(permute_k8(o, 64, 8), 64, 8, 8);
  };
  std::vector<float> out;
  for (const auto& c : {k8(M, 0), k8(M, 64), k8(Wab, 0)}) out.insert(out.end(), c.begin(), c.end());
  for (int j = 0; j < 128; j++) out.push_back(M[(size_t)j * NR + 8]);
  for (int c = 0; c < 64; c++) out.push_back(Wab[(size_t)c * NR + 8]);
  B2M_REQUIRE(out.size() == ATOM_RAD, B2M_ERR_INVALID, "atom-conv radial block size");
  return out;
}

// a [K][N] row-major weight (y = x W, K and N multiples of 64) as the wgmma blocks of tc_mm, packed into P: K chunks of
// kmax (128 or 64; 64 for a remainder), per chunk N blocks of 64, or of 128 when the chunk is 64 deep
static TcW pack_tc(Packer& P, const std::vector<float>& W, int K, int N, int kmax = 128) {
  TcW w;
  w.K = K, w.N = N;
  for (int k0 = 0; k0 < K;) {
    const int kc = K - k0 >= kmax ? kmax : 64;
    for (int n0 = 0; n0 < N;) {
      const int nc = kc == 64 && N - n0 >= 128 ? 128 : 64;
      std::vector<float> raw((size_t)nc * kc);  // B[n][k] = W[k0 + k][n0 + n]
      for (int n = 0; n < nc; n++)
        for (int k = 0; k < kc; k++) raw[(size_t)n * kc + k] = W[(size_t)(k0 + k) * N + n0 + n];
      w.blk.push_back({k0, kc, n0, nc, P.add(canon_split(raw, nc, kc, kc))});
      n0 += nc;
    }
    k0 += kc;
  }
  return w;
}
// the weight and its transpose [N][K] (the reverse pass's product, in K chunks of rev_kmax)
static void pack_tc2(Packer& P, const std::vector<float>& W, int K, int N, TcW& fwd, TcW& rev, int rev_kmax = 128) {
  fwd = pack_tc(P, W, K, N);
  rev = pack_tc(P, transpose(W, K, N), N, K, rev_kmax);
}
// out[M][N] (+)= epi(A[M][K] @ W + bias) (+ R, pitch ldr): the K chunks after the first accumulate in place, so bias and R
// go with the first; epi 1 (SiLU, pre-activation kept in Cpre) needs a single K chunk, epi 2 (times SiLU'(Pre)) is applied
// by the last one
static void tc_mm(b2m_engine* e, const float* A, int lda, const TcW& W, float* out, int ldc, int M, bool accum,
                  const float* bias = nullptr, const float* R = nullptr, int ldr = 0, int epi = 0, float* Cpre = nullptr,
                  const float* Pre = nullptr, int ldp = 0) {
  B2M_REQUIRE(epi != 1 || W.blk.back().k0 == 0, B2M_ERR_INVALID, "row GEMM: SiLU epilogue over several K chunks");
  for (const TcW::Blk& b : W.blk) {
    const bool first = b.k0 == 0, last = b.k0 + b.kc == W.K;
    launch_gemm_wg(e->st, A + b.k0, lda, e->wbuf.p + b.off, out + b.n0, ldc, M, b.nc, b.kc,
                   first && bias ? bias + b.n0 : nullptr, first && R ? R + b.n0 : nullptr, ldr, accum || !first,
                   epi == 2 && !last ? 0 : epi, Cpre ? Cpre + b.n0 : nullptr, epi == 2 && last ? Pre + b.n0 : nullptr,
                   ldp, e->num_sms);
  }
}

static void finalize_weights(b2m_engine* e) {
  const int nb = e->desc.n_blocks;
  for (auto& kv : e->host_w) {
    const std::string& k = kv.first;
    bool bad = k.find("atom_graph_layers") != std::string::npos &&
               (k.find("edge_update_func") != std::string::npos || k.find("weight_func") != std::string::npos);
    bad = bad || (k.find("bond_graph_layers") != std::string::npos && k.find("weight_func") != std::string::npos);
    bad = bad || k.find("state_embedding") != std::string::npos || k.find("normalization") != std::string::npos;
    B2M_REQUIRE(!bad, B2M_ERR_INVALID,
                "unsupported CHGNet option (bond_update_hidden_dims / layer_bond_weights / state / norm): " + k);
  }
  e->consumed.clear();
  Packer P;
  std::map<std::string, size_t> off;
  auto put = [&](const std::string& name, const std::vector<float>& v) { off[name] = P.add(v); };
  // an nn.Linear weight [out][in] as the row GEMM x . W^T (K = in) and its reverse g . W
  auto linear = [&](const std::vector<float>& w, int out, int in, TcW& fwd, TcW& rev) {
    pack_tc2(P, transpose(w, out, in), in, out, fwd, rev);
  };

  const auto& f2 = W(e, "bond_expansion.frequencies", {NR});
  const auto& f3 = W(e, "threebody_bond_expansion.frequencies", {NR});
  const auto& fa = W(e, "angle_expansion.frequencies", {5});
  for (int k = 0; k < NR; k++) {
    e->rp2.freq[k] = f2[k];
    e->rp3.freq[k] = f3[k];
  }
  e->rp2.rc = (float)e->desc.cutoff;
  e->rp3.rc = (float)e->desc.three_body_cutoff;
  e->rp2.norm = (float)std::sqrt(2.0 / e->desc.cutoff);
  e->rp3.norm = (float)std::sqrt(2.0 / e->desc.three_body_cutoff);
  e->rp2.p = e->rp3.p = e->desc.cutoff_exponent;
  put("fa", fa);
  put("emb", W(e, "atom_embedding.weight", {e->desc.n_elem, D}));
  const auto& Wbe = W(e, "bond_embedding.layers.0.weight", {D, NR});
  put("Wbe", Wbe);
  put("Wae", W(e, "angle_embedding.layers.0.weight", {D, NF}));
  const auto& Wabw = W(e, "atom_bond_weights.weight", {D, NR});
  put("W3bw", W(e, "threebody_bond_weights.weight", {D, NR}));

  e->aw.resize(nb);
  for (int l = 0; l < nb; l++) {
    const std::string p = "atom_graph_layers." + std::to_string(l) + ".conv_layer.";
    const auto W1 = vcat(W(e, p + "node_update_func.layers.layers.0.weight", {D, 3 * D}),
                         W(e, p + "node_update_func.gates.layers.0.weight", {D, 3 * D}));  // [128][192]
    const auto b1 = vcat(W(e, p + "node_update_func.layers.layers.0.bias", {D}),
                         W(e, p + "node_update_func.gates.layers.0.bias", {D}));
    const auto W1s = cols(W1, 128, 192, 0), W1e = cols(W1, 128, 192, 64), W1t = cols(W1, 128, 192, 128);
    const auto W2 = vcat(W(e, p + "node_update_func.layers.layers.1.weight", {D, D}),
                         W(e, p + "node_update_func.gates.layers.1.weight", {D, D}));
    const auto b2 = vcat(W(e, p + "node_update_func.layers.layers.1.bias", {D}),
                         W(e, p + "node_update_func.gates.layers.1.bias", {D}));
    const auto& Wout = W(e, p + "node_out_func.weight", {D, D});
    std::vector<float> M(128 * 9);
    for (int j = 0; j < 128; j++)
      for (int k = 0; k < 9; k++) {
        double s = 0;
        for (int c = 0; c < 64; c++) s += (double)W1e[(size_t)j * 64 + c] * (double)Wbe[(size_t)c * 9 + k];
        M[j * 9 + k] = (float)s;
      }
    const std::string q = "a" + std::to_string(l) + ".";
    AtomLayerW& w = e->aw[l];
    linear(W1s, 128, 64, w.W1s, w.W1sT);
    linear(W1e, 128, 64, w.W1e, w.W1eT);
    linear(W1t, 128, 64, w.W1t, w.W1tT);
    linear(Wout, 64, 64, w.Wout, w.WoutT);
    put(q + "b1", b1);
    put(q + "radial", radial_can(M, Wabw));
    put(q + "W2can", second_layer_can(W2, false));
    put(q + "W2Tcan", second_layer_can(W2, true));
    put(q + "b2", b2);
  }
  e->bw.resize(nb - 1);
  for (int l = 0; l < nb - 1; l++) {
    const std::string p = "bond_graph_layers." + std::to_string(l) + ".conv_layer.";
    const auto W1 = vcat(W(e, p + "node_update_func.layers.layers.0.weight", {D, 4 * D}),
                         W(e, p + "node_update_func.gates.layers.0.weight", {D, 4 * D}));  // [128][256]
    const auto b1 = vcat(W(e, p + "node_update_func.layers.layers.0.bias", {D}),
                         W(e, p + "node_update_func.gates.layers.0.bias", {D}));
    const auto W1a = cols(W1, 128, 256, 0), W1g = cols(W1, 128, 256, 64), W1c = cols(W1, 128, 256, 128),
               W1b = cols(W1, 128, 256, 192);
    const auto W2 = vcat(W(e, p + "node_update_func.layers.layers.1.weight", {D, D}),
                         W(e, p + "node_update_func.gates.layers.1.weight", {D, D}));
    const auto b2 = vcat(W(e, p + "node_update_func.layers.layers.1.bias", {D}),
                         W(e, p + "node_update_func.gates.layers.1.bias", {D}));
    const auto& Wout = W(e, p + "node_out_func.weight", {D, D});
    const auto WA = vcat(W(e, p + "edge_update_func.layers.layers.0.weight", {D, 4 * D}),
                         W(e, p + "edge_update_func.gates.layers.0.weight", {D, 4 * D}));
    const auto bA = vcat(W(e, p + "edge_update_func.layers.layers.0.bias", {D}),
                         W(e, p + "edge_update_func.gates.layers.0.bias", {D}));
    const auto WAa = cols(WA, 128, 256, 0), WAg = cols(WA, 128, 256, 64), WAc = cols(WA, 128, 256, 128),
               WAb = cols(WA, 128, 256, 192);
    const std::string q = "b" + std::to_string(l) + ".";
    BondLayerW& w = e->bw[l];
    linear(W1a, 128, 64, w.W1a, w.W1aT);
    linear(W1b, 128, 64, w.W1b, w.W1bT);
    linear(W1c, 128, 64, w.W1c, w.W1cT);
    linear(Wout, 64, 64, w.Wout, w.WoutT);
    linear(WAa, 128, 64, w.WAa, w.WAaT);
    linear(WAb, 128, 64, w.WAb, w.WAbT);
    linear(WAc, 128, 64, w.WAc, w.WAcT);
    put(q + "Wgcan", second_layer_can(W1g, false));
    put(q + "b1", b1);
    put(q + "WgTcan", line_reverse_can(W1g));
    put(q + "W2can", second_layer_can(W2, false));
    put(q + "W2Tcan", second_layer_can(W2, true));
    put(q + "b2", b2);
    put(q + "WAgcan", second_layer_can(WAg, false));
    put(q + "bA", bA);
    put(q + "WAgTcan", line_reverse_can(WAg));
  }
  linear(W(e, "final_layer.layers.0.weight", {D, D}), 64, 64, e->F0, e->F0T);
  put("c0", W(e, "final_layer.layers.0.bias", {D}));
  linear(W(e, "final_layer.layers.1.weight", {D, D}), 64, 64, e->F1, e->F1T);
  put("c1", W(e, "final_layer.layers.1.bias", {D}));
  put("F2", W(e, "final_layer.layers.2.weight", {1, D}));
  e->c2 = W(e, "final_layer.layers.2.bias", {1})[0];
  put("Ws", W(e, "sitewise_readout.weight", {1, D}));
  e->bs = W(e, "sitewise_readout.bias", {1})[0];
  // every tensor of the state_dict must have been used: an extra bias / normalisation / per-layer weight function of
  // a non-default CHGNet configuration would otherwise be dropped silently and give wrong energies (ADVICE r1).
  // bond_bond_weights is part of the default model but feeds only the (absent) bond update of the atom graph.
  for (auto& kv : e->host_w) {
    if (e->consumed.count(kv.first) || kv.first == "bond_bond_weights.weight") continue;
    throw Error(B2M_ERR_INVALID, "state_dict tensor '" + kv.first +
                                     "' is not used by this engine (unsupported CHGNet configuration; refusing to ignore it)");
  }
  if (!e->elem_refs.empty()) {
    e->erefbuf.ensure(e->elem_refs.size());
    B2M_CK(cudaMemcpyAsync(e->erefbuf.p, e->elem_refs.data(), e->elem_refs.size() * sizeof(double), cudaMemcpyHostToDevice,
                           e->st));
  }
  e->wbuf.ensure(P.host.size() + 64);
  B2M_CK(cudaMemcpyAsync(e->wbuf.p, P.host.data(), P.host.size() * sizeof(float), cudaMemcpyHostToDevice, e->st));
  B2M_CK(cudaStreamSynchronize(e->st));
  auto dp = [&](const std::string& n) { return e->wbuf.p + off.at(n); };
  e->d_fa = dp("fa");
  e->d_emb = dp("emb");
  e->d_Wbe = dp("Wbe");
  e->d_Wae = dp("Wae");
  e->d_W3bw = dp("W3bw");
  e->d_c0 = dp("c0"), e->d_c1 = dp("c1"), e->d_F2 = dp("F2"), e->d_Ws = dp("Ws");
  e->d_eref = e->elem_refs.empty() ? nullptr : e->erefbuf.p;
  for (int l = 0; l < nb; l++) {
    const std::string q = "a" + std::to_string(l) + ".";
    AtomLayerW& w = e->aw[l];
    w.b1 = dp(q + "b1"), w.radial = dp(q + "radial"), w.W2can = dp(q + "W2can"), w.W2Tcan = dp(q + "W2Tcan"), w.b2 = dp(q + "b2");
  }
  for (int l = 0; l < nb - 1; l++) {
    const std::string q = "b" + std::to_string(l) + ".";
    BondLayerW& w = e->bw[l];
    w.Wgcan = dp(q + "Wgcan"), w.WgTcan = dp(q + "WgTcan"), w.b1 = dp(q + "b1");
    w.W2can = dp(q + "W2can"), w.W2Tcan = dp(q + "W2Tcan"), w.b2 = dp(q + "b2");
    w.WAgcan = dp(q + "WAgcan"), w.WAgTcan = dp(q + "WAgTcan"), w.bA = dp(q + "bA");
  }
  e->finalized = true;
}

// ------------------------------------------------------------------------------------------
static void alloc_workspace(b2m_engine* e) {
  Graph& g = e->g;
  const int nb = e->desc.n_blocks;
  const size_t nl = g.n_loc, no = g.n_own, bl = g.B_loc, bo = g.B_own;
  const size_t A = (size_t)g.A, E = (size_t)g.E;
  e->x.resize(nb + 1);
  e->h.resize(nb);
  e->ang.resize(nb - 1);
  e->upd.resize(nb - 1);
  for (auto& b : e->x) b.ensure(nl * D + 64);
  for (auto& b : e->h) b.ensure(bl * D + 64);
  const size_t Apad = (A + 127) / 128 * 128;  // whole 128-row tiles
  for (auto& b : e->ang) b.ensure(Apad * D + 64);
  for (auto& b : e->upd) b.ensure(bo * D + 64);
  e->ApL.resize(nb), e->CpL.resize(nb), e->QpL.resize(nb);
  for (int l = 0; l < nb; l++) {
    e->ApL[l].ensure(nl * D2 + 64), e->CpL[l].ensure(no * D2 + 64);
    if (l > 0) e->QpL[l].ensure(bo * D2 + 64);
  }
  e->Ha.ensure(bl * D2 + 64), e->Hb.ensure(bo * D2 + 64), e->Xc.ensure(nl * D2 + 64);
  e->agg.ensure(no * D + 64), e->aggB.ensure(bo * D + 64);
  e->y1p.ensure(no * D), e->y1.ensure(no * D), e->y2p.ensure(no * D), e->y2.ensure(no * D);
  e->e_atom.ensure(no), e->site.ensure(no);
  e->gx.ensure(nl * D + 64), e->gh.ensure(bl * D + 64), e->gang.ensure(Apad * D + 64);
  e->gA.ensure(nl * D2 + 64), e->gC.ensure(no * D2 + 64), e->gQ.ensure(bo * D2 + 64);
  e->gHa.ensure(bl * D2 + 64), e->gHb.ensure(bo * D2 + 64), e->gXc.ensure(nl * D2 + 64);
  e->gagg.ensure(no * D + 64), e->gupd.ensure(bo * D + 64), e->gaggB.ensure(bo * D + 64);
  e->gd.ensure(E + 64), e->gdb.ensure(bl + 64), e->gbvec.ensure(bl * 3 + 64);
  e->gy1.ensure(no * D), e->gy2.ensure(no * D);
  e->forces.ensure((size_t)g.N * 3 + 64);
  e->site_full.ensure((size_t)g.N + 64);
  e->scal.ensure(16);
  if (e->world > 1) {
    size_t tot_to = 0, tot_bto = 0;
    for (int q = 0; q < e->world; q++) tot_to += g.n_to[q], tot_bto += g.nb_to[q];
    size_t m = std::max(tot_to * D, tot_bto * D);
    if (e->leader != nullptr) {
      e->precv[0].ensure(m + 64), e->precv[1].ensure(m + 64);
    } else {
      e->sendbuf.ensure(m + 64);
      e->recvbuf.ensure(m + 64);
    }
  }
}

// ---- halo exchange between slab neighbours ----
// Two transports: NCCL point-to-point (one process per GPU, world > 1 with a communicator) and, inside a single-process
// group, direct peer-memory traffic: the sender's pack kernel stores its boundary rows straight into the receiver's halo
// rows (forward) or copies its halo adjoints into the owner's receive buffer (backward); a CUDA event per exchange point
// orders the receiver's stream behind the sender's.
// kind 0: atom rows x[l] | 1: bond rows h[l] | 2: TensorNet atom tensors X[l] (10 x 64 floats per atom)
//      3: MACE node features h[l] (C floats per atom, 4 C for 0e+1o features)
static float* halo_buffer(b2m_engine* e, int kind, int l) {
  if (kind == 3) return e->mace->h[l].p;
  return kind == 1 ? e->h[l].p : (kind == 2 ? e->tn->X[l].p : e->x[l].p);
}
static int halo_width(const b2m_engine* e, int kind, int l) {
  if (kind == 3) return e->mace->hw[l];
  return kind == 2 ? 10 * D : D;
}

static cudaEvent_t next_halo_event(b2m_engine* e) {
  // the events are created in b2m_create: a neighbour's thread reads hev[k] concurrently, so the vector never grows here
  B2M_REQUIRE(e->hpoint < (int)e->hev.size(), B2M_ERR_STATE, "too many halo-exchange points in one evaluation");
  return e->hev[e->hpoint];
}

// forward: rows of tensor (bonds ? h : x)[l] listed in to_list[q] -> q's halo section; my halo section <- owners.
// Split in two so that the exchange runs on the engine's second stream while the compute stream does the projections
// that do not read the halo rows (the reference issues its copies on the compute stream, dist.py:344-356):
//   halo_forward_begin: [compute: producer done] -> [comm stream: pack, send / receive or peer stores]
//   halo_forward_end  : compute stream waits for the exchange (and, in a group, for the neighbours' stores)
static void halo_forward_begin(b2m_engine* e, int kind, int l) {
  if (e->world <= 1 || e->debug_no_halo) return;
  Graph& g = e->g;
  const bool bonds = kind == 1;
  const size_t W = (size_t)halo_width(e, kind, l);
  float* buf = halo_buffer(e, kind, l);
  const int* nto = bonds ? g.nb_to : g.n_to;
  const int* toff = bonds ? g.bto_off : g.to_off;
  const int* nfrom = bonds ? g.nb_from : g.n_from;
  const int* foff = bonds ? g.bfrom_off : g.from_off;
  const int* list = bonds ? g.bto_list.p : g.to_list.p;
  const size_t base = bonds ? (size_t)g.B_own : (size_t)g.n_own;
  B2M_CK(cudaEventRecord(e->ev_prod, e->st));
  B2M_CK(cudaStreamWaitEvent(e->cst, e->ev_prod, 0));
  if (e->leader != nullptr) {
    b2m_engine* L = e->leader;
    for (int q = 0; q < e->world; q++) {
      if (q == e->rank || nto[q] <= 0) continue;
      b2m_engine* pe = L->parts[q];
      Graph& pg = pe->g;
      const int pn = bonds ? pg.nb_from[e->rank] : pg.n_from[e->rank];
      B2M_REQUIRE(pn == nto[q], B2M_ERR_STATE, "halo sections of two partitions disagree");
      const size_t pbase = bonds ? (size_t)pg.B_own : (size_t)pg.n_own;
      const size_t pfoff = bonds ? (size_t)pg.bfrom_off[e->rank] : (size_t)pg.from_off[e->rank];
      launch_gather_rows(e->cst, nto[q], (int)W, list + toff[q], buf, halo_buffer(pe, kind, l) + (pbase + pfoff) * W);
    }
    B2M_CK(cudaEventRecord(next_halo_event(e), e->cst));
    return;
  }
  for (int q = 0; q < e->world; q++)
    if (nto[q] > 0)
      launch_gather_rows(e->cst, nto[q], (int)W, list + toff[q], buf, e->sendbuf.p + (size_t)toff[q] * W);
  NCCL_CK(g_nccl.GroupStart());
  for (int q = 0; q < e->world; q++) {
    if (q == e->rank) continue;
    if (nto[q] > 0)
      NCCL_CK(g_nccl.Send(e->sendbuf.p + (size_t)toff[q] * W, (size_t)nto[q] * W, ncclFloat32, q, e->comm, e->cst));
    if (nfrom[q] > 0)
      NCCL_CK(g_nccl.Recv(buf + (base + foff[q]) * W, (size_t)nfrom[q] * W, ncclFloat32, q, e->comm, e->cst));
  }
  NCCL_CK(g_nccl.GroupEnd());
  B2M_CK(cudaEventRecord(e->ev_halo, e->cst));
}
static void halo_forward_end(b2m_engine* e) {
  if (e->world <= 1 || e->debug_no_halo) return;
  if (e->leader != nullptr) {
    b2m_engine* L = e->leader;
    const int k = e->hpoint++;
    L->gsync.arrive_and_wait();  // every partition has recorded its event for this point
    for (int q = 0; q < e->world; q++)  // own event too: my stores must precede any later reuse of the source rows
      B2M_CK(cudaStreamWaitEvent(e->st, L->parts[q]->hev[k], 0));
    return;
  }
  B2M_CK(cudaStreamWaitEvent(e->st, e->ev_halo, 0));
}
// backward: my halo rows of the adjoint -> owners (accumulate), then zero the halo rows
static void halo_backward(b2m_engine* e, float* gbuf, bool bonds, int width = D) {
  if (e->world <= 1 || e->debug_no_halo) return;
  Graph& g = e->g;
  const size_t W = (size_t)width;
  const int* nto = bonds ? g.nb_to : g.n_to;
  const int* toff = bonds ? g.bto_off : g.to_off;
  const int* nfrom = bonds ? g.nb_from : g.n_from;
  const int* foff = bonds ? g.bfrom_off : g.from_off;
  const int* list = bonds ? g.bto_list.p : g.to_list.p;
  const size_t base = bonds ? (size_t)g.B_own : (size_t)g.n_own;
  const size_t nhalo = bonds ? (size_t)g.B_halo : (size_t)g.n_halo;
  if (e->leader != nullptr) {
    b2m_engine* L = e->leader;
    const int k = e->hpoint;
    for (int q = 0; q < e->world; q++) {
      if (q == e->rank || nfrom[q] <= 0) continue;
      b2m_engine* pe = L->parts[q];
      const size_t ptoff = bonds ? (size_t)pe->g.bto_off[e->rank] : (size_t)pe->g.to_off[e->rank];
      // the owner's receive buffer of this parity was consumed two exchange points ago (see DESIGN.md, group mode)
      B2M_CK(cudaMemcpyAsync(pe->precv[k & 1].p + ptoff * W, gbuf + (base + foff[q]) * W, (size_t)nfrom[q] * W * sizeof(float),
                             cudaMemcpyDefault, e->st));
    }
    launch_zero_rows(e->st, gbuf + base * W, nhalo * W);
    cudaEvent_t ev = next_halo_event(e);
    B2M_CK(cudaEventRecord(ev, e->st));
    e->hpoint++;
    L->gsync.arrive_and_wait();
    for (int q = 0; q < e->world; q++)
      if (q != e->rank) B2M_CK(cudaStreamWaitEvent(e->st, L->parts[q]->hev[k], 0));
    for (int q = 0; q < e->world; q++)
      if (q != e->rank && nto[q] > 0)
        launch_scatter_add_rows(e->st, nto[q], (int)W, list + toff[q], e->precv[k & 1].p + (size_t)toff[q] * W, gbuf);
    return;
  }
  NCCL_CK(g_nccl.GroupStart());
  for (int q = 0; q < e->world; q++) {
    if (q == e->rank) continue;
    if (nfrom[q] > 0)
      NCCL_CK(g_nccl.Send(gbuf + (base + foff[q]) * W, (size_t)nfrom[q] * W, ncclFloat32, q, e->comm, e->st));
    if (nto[q] > 0)
      NCCL_CK(g_nccl.Recv(e->recvbuf.p + (size_t)toff[q] * W, (size_t)nto[q] * W, ncclFloat32, q, e->comm, e->st));
  }
  NCCL_CK(g_nccl.GroupEnd());
  for (int q = 0; q < e->world; q++)
    if (nto[q] > 0)
      launch_scatter_add_rows(e->st, nto[q], (int)W, list + toff[q], e->recvbuf.p + (size_t)toff[q] * W, gbuf);
  launch_zero_rows(e->st, gbuf + base * W, nhalo * W);
}

#include "engine_tn.inl"
#include "engine_mace.inl"

static AtomConvArgs atom_args(b2m_engine* e, int l) {
  Graph& g = e->g;
  const AtomLayerW& w = e->aw[l];
  AtomConvArgs a;
  memset(&a, 0, sizeof a);
  a.E = g.E;
  a.e_src = g.e_src.p, a.e_dst = g.e_dst.p, a.e_bond = g.e_bond.p, a.e_vec = g.e_vec.p;
  const int ps = e->proj_slot(l);
  a.Aproj = e->ApL[ps].p, a.Cproj = e->CpL[ps].p, a.Qproj = l > 0 ? e->QpL[ps].p : nullptr;
  a.radial = w.radial, a.W2can = w.W2can, a.W2Tcan = w.W2Tcan, a.b2 = w.b2;
  a.rp = e->rp2;
  return a;
}
static void atom_projections(b2m_engine* e, int l) {
  Graph& g = e->g;
  const AtomLayerW& w = e->aw[l];
  const int ps = e->proj_slot(l);
  tc_mm(e, e->x[l].p, D, w.W1s, e->ApL[ps].p, D2, g.n_loc, false);
  tc_mm(e, e->x[l].p, D, w.W1t, e->CpL[ps].p, D2, g.n_own, false, w.b1);
  if (l > 0) tc_mm(e, e->h[l].p, D, w.W1e, e->QpL[ps].p, D2, g.B_own, false);
}
static void atom_layer_fwd(b2m_engine* e, int l) {
  Graph& g = e->g;
  const AtomLayerW& w = e->aw[l];
  atom_projections(e, l);
  launch_zero_rows(e->st, e->agg.p, (int64_t)g.n_own * D);
  AtomConvArgs a = atom_args(e, l);
  a.agg = e->agg.p;
  cudaEvent_t e0, e1;
  B2M_CK(cudaEventCreate(&e0));
  B2M_CK(cudaEventCreate(&e1));
  B2M_CK(cudaEventRecord(e0, e->st));
  launch_atomconv_fwd(e->st, a, e->num_sms);
  B2M_CK(cudaEventRecord(e1, e->st));
  e->gather_ev.push_back({e0, e1});
  tc_mm(e, e->agg.p, D, w.Wout, e->x[l + 1].p, D, g.n_own, false, nullptr, e->x[l].p, D);
}
// in: gx = dE/dx[l+1] (owned rows valid, halo rows zero).  out: gx = dE/dx[l] (all local rows)
static void atom_layer_bwd(b2m_engine* e, int l) {
  Graph& g = e->g;
  const AtomLayerW& w = e->aw[l];
  tc_mm(e, e->gx.p, D, w.WoutT, e->gagg.p, D, g.n_own, false);
  // A / C / Q of this layer are still in their per-layer buffers from the forward: no recompute
  AtomConvArgs a = atom_args(e, l);
  a.gagg = e->gagg.p;
  a.gd = e->gd.p;
  const bool need_gx = l > 0;
  if (need_gx) {
    launch_zero_rows(e->st, e->gA.p, (int64_t)g.n_loc * D2);
    launch_zero_rows(e->st, e->gC.p, (int64_t)g.n_own * D2);
    a.gA = e->gA.p, a.gC = e->gC.p, a.gQ = e->gQ.p;
  }
  launch_atomconv_bwd(e->st, a, e->num_sms);
  if (need_gx) {
    tc_mm(e, e->gA.p, D2, w.W1sT, e->gx.p, D, g.n_loc, true);
    tc_mm(e, e->gC.p, D2, w.W1tT, e->gx.p, D, g.n_own, true);
    tc_mm(e, e->gQ.p, D2, w.W1eT, e->gh.p, D, g.B_own, true);
  }
}

static LineArgs line_args(b2m_engine* e, int l, bool hidden) {
  Graph& g = e->g;
  const BondLayerW& w = e->bw[l];
  LineArgs a;
  memset(&a, 0, sizeof a);
  a.A = g.A;
  a.a_in = g.a_in.p, a.a_out = g.a_out.p, a.a_ctr = g.a_ctr.p;
  a.ang = e->ang[l].p;
  a.Ha = e->Ha.p, a.Hb = e->Hb.p, a.Xc = e->Xc.p;
  if (hidden) {
    a.Wgcan = w.Wgcan, a.WgTcan = w.WgTcan, a.W2can = w.W2can, a.W2Tcan = w.W2Tcan, a.b2 = w.b2;
  } else {
    a.Wgcan = w.WAgcan, a.WgTcan = w.WAgTcan;
  }
  return a;
}
// first-layer projections of the line-graph MLPs: Ha / Hb from the bond features, Xc from the atom features
static void line_proj_Ha(b2m_engine* e, int l, bool hidden) {
  const BondLayerW& w = e->bw[l];
  const float* hsrc = hidden ? e->h[l].p : e->h[l + 1].p;
  tc_mm(e, hsrc, D, hidden ? w.W1a : w.WAa, e->Ha.p, D2, e->g.B_loc, false);
}
static void line_proj_Hb(b2m_engine* e, int l, bool hidden) {
  const BondLayerW& w = e->bw[l];
  const float* hsrc = hidden ? e->h[l].p : e->h[l + 1].p;
  tc_mm(e, hsrc, D, hidden ? w.W1b : w.WAb, e->Hb.p, D2, e->g.B_own, false, hidden ? w.b1 : w.bA);
}
static void line_proj_Xc(b2m_engine* e, int l, bool hidden) {
  const BondLayerW& w = e->bw[l];
  tc_mm(e, e->x[l + 1].p, D, hidden ? w.W1c : w.WAc, e->Xc.p, D2, e->g.n_loc, false);
}
static void line_projections(b2m_engine* e, int l, bool hidden) {
  line_proj_Ha(e, l, hidden), line_proj_Hb(e, l, hidden), line_proj_Xc(e, l, hidden);
}
static void line_bwd_common(b2m_engine* e, int l, bool hidden, LineArgs& a) {
  Graph& g = e->g;
  const BondLayerW& w = e->bw[l];
  launch_zero_rows(e->st, e->gHa.p, (int64_t)g.B_loc * D2);
  launch_zero_rows(e->st, e->gHb.p, (int64_t)g.B_own * D2);
  launch_zero_rows(e->st, e->gXc.p, (int64_t)g.n_loc * D2);
  a.gang = e->gang.p, a.gHa = e->gHa.p, a.gHb = e->gHb.p, a.gXc = e->gXc.p;
  launch_line_bwd(e->st, a, hidden, e->num_sms);
  tc_mm(e, e->gHa.p, D2, hidden ? w.W1aT : w.WAaT, e->gh.p, D, g.B_loc, true);
  tc_mm(e, e->gHb.p, D2, hidden ? w.W1bT : w.WAbT, e->gh.p, D, g.B_own, true);
  tc_mm(e, e->gXc.p, D2, hidden ? w.W1cT : w.WAcT, e->gx.p, D, g.n_loc, true);
}

static void forward(b2m_engine* e) {
  Graph& g = e->g;
  const int nb = e->desc.n_blocks;
  launch_embed(e->st, g.n_loc, g.type.p, e->d_emb, e->x[0].p);
  launch_bond_init(e->st, g.B_loc, g.b_vec.p, e->rp2, e->d_Wbe, e->h[0].p);
  launch_angle_init(e->st, g.A, g.a_in.p, g.a_out.p, g.b_vec.p, e->d_fa, e->d_Wae, e->ang[0].p);
  for (int l = 0; l < nb - 1; l++) {
    atom_layer_fwd(e, l);
    const BondLayerW& w = e->bw[l];
    // x^{l+1} halo rows travel while the two projections of the bond features run (they do not read x)
    halo_forward_begin(e, false, l + 1);
    line_proj_Ha(e, l, true), line_proj_Hb(e, l, true);
    halo_forward_end(e);
    line_proj_Xc(e, l, true);
    launch_zero_rows(e->st, e->aggB.p, (int64_t)g.B_own * D);
    LineArgs a = line_args(e, l, true);
    a.aggB = e->aggB.p;
    launch_line_fwd(e->st, a, true, e->num_sms);
    tc_mm(e, e->aggB.p, D, w.Wout, e->upd[l].p, D, g.B_own, false);
    launch_bond_update_fwd(e->st, g.B_own, g.b_vec.p, e->rp3, e->d_W3bw, e->h[l].p, e->upd[l].p, e->h[l + 1].p);
    if (l < nb - 2) {
      // the last block's angle update (and the halo copy of h feeding it) is dead code in the
      // reference (chgnet.py:353-368 on the last iteration): nothing reads it afterwards.
      // h^{l+1} halo rows travel while Hb (owned bonds only) and Xc (atoms) are projected; Ha reads the halo rows
      halo_forward_begin(e, true, l + 1);
      line_proj_Hb(e, l, false), line_proj_Xc(e, l, false);
      halo_forward_end(e);
      line_proj_Ha(e, l, false);
      LineArgs b = line_args(e, l, false);
      b.ang_out = e->ang[l + 1].p;
      launch_line_fwd(e->st, b, false, e->num_sms);
    }
  }
  // site-wise readout after block n-2 (chgnet.py:392-398)
  launch_rowdot(e->st, g.n_own, e->x[nb - 1].p, e->d_Ws, e->bs, e->site.p, nullptr, nullptr, nullptr, 1.f);
  atom_layer_fwd(e, nb - 1);
  // final MLP 64 -> 64 -> 64 -> 1, sum (chgnet.py:422-440); E = std * E + mean (+ element refs) (pes.py:109-113)
  tc_mm(e, e->x[nb].p, D, e->F0, e->y1p.p, D, g.n_own, false, e->d_c0);
  launch_silu(e->st, (int64_t)g.n_own * D, e->y1p.p, e->y1.p);
  tc_mm(e, e->y1.p, D, e->F1, e->y2p.p, D, g.n_own, false, e->d_c1);
  launch_silu(e->st, (int64_t)g.n_own * D, e->y2p.p, e->y2.p);
  B2M_CK(cudaMemsetAsync(e->scal.p, 0, 16 * sizeof(double), e->st));
  launch_rowdot(e->st, g.n_own, e->y2.p, e->d_F2, e->c2, e->e_atom.p, e->scal.p, g.type.p, e->d_eref,
                (float)e->desc.data_std, g.gid.p, e->atomic ? e->atom_e.p : nullptr, e->desc.data_mean / cell_atoms(e),
                e->hf_n ? e->hf_w.p : nullptr);
}

static void backward(b2m_engine* e) {
  Graph& g = e->g;
  const int nb = e->desc.n_blocks;
  launch_zero_rows(e->st, e->gd.p, g.E);
  launch_zero_rows(e->st, e->gdb.p, g.B_loc);
  launch_zero_rows(e->st, e->gbvec.p, (int64_t)g.B_loc * 3);
  launch_zero_rows(e->st, e->gh.p, (int64_t)g.B_loc * D);
  launch_zero_rows(e->st, e->gang.p, (g.A + 127) / 128 * 128 * D);
  launch_zero_rows(e->st, e->gx.p, (int64_t)g.n_loc * D);
  launch_zero_rows(e->st, e->forces.p, g.N * 3);
  // readout backward
  launch_readout_seed(e->st, g.n_own, e->y2p.p, e->d_F2, (float)e->desc.data_std, e->gy2.p, g.gid.p,
                      e->hf_n ? e->hf_w.p : nullptr);
  tc_mm(e, e->gy2.p, D, e->F1T, e->gy1.p, D, g.n_own, false);
  launch_dsilu_mul(e->st, (int64_t)g.n_own * D, e->y1p.p, e->gy1.p);
  tc_mm(e, e->gy1.p, D, e->F0T, e->gx.p, D, g.n_own, false);
  atom_layer_bwd(e, nb - 1);
  for (int l = nb - 2; l >= 0; l--) {
    const BondLayerW& w = e->bw[l];
    if (l < nb - 2) {
      // the first-layer projections of the angle update are recomputed (the buffers hold the next layer's)
      line_projections(e, l, false);
      LineArgs a = line_args(e, l, false);
      line_bwd_common(e, l, false, a);
      halo_backward(e, e->gh.p, true);
    }
    launch_bond_update_bwd(e->st, g.B_own, g.b_vec.p, e->rp3, e->d_W3bw, e->gh.p, e->upd[l].p, e->gupd.p, e->gdb.p);
    tc_mm(e, e->gupd.p, D, w.WoutT, e->gaggB.p, D, g.B_own, false);
    line_projections(e, l, true);
    LineArgs a = line_args(e, l, true);
    a.gaggB = e->gaggB.p;
    line_bwd_common(e, l, true, a);
    halo_backward(e, e->gx.p, false);
    atom_layer_bwd(e, l);
  }
  // geometry: h0 = W_be be(d_b), theta/Fourier, then edges -> forces and virial
  launch_h0_bwd(e->st, g.B_loc, g.b_vec.p, e->rp2, e->d_Wbe, e->gh.p, e->gdb.p);
  launch_angle_init_bwd(e->st, g.A, g.a_in.p, g.a_out.p, g.b_vec.p, e->d_fa, e->d_Wae, e->gang.p, e->gbvec.p);
  float* avir = e->atomic ? e->atom_vir.p : nullptr;
  launch_edge_final(e->st, g.E, g.e_src.p, g.e_dst.p, g.e_bond.p, g.e_vec.p, g.gid.p, e->gd.p, e->gdb.p, e->gbvec.p,
                    e->forces.p, e->scal.p + 1, avir);
  launch_halo_bond_final(e->st, g.B_own, g.B_loc, g.b_src_gid.p, g.b_dst.p, g.b_vec.p, g.gid.p, e->gdb.p, e->gbvec.p,
                         e->forces.p, e->scal.p + 1, avir);
}

// ------------------------------------------------------------------------------------------
// heat flux (DESIGN.md §10)
#define LAUNCH_HF(kern, n, st, ...)                              \
  do {                                                           \
    if ((n) > 0) {                                               \
      kern<<<cdiv((n), 256), 256, 0, st>>>(__VA_ARGS__);         \
      B2M_CK(cudaGetLastError());                                \
      g_launch_count++;                                          \
    }                                                            \
  } while (0)

// readout weight of every unfolded atom: images 0; cell atoms 1 (alpha < 0, the mask) or (r_j - c)_alpha (a seed)
__global__ void k_hf_weights(int64_t N, int64_t n, const double* __restrict__ cart, double cx, double cy, double cz,
                             int alpha, float* __restrict__ w) {
  const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (j >= N) return;
  const double c = alpha == 0 ? cx : alpha == 1 ? cy : cz;
  w[j] = j >= n ? 0.f : alpha < 0 ? 1.f : (float)(cart[3 * j + alpha] - c);
}

// out[image_of[j]][k] += src[j][k], k < width, rows of `pitch` floats (out zeroed before)
__global__ void k_hf_fold(int64_t N, const int* __restrict__ image_of, int width, int pitch,
                          const float* __restrict__ src, float* __restrict__ out) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= N * width) return;
  const int64_t j = t / width;
  const int k = (int)(t - j * width);
  atomicAdd(&out[(int64_t)image_of[j] * pitch + k], src[j * pitch + k]);
}

// J_pot^a = sum_j [ -F^a_j . v_j + (r_j - c)_a (F_j . v_j) ] over all unfolded atoms (F^a: forces of seed a, i.e. -G^a;
// F: forces of the masked pass; v_j the velocity of the cell atom j is an image of), J_conv^a = sum_{i<n} eps_i v_i,a.
// out[0..2] = J_pot, out[3..5] = J_conv, accumulated in f64.
__global__ void __launch_bounds__(256) k_hf_contract(int64_t N, int64_t n, const double* __restrict__ cart, double cx,
                                                     double cy, double cz, const int* __restrict__ image_of,
                                                     const double* __restrict__ vel, const float* __restrict__ F,
                                                     const float* __restrict__ FS, const double* __restrict__ eps,
                                                     double* __restrict__ out) {
  double acc[6] = {0, 0, 0, 0, 0, 0};
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < N; j += (int64_t)gridDim.x * blockDim.x) {
    const int i = image_of[j];
    const double v[3] = {vel[3 * i], vel[3 * i + 1], vel[3 * i + 2]};
    const double fv = F[3 * j] * v[0] + F[3 * j + 1] * v[1] + F[3 * j + 2] * v[2];
    const double r[3] = {cart[3 * j] - cx, cart[3 * j + 1] - cy, cart[3 * j + 2] - cz};
#pragma unroll
    for (int a = 0; a < 3; a++) {
      const float* Fa = FS + (size_t)a * N * 3 + 3 * j;
      acc[a] += r[a] * fv - (Fa[0] * v[0] + Fa[1] * v[1] + Fa[2] * v[2]);
      if (j < n) acc[3 + a] += eps[j] * v[a];
    }
  }
  __shared__ double red[6][8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 6; k++) {
    double x = acc[k];
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if (lane == 0) red[k][warp] = x;
  }
  __syncthreads();
  if (threadIdx.x < 6) {
    double s = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += red[threadIdx.x][w];
    atomicAdd(&out[threadIdx.x], s);
  }
}

static void run(b2m_engine* e, bool grads) {
  B2M_REQUIRE(e->finalized, B2M_ERR_STATE, "weights not finalized");
  B2M_REQUIRE(e->have_graph, B2M_ERR_STATE, "b2m_set_structure has not been called");
  B2M_REQUIRE(e->world == 1 || e->comm != nullptr || e->leader != nullptr || e->debug_no_halo, B2M_ERR_STATE,
              "world > 1 without a communicator (b2m_set_partition is a graph-only view)");
  e->hpoint = 0;
  for (auto& p : e->gather_ev) {
    cudaEventDestroy(p.first);
    cudaEventDestroy(p.second);
  }
  e->gather_ev.clear();
  const long long l0 = g_launch_count;
  B2M_CK(cudaEventRecord(e->ev[0], e->st));
  e->want_grads = grads;
  const size_t N = (size_t)e->g.N;
  if (e->atomic) {  // zeroed here, before the readout writes the energies and the backward accumulates the virials
    e->atom_e.ensure(N + 64);
    e->atom_e.zero(N, e->st);
    if (grads) {
      e->atom_vir.ensure(N * kVirPitch + 64);
      e->atom_vir.zero(N * kVirPitch, e->st);
    }
  }
  e->atomic_last = 0;
  if (e->hf_n) {
    LAUNCH_HF(k_hf_weights, e->g.N, e->st, e->g.N, e->hf_n, e->g.cart.p, e->hf_c[0], e->hf_c[1], e->hf_c[2], e->hf_seed,
              e->hf_w.p);
  }
  if (e->kind == 1) tn_forward(e);
  else if (e->kind == 2) mace_forward(e);
  else forward(e);
  B2M_CK(cudaEventRecord(e->ev[1], e->st));
  if (grads) {
    if (e->kind == 1) tn_backward(e);
    else if (e->kind == 2) mace_backward(e);
    else backward(e);
  }
  if (e->world > 1 && e->leader == nullptr && !e->debug_no_halo) {
    NCCL_CK(g_nccl.AllReduce(e->scal.p, e->scal.p, 10, ncclFloat64, ncclSum, e->comm, e->st));
    if (grads)
      NCCL_CK(g_nccl.AllReduce(e->forces.p, e->forces.p, (size_t)e->g.N * 3, ncclFloat32, ncclSum, e->comm, e->st));
    if (e->atomic) {
      NCCL_CK(g_nccl.AllReduce(e->atom_e.p, e->atom_e.p, N, ncclFloat64, ncclSum, e->comm, e->st));
      if (grads)
        NCCL_CK(g_nccl.AllReduce(e->atom_vir.p, e->atom_vir.p, N * kVirPitch, ncclFloat32, ncclSum, e->comm, e->st));
    }
  }
  B2M_CK(cudaEventRecord(e->ev[2], e->st));
  B2M_CK(cudaStreamSynchronize(e->st));
  e->launches_last = g_launch_count - l0;
  e->atomic_last = e->atomic ? (grads ? 2 : 1) : 0;
  float ms;
  B2M_CK(cudaEventElapsedTime(&ms, e->ev[0], e->ev[1]));
  e->t_fwd = ms;
  B2M_CK(cudaEventElapsedTime(&ms, e->ev[1], e->ev[2]));
  e->t_bwd = ms;
  double tg = 0;
  for (auto& p : e->gather_ev) {
    B2M_CK(cudaEventElapsedTime(&ms, p.first, p.second));
    tg += ms;
  }
  e->t_gather = e->gather_ev.empty() ? 0 : tg / e->gather_ev.size();
  e->t_total = e->t_fwd + e->t_bwd;
}

// parallel host copy (page-locked <-> pageable): a handful of threads saturate the host memory system, one does not
static void par_memcpy(void* dst, const void* src, size_t bytes) {
  const size_t kMin = 4u << 20;
  unsigned nt = (unsigned)std::min<size_t>(4, bytes / kMin);
  if (nt <= 1) {
    memcpy(dst, src, bytes);
    return;
  }
  std::vector<std::thread> th;
  const size_t chunk = (bytes / nt + 4095) & ~(size_t)4095;
  for (unsigned t = 0; t < nt; t++) {
    const size_t o = (size_t)t * chunk;
    if (o >= bytes) break;
    const size_t n = std::min(chunk, bytes - o);
    th.emplace_back([=] { memcpy((char*)dst + o, (const char*)src + o, n); });
  }
  for (auto& x : th) x.join();
}
static void ensure_pinned(void*& p, size_t& cap, size_t bytes) {
  if (bytes <= cap) return;
  if (p) cudaFreeHost(p);
  p = nullptr, cap = 0;
  B2M_CK(cudaHostAlloc(&p, bytes + bytes / 8, cudaHostAllocDefault));
  cap = bytes + bytes / 8;
}

__global__ void k_add_inplace(int64_t n, const float* __restrict__ src, float* __restrict__ dst) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) dst[i] += src[i];
}
__global__ void k_add_inplace_f64(int64_t n, const double* __restrict__ src, double* __restrict__ dst) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < n) dst[i] += src[i];
}

// Runs fn(partition) for every partition of a group, one host thread each (each sets its own device); the first
// exception wins and releases the others from the rendezvous.
template <class F>
static void for_each_part(b2m_engine* L, F fn) {
  const int n = (int)L->parts.size();
  L->gsync.reset(n);
  std::vector<std::string> errs(n);
  std::vector<int> codes(n, 0);
  std::vector<std::thread> th;
  for (int p = 0; p < n; p++)
    th.emplace_back([&, p] {
      try {
        B2M_CK(cudaSetDevice(L->parts[p]->device));
        fn(L->parts[p]);
      } catch (const b2m::Error& ex) {
        codes[p] = ex.code, errs[p] = ex.what();
        L->gsync.abort();
      } catch (const std::exception& ex) {
        codes[p] = B2M_ERR_INVALID, errs[p] = ex.what();
        L->gsync.abort();
      }
    });
  for (auto& t : th) t.join();
  cudaSetDevice(L->device);
  for (int p = 0; p < n; p++)
    if (codes[p] != 0 && errs[p].find("a partition of the group failed") == std::string::npos)
      throw Error(codes[p], "partition " + std::to_string(p) + ": " + errs[p]);
  for (int p = 0; p < n; p++)
    if (codes[p] != 0) throw Error(codes[p], errs[p]);
}

static void run_any(b2m_engine* e, bool grads) {
  if (e->parts.empty()) {
    run(e, grads);
    return;
  }
  for_each_part(e, [&](b2m_engine* pe) { run(pe, grads); });
  // slowest partition = the group's device time; launches summed
  long long launches = 0;
  for (auto* pe : e->parts) {
    e->t_fwd = std::max(e->t_fwd, pe->t_fwd), e->t_bwd = std::max(e->t_bwd, pe->t_bwd);
    e->t_total = std::max(e->t_total, pe->t_total);
    launches += pe->launches_last;
  }
  e->launches_last = launches;
}

// forces [N][3] of the whole structure on the leader's device: a group sums its partitions' arrays, a multi-process run
// has all-reduced them in run()
static const float* summed_forces(b2m_engine* e) {
  if (e->parts.empty()) return e->forces.p;
  const size_t n = (size_t)e->g.N * 3;
  e->ftmp.ensure(n + 64);
  e->fsum.ensure(n + 64);
  B2M_CK(cudaMemcpyAsync(e->fsum.p, e->forces.p, n * sizeof(float), cudaMemcpyDeviceToDevice, e->st));
  for (size_t p = 1; p < e->parts.size(); p++) {
    B2M_CK(cudaMemcpyAsync(e->ftmp.p, e->parts[p]->forces.p, n * sizeof(float), cudaMemcpyDefault, e->st));
    k_add_inplace<<<cdiv((int64_t)n, 256), 256, 0, e->st>>>((int64_t)n, e->ftmp.p, e->fsum.p);
    B2M_CK(cudaGetLastError());
  }
  return e->fsum.p;
}

// unfolded graph: rows [N][pitch] of every unfolded atom summed onto their cell atoms -> [n][pitch] (hf_fold)
static const float* fold_rows(b2m_engine* e, const float* src, int width, int pitch) {
  const int64_t N = e->g.N, n = e->hf_n;
  e->hf_fold.ensure((size_t)n * pitch + 64);
  e->hf_fold.zero((size_t)n * pitch, e->st);
  LAUNCH_HF(k_hf_fold, N * width, e->st, N, e->uf.image_of.p, width, pitch, src, e->hf_fold.p);
  return e->hf_fold.p;
}

static void fetch(b2m_engine* e, double* energy, float* forces, float* stress9) {
  double hs[10];
  B2M_CK(cudaMemcpyAsync(hs, e->scal.p, 10 * sizeof(double), cudaMemcpyDeviceToHost, e->st));
  const float* fsrc = forces ? summed_forces(e) : nullptr;
  if (forces && e->hf_n) fsrc = fold_rows(e, fsrc, 3, 3);  // periodic forces F_i = sum of F~ over i and its images
  const size_t fbytes = (size_t)cell_atoms(e) * 3 * sizeof(float);
  if (forces) {
    ensure_pinned(e->pin_out, e->pin_out_cap, fbytes);
    B2M_CK(cudaMemcpyAsync(e->pin_out, fsrc, fbytes, cudaMemcpyDeviceToHost, e->st));
  }
  B2M_CK(cudaStreamSynchronize(e->st));
  if (forces) par_memcpy(forces, e->pin_out, fbytes);
  for (size_t p = 1; p < e->parts.size(); p++) {  // energy and virial of the other partitions
    double ps[10];
    b2m_engine* pe = e->parts[p];
    B2M_CK(cudaSetDevice(pe->device));
    B2M_CK(cudaMemcpy(ps, pe->scal.p, 10 * sizeof(double), cudaMemcpyDeviceToHost));
    for (int k = 0; k < 10; k++) hs[k] += ps[k];
  }
  if (!e->parts.empty()) B2M_CK(cudaSetDevice(e->device));
  e->last_energy = hs[0] + e->desc.data_mean;
  if (energy) *energy = e->last_energy;
  if (stress9)
    for (int k = 0; k < 9; k++) stress9[k] = (float)(hs[1 + k] / e->g.volume * 160.21766208);  // pes.py:140-145
}

// per-atom energies [N] and virials [N][9] of the last evaluation; a group sums its partitions' arrays on the leader's
// device (energies: each atom has one owner; virials: every partition adds the edges and bond parts it holds), a
// multi-process run has all-reduced them in run()
static void fetch_atomic(b2m_engine* e, double* energies, float* virials) {
  const size_t N = (size_t)cell_atoms(e), NG = (size_t)e->g.N;  // unfolded graph: cell atoms out, all atoms summed
  const double* esrc = e->atom_e.p;
  const float* vsrc = e->atom_vir.p;
  if (!e->parts.empty()) {
    auto sum = [&](auto& total, auto& tmp, auto member_buf, size_t n, auto add) {
      total.ensure(n + 64);
      tmp.ensure(n + 64);
      B2M_CK(cudaMemcpyAsync(total.p, member_buf(e).p, n * sizeof(*total.p), cudaMemcpyDeviceToDevice, e->st));
      for (size_t p = 1; p < e->parts.size(); p++) {
        B2M_CK(cudaMemcpyAsync(tmp.p, member_buf(e->parts[p]).p, n * sizeof(*total.p), cudaMemcpyDefault, e->st));
        add<<<cdiv((int64_t)n, 256), 256, 0, e->st>>>((int64_t)n, tmp.p, total.p);
        B2M_CK(cudaGetLastError());
      }
      return total.p;
    };
    if (energies) esrc = sum(e->aesum, e->aetmp, [](b2m_engine* m) -> DBuf<double>& { return m->atom_e; }, NG, k_add_inplace_f64);
    if (virials)
      vsrc = sum(e->avsum, e->avtmp, [](b2m_engine* m) -> DBuf<float>& { return m->atom_vir; }, NG * kVirPitch, k_add_inplace);
  }
  // images carry no energy (weight 0); their virial halves belong to the cell atoms they are images of
  if (virials && e->hf_n) vsrc = fold_rows(e, vsrc, 9, kVirPitch);
  const size_t vbytes = N * kVirPitch * sizeof(float);
  if (virials) {
    ensure_pinned(e->pin_out, e->pin_out_cap, vbytes);
    B2M_CK(cudaMemcpyAsync(e->pin_out, vsrc, vbytes, cudaMemcpyDeviceToHost, e->st));
  }
  if (energies) B2M_CK(cudaMemcpyAsync(energies, esrc, N * sizeof(double), cudaMemcpyDeviceToHost, e->st));
  B2M_CK(cudaStreamSynchronize(e->st));
  if (virials) {
    const float* w = static_cast<const float*>(e->pin_out);
    for (size_t i = 0; i < N; i++) memcpy(virials + i * 9, w + i * kVirPitch, 9 * sizeof(float));
  }
}

// One forward + backward per readout weight: the three seeds (r_j - c)_alpha, then the cell mask, so that the handle is
// left holding the masked (periodic) evaluation for fetch / b2m_get_results / b2m_get_atomic.  Every pass re-runs the
// forward: the backward recomputes its projection buffers in place, so a second backward on the same forward state is
// not possible without keeping copies of them.
static void heat_flux(b2m_engine* h, const double* vel, double* flux6) {
  const int64_t N = h->g.N, n = h->hf_n;
  const std::vector<b2m_engine*> members = h->parts.empty() ? std::vector<b2m_engine*>{h} : h->parts;
  std::vector<bool> atomic_flag;
  for (auto* e : members) atomic_flag.push_back(e->atomic);
  auto restore = [&] {  // the handle's own state: masked readout, its b2m_set_atomic flag
    for (size_t k = 0; k < members.size(); k++) members[k]->hf_seed = -1, members[k]->atomic = atomic_flag[k];
  };
  try {
    h->hf_G.ensure((size_t)N * 9 + 64);
    for (int a = 0; a < 3; a++) {
      for (auto* e : members) e->hf_seed = a;
      run_any(h, true);
      B2M_CK(cudaMemcpyAsync(h->hf_G.p + (size_t)a * N * 3, summed_forces(h), (size_t)N * 3 * sizeof(float),
                             cudaMemcpyDeviceToDevice, h->st));
    }
    // the masked pass also writes the per-atom energies (J_conv) whatever the handle's b2m_set_atomic flag
    for (auto* e : members) e->hf_seed = -1, e->atomic = true;
    run_any(h, true);
  } catch (...) {
    restore();
    throw;
  }
  restore();
  const float* F = summed_forces(h);
  const double* eps = h->atom_e.p;
  if (!h->parts.empty()) {
    h->aesum.ensure(N + 64);
    h->aetmp.ensure(N + 64);
    B2M_CK(cudaMemcpyAsync(h->aesum.p, h->atom_e.p, N * sizeof(double), cudaMemcpyDeviceToDevice, h->st));
    for (size_t p = 1; p < h->parts.size(); p++) {
      B2M_CK(cudaMemcpyAsync(h->aetmp.p, h->parts[p]->atom_e.p, N * sizeof(double), cudaMemcpyDefault, h->st));
      k_add_inplace_f64<<<cdiv(N, 256), 256, 0, h->st>>>(N, h->aetmp.p, h->aesum.p);
      B2M_CK(cudaGetLastError());
    }
    eps = h->aesum.p;
  }
  h->hf_vel.ensure((size_t)n * 3 + 64);
  h->hf_out.ensure(64);
  B2M_CK(cudaMemcpyAsync(h->hf_vel.p, vel, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, h->st));
  h->hf_out.zero(6, h->st);
  const int grid = std::max(1, std::min(cdiv(N, 256), 4 * h->num_sms));
  k_hf_contract<<<grid, 256, 0, h->st>>>(N, n, h->g.cart.p, h->hf_c[0], h->hf_c[1], h->hf_c[2], h->uf.image_of.p,
                                         h->hf_vel.p, F, h->hf_G.p, eps, h->hf_out.p);
  B2M_CK(cudaGetLastError());
  g_launch_count++;
  B2M_CK(cudaMemcpyAsync(flux6, h->hf_out.p, 6 * sizeof(double), cudaMemcpyDeviceToHost, h->st));
  B2M_CK(cudaStreamSynchronize(h->st));
}

}  // namespace b2m

// ==========================================================================================
// C ABI
// ==========================================================================================
#define API_BEGIN                               \
  if (!h) return B2M_ERR_INVALID;               \
  try {                                         \
    cudaSetDevice(h->device);
#define API_END                                 \
  }                                             \
  catch (const b2m::Error& ex) {                \
    h->err = ex.what();                         \
    return ex.code;                             \
  }                                             \
  catch (const std::exception& ex) {            \
    h->err = ex.what();                         \
    return B2M_ERR_INVALID;                     \
  }                                             \
  return B2M_OK;

static std::string g_create_err;

// partition of a single-process group that the inspection calls address (b2m_set_view; the handle itself otherwise)
static b2m_engine* viewed(b2m_engine* h) { return h->parts.empty() ? h : h->parts[h->view]; }

// every partition of a single-process group holds the replicated weights (chgnet.py:455-549 deep-copies them per GPU)
template <class F>
static void each_member(b2m_engine* h, F fn) {
  if (h->parts.empty()) {
    fn(h);
    return;
  }
  for (auto* pe : h->parts) {
    B2M_CK(cudaSetDevice(pe->device));
    fn(pe);
  }
  B2M_CK(cudaSetDevice(h->device));
}


extern "C" {

static b2m_engine* create_one(const b2m_model_desc* desc, int device, int count) {
  B2M_REQUIRE(device >= 0 && device < count, B2M_ERR_INVALID, "bad device ordinal");
  b2m_engine* e = new b2m_engine();
  try {
    e->desc = *desc;
    e->device = device;
    B2M_CK(cudaSetDevice(e->device));
    cudaDeviceProp prop;
    B2M_CK(cudaGetDeviceProperties(&prop, e->device));
    if (prop.major != 9 || prop.minor != 0) throw Error(B2M_ERR_CUDA, "libb200mlip is built for sm_90a (H100) only");
    e->num_sms = prop.multiProcessorCount;
    const char* nh = getenv("B2M_DEBUG_NO_HALO");
    e->debug_no_halo = nh && nh[0] == '1';
    B2M_CK(cudaStreamCreateWithFlags(&e->st, cudaStreamNonBlocking));
    B2M_CK(cudaStreamCreateWithFlags(&e->cst, cudaStreamNonBlocking));
    B2M_CK(cudaEventCreateWithFlags(&e->ev_prod, cudaEventDisableTiming));
    B2M_CK(cudaEventCreateWithFlags(&e->ev_halo, cudaEventDisableTiming));
    for (auto& ev : e->ev) B2M_CK(cudaEventCreate(&ev));
  } catch (...) {
    delete e;
    throw;
  }
  return e;
}

static int create_any(const b2m_model_desc* desc, const b2m_tensornet_desc* tdesc, const int* devices, int ndev,
                      b2m_handle* out, const b2m_mace_desc* mdesc = nullptr) {
  if (!desc || !devices || !out) return B2M_ERR_INVALID;
  std::vector<b2m_engine*> made;
  try {
    B2M_REQUIRE(ndev >= 1 && ndev <= MAXP, B2M_ERR_PARTITIONS, "ndev must be in [1,16]");
    if (mdesc) {
      B2M_REQUIRE(mdesc->channels >= 32 && mdesc->channels <= 128 && mdesc->channels % 32 == 0, B2M_ERR_INVALID,
                  "MACE engine supports hidden_irreps = C x 0e (+ C x 1o) with C a multiple of 32, C <= 128");
      B2M_REQUIRE(mdesc->hidden_max_l == 0 || mdesc->hidden_max_l == 1, B2M_ERR_INVALID,
                  "MACE engine supports hidden_max_l 0 (C x 0e) or 1 (C x 0e + C x 1o)");
      B2M_REQUIRE(mdesc->hidden_max_l == 0 || mdesc->max_ell >= 1, B2M_ERR_INVALID,
                  "0e+1o hidden features need max_ell >= 1");
      B2M_REQUIRE(mdesc->max_ell >= 0 && mdesc->max_ell <= 3, B2M_ERR_INVALID, "MACE engine supports max_ell <= 3");
      B2M_REQUIRE(mdesc->correlation >= 1 && mdesc->correlation <= 3, B2M_ERR_INVALID, "MACE engine supports correlation <= 3");
      B2M_REQUIRE(mdesc->num_interactions >= 1 && mdesc->num_interactions <= kMaceMaxLayers, B2M_ERR_INVALID,
                  "num_interactions must be in [1,8]");
      B2M_REQUIRE(mdesc->num_bessel >= 1 && mdesc->num_bessel <= 64, B2M_ERR_INVALID, "num_bessel must be in [1,64]");
      B2M_REQUIRE(mdesc->mlp_hidden >= 1 && mdesc->mlp_hidden <= 256, B2M_ERR_INVALID, "readout MLP width must be in [1,256]");
      B2M_REQUIRE(mdesc->num_polynomial_cutoff >= 1 && mdesc->r_max > 0 && mdesc->c_act > 0, B2M_ERR_INVALID,
                  "r_max, the cutoff exponent and c_act must be positive");
      for (int t = 0; t < mdesc->num_interactions; t++)
        B2M_REQUIRE(mdesc->avg_num_neighbors[t] > 0, B2M_ERR_INVALID, "avg_num_neighbors must be positive");
    } else if (tdesc) {
      B2M_REQUIRE(tdesc->units == D, B2M_ERR_INVALID, "TensorNet engine supports units = 64");
      B2M_REQUIRE(tdesc->num_rbf >= 1 && tdesc->num_rbf <= 64, B2M_ERR_INVALID, "num_rbf must be in [1,64]");
      B2M_REQUIRE(tdesc->n_blocks >= 1 && tdesc->n_blocks <= 16, B2M_ERR_INVALID, "nblocks must be in [1,16]");
      B2M_REQUIRE(tdesc->cutoff > 0 && tdesc->rbf_width > 0, B2M_ERR_INVALID, "cutoff and rbf width must be positive");
    } else {
      B2M_REQUIRE(desc->dim == D && desc->max_n == NR && desc->max_f == 4, B2M_ERR_INVALID,
                  "engine supports dim=64, max_n=9, max_f=4");
      B2M_REQUIRE(desc->n_blocks >= 2 && desc->n_blocks <= 16, B2M_ERR_INVALID, "n_blocks must be in [2,16]");
      B2M_REQUIRE(desc->cutoff > 0 && desc->three_body_cutoff > 0 && desc->three_body_cutoff <= desc->cutoff,
                  B2M_ERR_INVALID, "bond_r cannot be greater than regular cutoff");
    }
    int count = 0;
    cudaError_t ce = cudaGetDeviceCount(&count);
    if (ce != cudaSuccess || count <= 0)
      throw Error(B2M_ERR_CUDA, std::string("no CUDA device available (libb200mlip has no CPU fallback): ") +
                                    cudaGetErrorString(ce));
    for (int p = 0; p < ndev; p++) {
      made.push_back(create_one(desc, devices[p], count));
      if (mdesc) {
        b2m_engine* m = made.back();
        m->kind = 2;
        m->mace = new MaceState();
        MaceState& M = *m->mace;
        M.Cr = mdesc->channels, M.C = (mdesc->channels + 63) / 64 * 64;
        M.L1 = mdesc->max_ell + 1, M.nsh = M.L1 * M.L1, M.T = mdesc->num_interactions;
        M.correlation = mdesc->correlation, M.H = mdesc->mlp_hidden, M.c_act = mdesc->c_act;
        M.hidden_max_l = mdesc->hidden_max_l;
        M.hw.assign(M.T + 1, M.C);  // h[t] of 0 < t < T carries 0e+1o when hidden_max_l = 1
        for (int t = 1; t < M.T; t++) M.hw[t] = M.hidden_max_l ? 4 * M.C : M.C;
        M.rp.nb = mdesc->num_bessel, M.rp.nbp = 64, M.rp.p = mdesc->num_polynomial_cutoff;
        M.rp.r_max = (float)mdesc->r_max, M.rp.pref = (float)std::sqrt(2.0 / mdesc->r_max);
        for (int t = 0; t < M.T; t++)
          M.interaction_residual[t] = (mdesc->residual_mask >> t) & 1, M.avg_nb[t] = mdesc->avg_num_neighbors[t];
      } else if (tdesc) {
        b2m_engine* m = made.back();
        m->kind = 1;
        m->tn = new TnState();
        m->tn->units = tdesc->units, m->tn->num_rbf = tdesc->num_rbf, m->tn->nblocks = tdesc->n_blocks;
        m->tn->so3 = tdesc->so3 ? 1 : 0;
        m->tn->rp.nr = tdesc->num_rbf, m->tn->rp.nrp = 64;
        m->tn->rp.width = (float)tdesc->rbf_width, m->tn->rp.rc = (float)tdesc->cutoff;
        for (float& v : m->tn->rp.mu) v = 0.f;
      }
    }
    b2m_engine* e = made[0];
    if (ndev > 1) {
      // single-process group: partition p lives on devices[p] (ordinals may repeat: several partitions on one GPU);
      // peer access between distinct devices so that halo rows are plain stores into the neighbour's memory
      for (int p = 0; p < ndev; p++) {
        made[p]->rank = p, made[p]->world = ndev, made[p]->leader = e;
        B2M_CK(cudaSetDevice(made[p]->device));
        made[p]->hev.resize(4 * 16 + 8);  // 2 forward + 2 backward exchange points per block, n_blocks <= 16
        for (auto& ev : made[p]->hev) B2M_CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        for (int q = 0; q < ndev; q++) {
          if (made[q]->device == made[p]->device) continue;
          int can = 0;
          B2M_CK(cudaDeviceCanAccessPeer(&can, made[p]->device, made[q]->device));
          B2M_REQUIRE(can, B2M_ERR_CUDA, "devices of a single-process group need peer access (NVLink / NVSwitch)");
          cudaError_t pe = cudaDeviceEnablePeerAccess(made[q]->device, 0);
          if (pe == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
          else B2M_CK(pe);
        }
      }
      e->parts = made;
      B2M_CK(cudaSetDevice(e->device));
    }
    *out = e;
  } catch (const b2m::Error& ex) {
    for (auto* m : made) {
      delete m->tn;
      delete m->mace;
      delete m;
    }
    g_create_err = ex.what();
    return ex.code;
  }
  return B2M_OK;
}

int b2m_create(const b2m_model_desc* desc, const int* devices, int ndev, b2m_handle* out) {
  return create_any(desc, nullptr, devices, ndev, out);
}

int b2m_create_tensornet(const b2m_tensornet_desc* tdesc, const int* devices, int ndev, b2m_handle* out) {
  if (!tdesc) return B2M_ERR_INVALID;
  // the shared part of the engine (graph build, scaling, transport) reads the CHGNet-shaped description: no bond graph
  // (use_bond_graph False, three_body_cutoff 0: pes.py:79-80)
  b2m_model_desc d;
  memset(&d, 0, sizeof d);
  d.n_elem = tdesc->n_elem, d.dim = D, d.max_n = NR, d.max_f = 4, d.n_blocks = tdesc->n_blocks, d.cutoff_exponent = 0;
  d.cutoff = tdesc->cutoff, d.three_body_cutoff = 0.0, d.data_mean = tdesc->data_mean, d.data_std = tdesc->data_std;
  return create_any(&d, tdesc, devices, ndev, out);
}

int b2m_create_mace(const b2m_mace_desc* mdesc, const int* devices, int ndev, b2m_handle* out) {
  if (!mdesc) return B2M_ERR_INVALID;
  // the shared part of the engine (graph build, transport) reads the CHGNet-shaped description: no bond graph, r_max as
  // the cutoff, no Potential scaling (scale, shift and E0 are part of the model)
  b2m_model_desc d;
  memset(&d, 0, sizeof d);
  d.n_elem = mdesc->n_elem, d.dim = D, d.max_n = NR, d.max_f = 4, d.n_blocks = mdesc->num_interactions;
  d.cutoff = mdesc->r_max, d.three_body_cutoff = 0.0, d.data_mean = 0.0, d.data_std = 1.0;
  return create_any(&d, nullptr, devices, ndev, out, mdesc);
}

static void destroy_one(b2m_engine* h) {
  cudaSetDevice(h->device);
  delete h->tn;  // frees its device buffers
  delete h->mace;
  if (h->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(h->comm);
  for (auto& p : h->gather_ev) {
    cudaEventDestroy(p.first);
    cudaEventDestroy(p.second);
  }
  for (auto& ev : h->ev)
    if (ev) cudaEventDestroy(ev);
  for (auto& ev : h->hev) cudaEventDestroy(ev);
  if (h->pin_in) cudaFreeHost(h->pin_in);
  if (h->pin_out) cudaFreeHost(h->pin_out);
  if (h->ev_prod) cudaEventDestroy(h->ev_prod);
  if (h->ev_halo) cudaEventDestroy(h->ev_halo);
  if (h->cst) cudaStreamDestroy(h->cst);
  if (h->st) cudaStreamDestroy(h->st);
  delete h;
}

int b2m_destroy(b2m_handle h) {
  if (!h) return B2M_ERR_INVALID;
  std::vector<b2m_engine*> members(h->parts.begin(), h->parts.end());
  for (size_t p = 1; p < members.size(); p++) destroy_one(members[p]);
  destroy_one(h);
  return B2M_OK;
}

const char* b2m_last_error(b2m_handle h) { return h ? h->err.c_str() : g_create_err.c_str(); }

int b2m_load_weights(b2m_handle h, const char* name, const float* host_ptr, const int64_t* shape, int ndim) {
  API_BEGIN
  // up to 5 dimensions: the 1o symmetric-contraction tensor U_matrix_3 of MACE is [3, nsh, nsh, nsh, K]
  B2M_REQUIRE(name && host_ptr && shape && ndim >= 1 && ndim <= 5, B2M_ERR_INVALID, "bad weight arguments");
  size_t n = 1;
  std::vector<int64_t> sh(shape, shape + ndim);
  for (auto s : sh) n *= (size_t)s;
  each_member(h, [&](b2m_engine* e) {
    e->host_w[name] = std::vector<float>(host_ptr, host_ptr + n);
    e->host_shape[name] = sh;
    e->finalized = false;
  });
  API_END
}

int b2m_set_element_refs(b2m_handle h, const double* offsets, int n) {
  API_BEGIN
  B2M_REQUIRE(h->kind != 2, B2M_ERR_INVALID, "a MACE model carries its own atomic energies (atomic_energies_fn)");
  B2M_REQUIRE(offsets == nullptr || n == 0 || n == h->desc.n_elem, B2M_ERR_INVALID, "element_refs length must equal n_elem");
  each_member(h, [&](b2m_engine* e) {
    if (offsets == nullptr || n == 0) {  // clear: a later Potential without element_refs must not inherit the old offsets
      e->elem_refs.clear();
      e->d_eref = nullptr;
    } else {
      e->elem_refs.assign(offsets, offsets + n);
    }
    e->finalized = false;
  });
  API_END
}

int b2m_set_scaling(b2m_handle h, double data_mean, double data_std) {
  API_BEGIN
  B2M_REQUIRE(h->kind != 2, B2M_ERR_INVALID, "a MACE model carries its own scale and shift (scale_shift)");
  each_member(h, [&](b2m_engine* e) {
    e->desc.data_mean = data_mean;
    e->desc.data_std = data_std;
  });
  API_END
}

int b2m_finalize_weights(b2m_handle h) {
  API_BEGIN
  each_member(h, [&](b2m_engine* e) {
    if (e->kind == 1) tn_finalize_weights(e);
    else if (e->kind == 2) mace_finalize_weights(e);
    else finalize_weights(e);
  });
  API_END
}

int b2m_comm_unique_id(char* out128) {
  if (!out128) return B2M_ERR_INVALID;
  try {
    g_nccl.load();
    ncclUniqueId id;
    NCCL_CK(g_nccl.GetUniqueId(&id));
    static_assert(sizeof(id) == 128, "ncclUniqueId size");
    memcpy(out128, &id, 128);
  } catch (const b2m::Error& ex) {
    g_create_err = ex.what();
    return ex.code;
  }
  return B2M_OK;
}

int b2m_comm_init(b2m_handle h, const char* id128, int rank, int world) {
  API_BEGIN
  B2M_REQUIRE(world >= 1 && world <= MAXP && rank >= 0 && rank < world, B2M_ERR_PARTITIONS, "bad rank/world");
  B2M_REQUIRE(h->parts.empty(), B2M_ERR_STATE, "a single-process group (ndev > 1) needs no communicator");
  h->rank = rank;
  h->world = world;
  if (world > 1) {
    B2M_REQUIRE(id128 != nullptr, B2M_ERR_INVALID, "unique id required");
    g_nccl.load();
    ncclUniqueId id;
    memcpy(&id, id128, 128);
    NCCL_CK(g_nccl.CommInitRank(&h->comm, world, id, rank));
  }
  API_END
}

int b2m_set_partition(b2m_handle h, int rank, int world) {
  API_BEGIN
  B2M_REQUIRE(world >= 1 && world <= MAXP && rank >= 0 && rank < world, B2M_ERR_PARTITIONS, "bad rank/world");
  B2M_REQUIRE(h->comm == nullptr, B2M_ERR_STATE, "communicator already initialised");
  B2M_REQUIRE(h->parts.empty(), B2M_ERR_STATE, "the partitions of a single-process group are fixed by b2m_create");
  h->rank = rank;
  h->world = world;
  h->have_graph = false;
  API_END
}

static void set_structure_one(b2m_engine* h, int64_t natoms, const double* cart, const double* lattice9,
                              const int32_t* species, const int* pbc3, double tol) {
  h->have_graph = false;
  // positions and species through the library's page-locked staging (asynchronous upload inside the build)
  if (natoms > 0 && natoms < (1LL << 31) / 4) {
    const size_t cb = (size_t)natoms * 3 * sizeof(double), sb = (size_t)natoms * sizeof(int32_t);
    ensure_pinned(h->pin_in, h->pin_in_cap, cb + sb);
    par_memcpy(h->pin_in, cart, cb);
    memcpy((char*)h->pin_in + cb, species, sb);
    cart = reinterpret_cast<const double*>(h->pin_in);
    species = reinterpret_cast<const int32_t*>((const char*)h->pin_in + cb);
  }
  B2M_CK(cudaEventRecord(h->ev[3], h->st));
  h->atomic_last = 0;  // per-atom results of an earlier structure are gone
  h->hf_n = 0, h->hf_seed = -1;
  if (h->hf_reach > 0) {
    // heat flux: the unfolded cell, built on the device, is the graph's input; no periodicity
    h->uf.build(h->st, natoms, cart, species, lattice9, pbc3, h->hf_reach);
    const int no_pbc[3] = {0, 0, 0};
    h->g.walls_from_min = true;
    h->g.build(h->st, h->uf.N, h->uf.cart.p, lattice9, h->uf.species.p, no_pbc, h->desc.cutoff,
               h->desc.three_body_cutoff, tol, h->rank, h->world);
    h->hf_n = natoms;
    h->hf_w.ensure((size_t)h->uf.N + 64);
    for (int m = 0; m < 3; m++) h->hf_c[m] = 0.5 * (lattice9[m] + lattice9[3 + m] + lattice9[6 + m]);
  } else {
    h->g.walls_from_min = false;
    h->g.build(h->st, natoms, cart, lattice9, species, pbc3, h->desc.cutoff, h->desc.three_body_cutoff, tol, h->rank,
               h->world);
  }
  if (h->kind == 1) tn_alloc_workspace(h);
  else if (h->kind == 2) mace_alloc_workspace(h);
  else alloc_workspace(h);
  B2M_CK(cudaEventRecord(h->ev[4], h->st));
  B2M_CK(cudaStreamSynchronize(h->st));
  float ms;
  B2M_CK(cudaEventElapsedTime(&ms, h->ev[3], h->ev[4]));
  h->t_graph = ms;
  h->have_graph = true;
}

int b2m_set_structure(b2m_handle h, int64_t natoms, const double* cart, const double* lattice9,
                      const int32_t* species, const int* pbc3, double tol) {
  API_BEGIN
  B2M_REQUIRE(cart && lattice9 && species && pbc3, B2M_ERR_INVALID, "null structure argument");
  if (h->parts.empty()) {
    set_structure_one(h, natoms, cart, lattice9, species, pbc3, tol);
  } else {  // every partition builds its own slab on its own device, concurrently
    for_each_part(h, [&](b2m_engine* pe) { set_structure_one(pe, natoms, cart, lattice9, species, pbc3, tol); });
    for (auto* pe : h->parts) h->t_graph = std::max(h->t_graph, pe->t_graph);
  }
  API_END
}

int b2m_compute(b2m_handle h, int want_forces, int want_stress, double* energy, float* forces, float* stress9) {
  API_BEGIN
  run_any(h, want_forces || want_stress);
  fetch(h, energy, want_forces ? forces : nullptr, want_stress ? stress9 : nullptr);
  API_END
}

int b2m_compute_resident(b2m_handle h, int want_forces, int want_stress, int reps, double* energy, float* ms) {
  API_BEGIN
  B2M_REQUIRE(reps >= 1, B2M_ERR_INVALID, "reps >= 1");
  for (int r = 0; r < reps; r++) run_any(h, want_forces || want_stress);
  fetch(h, energy, nullptr, nullptr);
  if (ms) *ms = (float)h->t_total;
  API_END
}

int b2m_get_results(b2m_handle h, double* energy, float* forces, float* stress9) {
  API_BEGIN
  B2M_REQUIRE(h->have_graph, B2M_ERR_STATE, "no structure");
  fetch(h, energy, forces, stress9);
  API_END
}

int b2m_set_heat_flux(b2m_handle h, double reach) {
  API_BEGIN
  B2M_REQUIRE(reach >= 0 && std::isfinite(reach), B2M_ERR_INVALID, "heat-flux reach must be >= 0");
  each_member(h, [&](b2m_engine* e) { e->hf_reach = reach; });
  API_END
}

int b2m_compute_heat_flux(b2m_handle h, const double* vel, double* energy, float* forces, float* stress9,
                          double* flux6) {
  API_BEGIN
  B2M_REQUIRE(vel && flux6, B2M_ERR_INVALID, "velocities and flux6 are required");
  B2M_REQUIRE(h->hf_reach > 0, B2M_ERR_STATE, "heat flux is off (b2m_set_heat_flux(h, reach > 0) first)");
  B2M_REQUIRE(h->have_graph && h->hf_n > 0, B2M_ERR_STATE,
              "the resident structure is not unfolded (b2m_set_structure after b2m_set_heat_flux)");
  heat_flux(h, vel, flux6);
  fetch(h, energy, forces, stress9);
  API_END
}

int b2m_set_atomic(b2m_handle h, int on) {
  API_BEGIN
  each_member(h, [&](b2m_engine* e) { e->atomic = on != 0; });
  API_END
}

int b2m_get_atomic(b2m_handle h, double* energies, float* virials) {
  API_BEGIN
  B2M_REQUIRE(h->have_graph, B2M_ERR_STATE, "no structure");
  B2M_REQUIRE(h->atomic_last > 0, B2M_ERR_STATE,
              "the last evaluation ran without per-atom energies and virials (b2m_set_atomic(h, 1) first)");
  B2M_REQUIRE(virials == nullptr || h->atomic_last == 2, B2M_ERR_STATE,
              "per-atom virials need an evaluation with a backward (want_forces or want_stress)");
  fetch_atomic(h, energies, virials);
  API_END
}

int b2m_get_sitewise(b2m_handle h, float* out) {
  API_BEGIN
  B2M_REQUIRE(h->have_graph && out, B2M_ERR_STATE, "no structure");
  B2M_REQUIRE(h->kind == 0, B2M_ERR_INVALID, "the site-wise readout belongs to CHGNet (TensorNet and MACE have none)");
  std::vector<float> full(h->g.N, 0.f);
  auto collect = [&](b2m_engine* e) {  // owned rows of one partition -> global order
    Graph& g = e->g;
    std::vector<float> loc(g.n_own);
    std::vector<int> gid(g.n_own);
    B2M_CK(cudaMemcpyAsync(loc.data(), e->site.p, g.n_own * sizeof(float), cudaMemcpyDeviceToHost, e->st));
    B2M_CK(cudaMemcpyAsync(gid.data(), g.gid.p, g.n_own * sizeof(int), cudaMemcpyDeviceToHost, e->st));
    B2M_CK(cudaStreamSynchronize(e->st));
    for (int i = 0; i < g.n_own; i++) full[gid[i]] = loc[i];
  };
  each_member(h, collect);
  Graph& g = h->g;
  if (h->world > 1 && h->parts.empty()) {
    B2M_CK(cudaMemcpyAsync(h->site_full.p, full.data(), g.N * sizeof(float), cudaMemcpyHostToDevice, h->st));
    NCCL_CK(g_nccl.AllReduce(h->site_full.p, h->site_full.p, (size_t)g.N, ncclFloat32, ncclSum, h->comm, h->st));
    B2M_CK(cudaMemcpyAsync(full.data(), h->site_full.p, g.N * sizeof(float), cudaMemcpyDeviceToHost, h->st));
    B2M_CK(cudaStreamSynchronize(h->st));
  }
  memcpy(out, full.data(), cell_atoms(h) * sizeof(float));  // unfolded graph: the cell atoms come first
  API_END
}

int b2m_set_view(b2m_handle h, int part) {
  API_BEGIN
  const int n = h->parts.empty() ? 1 : (int)h->parts.size();
  B2M_REQUIRE(part >= 0 && part < n, B2M_ERR_PARTITIONS, "no such partition in this handle");
  h->view = part;
  API_END
}

int b2m_get_counts(b2m_handle h, int64_t* out, int n) {
  API_BEGIN
  B2M_REQUIRE(out && n >= 10, B2M_ERR_INVALID, "need room for 10 counts");
  b2m_engine* v = viewed(h);
  Graph& g = v->g;
  out[0] = g.n_own, out[1] = g.n_halo, out[2] = g.E, out[3] = g.B_own, out[4] = g.B_halo, out[5] = g.A;
  out[6] = g.axis, out[7] = v->rank, out[8] = v->world, out[9] = h->launches_last;
  API_END
}

int64_t b2m_get_partition_info(b2m_handle h, int which, int64_t* out, int64_t cap) {
  if (!h) return B2M_ERR_INVALID;
  try {
    b2m_engine* v = viewed(h);
    cudaSetDevice(v->device);
    B2M_REQUIRE(v->have_graph && out, B2M_ERR_STATE, "no structure");
    const int64_t n = v->g.export_info(v->st, which, out, cap);
    cudaSetDevice(h->device);
    return n;
  } catch (const b2m::Error& ex) {
    h->err = ex.what();
    return ex.code;
  }
}

int b2m_debug_tensor(b2m_handle h, const char* name, float* out, int64_t cap, int64_t* rows, int64_t* cols) {
  API_BEGIN
  B2M_REQUIRE(h->have_graph && name && out && rows && cols, B2M_ERR_STATE, "no structure");
  Graph& g = h->g;
  std::string n(name);
  const float* src = nullptr;
  int64_t r = 0, c = D;
  auto idx = [&](const std::string& pre) { return atoi(n.c_str() + pre.size()); };
  if (h->kind == 1) {
    B2M_REQUIRE(tn_debug_lookup(h, n, src, r, c), B2M_ERR_INVALID, "unknown debug tensor: " + n);
  } else if (h->kind == 2) {
    B2M_REQUIRE(mace_debug_lookup(h, n, src, r, c), B2M_ERR_INVALID, "unknown debug tensor: " + n);
  } else if (n[0] == 'x' && isdigit(n[1])) {
    int l = idx("x");
    B2M_REQUIRE(l >= 0 && l < (int)h->x.size(), B2M_ERR_INVALID, "bad layer");
    src = h->x[l].p, r = l == (int)h->x.size() - 1 ? g.n_own : g.n_loc;
  } else if (n[0] == 'h' && isdigit(n[1])) {
    int l = idx("h");
    B2M_REQUIRE(l >= 0 && l < (int)h->h.size(), B2M_ERR_INVALID, "bad layer");
    src = h->h[l].p, r = g.B_own;
  } else if (n.rfind("ang", 0) == 0 && isdigit(n[3])) {
    int l = idx("ang");
    B2M_REQUIRE(l >= 0 && l < (int)h->ang.size(), B2M_ERR_INVALID, "bad layer");
    src = h->ang[l].p, r = g.A;
  } else if (n == "e_atom") {
    src = h->e_atom.p, r = g.n_own, c = 1;
  } else if (n == "gd") {
    src = h->gd.p, r = g.E, c = 1;
  } else if (n == "gdb") {
    src = h->gdb.p, r = g.B_loc, c = 1;
  } else if (n == "gbvec") {
    src = h->gbvec.p, r = g.B_loc, c = 3;
  } else if (n == "gx") {
    src = h->gx.p, r = g.n_loc;
  } else if (n == "gh") {
    src = h->gh.p, r = g.B_loc;
  } else if (n == "gang") {
    src = h->gang.p, r = g.A;
  } else if (n == "e_vec") {
    src = reinterpret_cast<const float*>(g.e_vec.p), r = g.E, c = 4;
  } else {
    throw Error(B2M_ERR_INVALID, "unknown debug tensor: " + n);
  }
  B2M_REQUIRE(r * c <= cap, B2M_ERR_INVALID, "debug buffer too small");
  B2M_CK(cudaMemcpyAsync(out, src, r * c * sizeof(float), cudaMemcpyDeviceToHost, h->st));
  B2M_CK(cudaStreamSynchronize(h->st));
  *rows = r, *cols = c;
  API_END
}

int b2m_release_workspace(b2m_handle h) {
  API_BEGIN
  each_member(h, [&](b2m_engine* e) {
    B2M_CK(cudaStreamSynchronize(e->st));
    e->have_graph = false;
    auto drop = [](auto& b) {
      if (b.p) cudaFree(b.p);
      b.p = nullptr, b.cap = 0;
    };
    for (auto* v : {&e->x, &e->h, &e->ang, &e->upd, &e->ApL, &e->CpL, &e->QpL})
      for (auto& b : *v) drop(b);
    for (auto* b : {&e->Ha, &e->Hb, &e->Xc, &e->agg, &e->aggB, &e->y1p, &e->y1, &e->y2p, &e->y2,
                    &e->e_atom, &e->site, &e->gx, &e->gh, &e->gang, &e->gA, &e->gC, &e->gQ, &e->gHa, &e->gHb, &e->gXc,
                    &e->gagg, &e->gupd, &e->gaggB, &e->gd, &e->gdb, &e->gbvec, &e->gy1, &e->gy2, &e->forces,
                    &e->sendbuf, &e->recvbuf, &e->site_full, &e->precv[0], &e->precv[1], &e->ftmp, &e->fsum,
                    &e->atom_vir, &e->avsum, &e->avtmp, &e->hf_w, &e->hf_G, &e->hf_fold})
      drop(*b);
    for (auto* b : {&e->atom_e, &e->aesum, &e->aetmp, &e->hf_vel, &e->hf_out}) drop(*b);
    e->atomic_last = 0;
    e->hf_n = 0;
    e->uf.~Unfold();
    new (&e->uf) Unfold();
    tn_release(e);
    mace_release(e);
    e->g.~Graph();  // the resident graph goes too
    new (&e->g) Graph();
  });
  API_END
}

int b2m_last_timings(b2m_handle h, double* out, int n) {
  API_BEGIN
  B2M_REQUIRE(out && n >= 5, B2M_ERR_INVALID, "need room for 5 timings");
  out[0] = h->t_graph, out[1] = h->t_fwd, out[2] = h->t_bwd, out[3] = h->t_gather, out[4] = h->t_total;
  API_END
}

}  // extern "C"
