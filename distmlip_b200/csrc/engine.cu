// engine.cu -- host orchestration behind the C-ABI (include/b200mlip.h): the frame every model runs in (weight upload,
// GPU-resident workspace, halo exchange between slab neighbours (NCCL point-to-point between processes, peer-memory
// stores inside a single-process group), partition sums, heat flux) and the extern "C" entry points.  The models plug in
// through `Model`: CHGNet (engine_chgnet.inl), TensorNet (engine_tn.inl) and MACE (engine_mace.inl).
#include <dlfcn.h>
#include <nccl.h>

#include <cmath>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <new>
#include <set>
#include <string>
#include <vector>

#include <algorithm>
#include <array>

#include "final_tail.cuh"
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

struct Packer {
  std::vector<float> host;
  std::map<std::string, size_t> off;  // named images (put)
  float* dev = nullptr;               // their device copy, once uploaded
  size_t add(const std::vector<float>& v) {
    size_t o = (host.size() + 63) / 64 * 64;  // 256 B alignment
    host.resize(o + v.size());
    memcpy(host.data() + o, v.data(), v.size() * sizeof(float));
    return o;
  }
  void put(const std::string& name, const std::vector<float>& v) { off[name] = add(v); }
  float* at(const std::string& name) const { return dev + off.at(name); }
};

struct HaloRows {
  float* p;
  int width;  // floats per row
};

// A model on the engine: CHGNet (engine_chgnet.inl), TensorNet (engine_tn.inl), MACE (engine_mace.inl).  The frame
// calls it for everything that differs between models; a model is built by its factory (make_*), which checks the
// description, and owns its weights and its per-structure workspace.
struct Model {
  const char* name = "";        // names the configuration in the refusal of an unused state_dict tensor
  const char* trace = nullptr;  // stage() prefix when the model's B2M_<MODEL>_TRACE=1
  bool sitewise = false;        // has a site-wise readout (b2m_get_sitewise)
  bool own_scaling = false;     // carries its own scale, shift and E0 (b2m_set_scaling / b2m_set_element_refs refuse)
  virtual ~Model() = default;
  // state_dict -> weight images in P (each tensor read through weight()); after the upload, the device pointers
  virtual void pack(b2m_engine* e, Packer& P) = 0;
  virtual void bind(const Packer& P) = 0;
  virtual void alloc(b2m_engine* e) = 0;  // workspace of the resident graph
  virtual void release() = 0;             // frees that workspace
  virtual void forward(b2m_engine* e) = 0;
  virtual void backward(b2m_engine* e) = 0;
  virtual HaloRows halo(int l, bool bonds) = 0;  // rows exchanged for layer l: atom rows, or bond rows
  virtual int halo_width() const = 0;            // widest halo row, sizes the transport buffers
  // name -> (pointer, rows, cols) for b2m_debug_tensor; false: no such tensor
  virtual bool debug(b2m_engine* e, const std::string& n, const float*& src, int64_t& r, int64_t& c) = 0;
};

// per-structure buffers of the frame (b2m_release_workspace replaces them with empty ones)
struct Bufs {
  DBuf<float> forces, sendbuf, recvbuf;
  DBuf<double> scal;   // [0]=energy, [1..9]=virial
  DBuf<float> precv[2];  // adjoint rows pushed by my neighbours (backward), double-buffered by point parity
  DBuf<float> ftmp;      // leader: staging of a peer's force array
  DBuf<float> fsum;      // leader: the group's summed forces (the partitions' own arrays stay untouched)
  DBuf<float> site, site_full;  // site-wise readout: owned rows, the whole structure
  // per-atom energies and virials (b2m_set_atomic; DESIGN.md "Per-atom energies and virials"): allocated on the first
  // evaluation with the flag on, indexed by global atom id like `forces`
  DBuf<double> atom_e;        // [N]
  DBuf<float> atom_vir;       // [N][kVirPitch]
  DBuf<double> aesum, aetmp;  // leader of a group: the summed energies / staging of a peer's array
  DBuf<float> avsum, avtmp;   // same for the virials
  DBuf<float> hf_w;       // [N] readout weight of every unfolded atom (heat flux)
  DBuf<float> hf_G;       // leader: [3][N][3] forces of the three seeded passes
  DBuf<float> hf_fold;    // leader: folded forces [n][3] or virials [n][kVirPitch]
  DBuf<double> hf_vel, hf_out;
  DBuf<double> bsum;      // batch: [S][10] energy and virial of every structure
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
  std::unique_ptr<b2m::Model> model;
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
  const double* d_eref = nullptr;  // per-element energy offsets, double like the energy accumulator
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
  int view = 0;                    // leader: partition addressed by the inspection calls (b2m_set_view)
  int partition_policy = B2M_PARTITION_EQUAL;  // b2m_set_partition_policy, applied at the next graph build
  // page-locked staging owned by the library: host arrays go through it with a few copy threads (a single-threaded
  // memcpy of 24 MB of positions was the largest host item of an end-to-end step at 1 M atoms)
  void* pin_in = nullptr;   // [N,3] f64 positions followed by [N] i32 species
  size_t pin_in_cap = 0;
  void* pin_out = nullptr;  // [N,3] f32 forces
  size_t pin_out_cap = 0;
  // resident graph and the per-structure buffers
  Graph g;
  bool have_graph = false;
  b2m::Bufs buf;
  bool atomic = false;      // b2m_set_atomic
  int atomic_last = 0;      // what the last evaluation left in them: 0 nothing, 1 energies, 2 energies and virials
  // heat flux (b2m_set_heat_flux; DESIGN.md §10): with hf_reach > 0 b2m_set_structure builds the unfolded cell (`uf`) and
  // the graph of it without periodicity; every readout then weights atom j's energy by hf_w[j]
  double hf_reach = 0;
  Unfold uf;
  int64_t hf_n = 0;       // cell atoms of the resident unfolded graph; 0: the graph is the structure itself
  int hf_seed = -1;       // weight of the next evaluation: -1 the cell mask (1 / 0), 0..2 the seed (r_j - c)_alpha
  double hf_c[3] = {0, 0, 0};  // cell centre
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

// a batch of structures is resident (b2m_set_structures, DESIGN.md §12)
static bool batched(const b2m_engine* e) { return e->have_graph && e->g.S > 0; }

// optional outputs of an evaluation and the readout weights, null where they are off: per-atom energies and virials
// (b2m_set_atomic; always on for a batch, whose per-structure sums are taken from them), and each atom's energy weight
// (heat flux, DESIGN.md §10)
static bool per_atom_on(const b2m_engine* e) { return e->atomic || batched(e); }
static double* atom_e_out(b2m_engine* e) { return per_atom_on(e) ? e->buf.atom_e.p : nullptr; }
static float* atom_vir_out(b2m_engine* e) { return per_atom_on(e) ? e->buf.atom_vir.p : nullptr; }
// data_mean's share of each per-atom energy in the readout; a batch adds each structure's share in k_batch_sums
static double mean_per_atom(const b2m_engine* e) { return batched(e) ? 0.0 : e->desc.data_mean / cell_atoms(e); }
static const float* readout_wgt(const b2m_engine* e) { return e->hf_n ? e->buf.hf_w.p : nullptr; }

// state_dict tensor k, marked as used; its shape must be `shape`, or with `flat` only hold as many elements
static const std::vector<float>& weight(b2m_engine* e, const std::string& k, const std::vector<int64_t>& shape,
                                        const char* shape_err, bool flat = false) {
  auto it = e->host_w.find(k);
  B2M_REQUIRE(it != e->host_w.end(), B2M_ERR_INVALID, "missing weight: " + k);
  e->consumed.insert(k);
  size_t n = 1;
  for (auto s : shape) n *= (size_t)s;
  B2M_REQUIRE(it->second.size() == n && (flat || e->host_shape[k] == shape), B2M_ERR_INVALID,
              "weight '" + k + "' has an unsupported shape" + shape_err);
  return it->second;
}

// B2M_TN_TRACE=1 / B2M_MACE_TRACE=1: synchronise after every stage of that model and name it on stderr (locating a
// faulting or hanging kernel)
static const char* trace_tag(const char* env, const char* tag) {
  const char* v = getenv(env);
  return v && v[0] == '1' ? tag : nullptr;
}
static void stage(b2m_engine* e, const char* name) {
  if (!e->model->trace) return;
  fprintf(stderr, "[%s] %s ...", e->model->trace, name);
  fflush(stderr);
  cudaError_t r = cudaStreamSynchronize(e->st);
  fprintf(stderr, " %s\n", cudaGetErrorString(r));
  fflush(stderr);
}


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
  e->consumed.clear();
  Packer P;
  e->model->pack(e, P);
  // every tensor of the state_dict must have been used: an extra bias / normalisation / per-layer weight function of
  // a configuration the engine does not build would otherwise be dropped silently and give wrong energies (ADVICE r1)
  for (auto& kv : e->host_w)
    if (!e->consumed.count(kv.first))
      throw Error(B2M_ERR_INVALID, "state_dict tensor '" + kv.first + "' is not used by this engine (unsupported " +
                                       e->model->name + " configuration; refusing to ignore it)");
  if (!e->elem_refs.empty()) {
    e->erefbuf.ensure(e->elem_refs.size());
    B2M_CK(cudaMemcpyAsync(e->erefbuf.p, e->elem_refs.data(), e->elem_refs.size() * sizeof(double), cudaMemcpyHostToDevice,
                           e->st));
  }
  e->wbuf.ensure(P.host.size() + 64);
  B2M_CK(cudaMemcpyAsync(e->wbuf.p, P.host.data(), P.host.size() * sizeof(float), cudaMemcpyHostToDevice, e->st));
  B2M_CK(cudaStreamSynchronize(e->st));
  P.dev = e->wbuf.p;
  e->model->bind(P);
  e->d_eref = e->elem_refs.empty() ? nullptr : e->erefbuf.p;
  e->finalized = true;
}

// ------------------------------------------------------------------------------------------
static void alloc_workspace(b2m_engine* e) {
  e->model->alloc(e);
  Graph& g = e->g;
  Bufs& b = e->buf;
  b.forces.ensure((size_t)g.N * 3 + 64);
  b.scal.ensure(16);
  if (e->model->sitewise) b.site.ensure(g.n_own), b.site_full.ensure((size_t)g.N + 64);
  if (e->world > 1) {
    size_t tot_to = 0, tot_bto = 0;
    for (int q = 0; q < e->world; q++) tot_to += g.n_to[q], tot_bto += g.nb_to[q];
    const size_t m = std::max(tot_to, tot_bto) * e->model->halo_width();
    if (e->leader != nullptr) {
      b.precv[0].ensure(m + 64), b.precv[1].ensure(m + 64);
    } else {
      b.sendbuf.ensure(m + 64), b.recvbuf.ensure(m + 64);
    }
  }
}

// ---- halo exchange between slab neighbours ----
// Two transports: NCCL point-to-point (one process per GPU, world > 1 with a communicator) and, inside a single-process
// group, direct peer-memory traffic: the sender's pack kernel stores its boundary rows straight into the receiver's halo
// rows (forward) or copies its halo adjoints into the owner's receive buffer (backward); a CUDA event per exchange point
// orders the receiver's stream behind the sender's.

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
static void halo_forward_begin(b2m_engine* e, bool bonds, int l) {
  if (e->world <= 1 || e->debug_no_halo) return;
  Graph& g = e->g;
  const HaloRows rows = e->model->halo(l, bonds);
  const size_t W = (size_t)rows.width;
  float* buf = rows.p;
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
      launch_gather_rows(e->cst, nto[q], (int)W, list + toff[q], buf, pe->model->halo(l, bonds).p + (pbase + pfoff) * W);
    }
    B2M_CK(cudaEventRecord(next_halo_event(e), e->cst));
    return;
  }
  for (int q = 0; q < e->world; q++)
    if (nto[q] > 0)
      launch_gather_rows(e->cst, nto[q], (int)W, list + toff[q], buf, e->buf.sendbuf.p + (size_t)toff[q] * W);
  NCCL_CK(g_nccl.GroupStart());
  for (int q = 0; q < e->world; q++) {
    if (q == e->rank) continue;
    if (nto[q] > 0)
      NCCL_CK(g_nccl.Send(e->buf.sendbuf.p + (size_t)toff[q] * W, (size_t)nto[q] * W, ncclFloat32, q, e->comm, e->cst));
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
      B2M_CK(cudaMemcpyAsync(pe->buf.precv[k & 1].p + ptoff * W, gbuf + (base + foff[q]) * W,
                             (size_t)nfrom[q] * W * sizeof(float), cudaMemcpyDefault, e->st));
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
        launch_scatter_add_rows(e->st, nto[q], (int)W, list + toff[q], e->buf.precv[k & 1].p + (size_t)toff[q] * W, gbuf);
    return;
  }
  NCCL_CK(g_nccl.GroupStart());
  for (int q = 0; q < e->world; q++) {
    if (q == e->rank) continue;
    if (nfrom[q] > 0)
      NCCL_CK(g_nccl.Send(gbuf + (base + foff[q]) * W, (size_t)nfrom[q] * W, ncclFloat32, q, e->comm, e->st));
    if (nto[q] > 0)
      NCCL_CK(g_nccl.Recv(e->buf.recvbuf.p + (size_t)toff[q] * W, (size_t)nto[q] * W, ncclFloat32, q, e->comm, e->st));
  }
  NCCL_CK(g_nccl.GroupEnd());
  for (int q = 0; q < e->world; q++)
    if (nto[q] > 0)
      launch_scatter_add_rows(e->st, nto[q], (int)W, list + toff[q], e->buf.recvbuf.p + (size_t)toff[q] * W, gbuf);
  launch_zero_rows(e->st, gbuf + base * W, nhalo * W);
}

#include "engine_chgnet.inl"
#include "engine_tn.inl"
#include "engine_mace.inl"


// ------------------------------------------------------------------------------------------
// heat flux (DESIGN.md §10)
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
  block_sum_add(acc, out);
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
  const size_t N = (size_t)e->g.N;
  if (per_atom_on(e)) {  // zeroed here, before the readout writes the energies and the backward accumulates the virials
    e->buf.atom_e.ensure(N + 64);
    e->buf.atom_e.zero(N, e->st);
    if (grads) {
      e->buf.atom_vir.ensure(N * kVirPitch + 64);
      e->buf.atom_vir.zero(N * kVirPitch, e->st);
    }
  }
  e->atomic_last = 0;
  if (e->hf_n) {
    launch(k_hf_weights, cdiv(e->g.N, 256), 256, 0, e->st, e->g.N, e->hf_n, e->g.cart.p, e->hf_c[0], e->hf_c[1],
           e->hf_c[2], e->hf_seed, e->buf.hf_w.p);
  }
  e->model->forward(e);
  B2M_CK(cudaEventRecord(e->ev[1], e->st));
  if (grads) e->model->backward(e);
  if (e->world > 1 && e->leader == nullptr && !e->debug_no_halo) {
    NCCL_CK(g_nccl.AllReduce(e->buf.scal.p, e->buf.scal.p, 10, ncclFloat64, ncclSum, e->comm, e->st));
    if (grads)
      NCCL_CK(g_nccl.AllReduce(e->buf.forces.p, e->buf.forces.p, (size_t)e->g.N * 3, ncclFloat32, ncclSum, e->comm, e->st));
    if (e->atomic) {
      NCCL_CK(g_nccl.AllReduce(e->buf.atom_e.p, e->buf.atom_e.p, N, ncclFloat64, ncclSum, e->comm, e->st));
      if (grads)
        NCCL_CK(g_nccl.AllReduce(e->buf.atom_vir.p, e->buf.atom_vir.p, N * kVirPitch, ncclFloat32, ncclSum, e->comm, e->st));
    }
  }
  B2M_CK(cudaEventRecord(e->ev[2], e->st));
  B2M_CK(cudaStreamSynchronize(e->st));
  e->launches_last = g_launch_count - l0;
  e->atomic_last = per_atom_on(e) ? (grads ? 2 : 1) : 0;
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

template <class T>
__global__ void k_add_inplace(int64_t n, const T* __restrict__ src, T* __restrict__ dst) {
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

// `arr` [n] summed over the partitions of the group led by L, on L's device: into `sum`, each peer's array staged in `tmp`
template <class T>
static const T* part_sum(b2m_engine* L, DBuf<T> Bufs::*arr, DBuf<T>& sum, DBuf<T>& tmp, size_t n) {
  sum.ensure(n + 64);
  tmp.ensure(n + 64);
  B2M_CK(cudaMemcpyAsync(sum.p, (L->buf.*arr).p, n * sizeof(T), cudaMemcpyDeviceToDevice, L->st));
  for (size_t p = 1; p < L->parts.size(); p++) {
    B2M_CK(cudaMemcpyAsync(tmp.p, (L->parts[p]->buf.*arr).p, n * sizeof(T), cudaMemcpyDefault, L->st));
    launch(k_add_inplace<T>, cdiv((int64_t)n, 256), 256, 0, L->st, (int64_t)n, tmp.p, sum.p);
  }
  return sum.p;
}

// forces [N][3] of the whole structure on the leader's device: a group sums its partitions' arrays, a multi-process run
// has all-reduced them in run()
static const float* summed_forces(b2m_engine* e) {
  if (e->parts.empty()) return e->buf.forces.p;
  return part_sum(e, &Bufs::forces, e->buf.fsum, e->buf.ftmp, (size_t)e->g.N * 3);
}


// unfolded graph: rows [N][pitch] of every unfolded atom summed onto their cell atoms -> [n][pitch] (hf_fold)
static const float* fold_rows(b2m_engine* e, const float* src, int width, int pitch) {
  const int64_t N = e->g.N, n = e->hf_n;
  e->buf.hf_fold.ensure((size_t)n * pitch + 64);
  e->buf.hf_fold.zero((size_t)n * pitch, e->st);
  launch(k_hf_fold, cdiv(N * width, 256), 256, 0, e->st, N, e->uf.image_of.p, width, pitch, src, e->buf.hf_fold.p);
  return e->buf.hf_fold.p;
}

static void fetch(b2m_engine* e, double* energy, float* forces, float* stress9) {
  double hs[10];
  B2M_CK(cudaMemcpyAsync(hs, e->buf.scal.p, 10 * sizeof(double), cudaMemcpyDeviceToHost, e->st));
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
    B2M_CK(cudaMemcpy(ps, pe->buf.scal.p, 10 * sizeof(double), cudaMemcpyDeviceToHost));
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
  const double* esrc = e->buf.atom_e.p;
  const float* vsrc = e->buf.atom_vir.p;
  if (!e->parts.empty()) {
    if (energies) esrc = part_sum(e, &Bufs::atom_e, e->buf.aesum, e->buf.aetmp, NG);
    if (virials) vsrc = part_sum(e, &Bufs::atom_vir, e->buf.avsum, e->buf.avtmp, NG * kVirPitch);
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

// Batch (DESIGN.md §12): block s sums the per-atom energies and virials (f32 summed in f64; null: energies only) of
// structure s, the atoms off[s] .. off[s + 1] - 1, into out[s][0] and out[s][1..9] (zeroed before), and adds data_mean's
// per-atom share data_mean / n_s to each of its per-atom energies, as a single evaluation of the structure has them
__global__ void __launch_bounds__(256) k_batch_sums(const int64_t* __restrict__ off, double data_mean,
                                                    double* __restrict__ atom_e, const float* __restrict__ atom_vir,
                                                    double* __restrict__ out) {
  const int64_t b = off[blockIdx.x], end = off[blockIdx.x + 1];
  const double m = data_mean / (end - b);
  double acc[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int64_t i = b + threadIdx.x; i < end; i += blockDim.x) {
    acc[0] += atom_e[i];
    atom_e[i] += m;
    if (atom_vir)
      for (int k = 0; k < 9; k++) acc[1 + k] += (double)atom_vir[i * kVirPitch + k];
  }
  block_sum_add(acc, out + 10 * blockIdx.x);
}

// energies [S], forces [N][3] and stress9 [S][9] of the batch just evaluated (any may be null); one launch for any S
static void fetch_batch(b2m_engine* e, bool grads, double* energies, float* forces, float* stress9) {
  const Graph& g = e->g;
  e->buf.bsum.ensure((size_t)g.S * 10 + 64);
  e->buf.bsum.zero((size_t)g.S * 10, e->st);
  launch(k_batch_sums, g.S, 256, 0, e->st, g.b_doff.p, e->desc.data_mean, e->buf.atom_e.p,
         grads ? (const float*)e->buf.atom_vir.p : nullptr, e->buf.bsum.p);
  std::vector<double> hs((size_t)g.S * 10);
  B2M_CK(cudaMemcpyAsync(hs.data(), e->buf.bsum.p, hs.size() * sizeof(double), cudaMemcpyDeviceToHost, e->st));
  fetch(e, nullptr, forces, nullptr);  // forces, and the stream synchronised
  for (int s = 0; s < g.S; s++) {
    if (energies) energies[s] = hs[10 * s] + e->desc.data_mean;
    if (stress9)
      for (int k = 0; k < 9; k++) stress9[9 * s + k] = (float)(hs[10 * s + 1 + k] / g.b_volume[s] * 160.21766208);
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
    h->buf.hf_G.ensure((size_t)N * 9 + 64);
    for (int a = 0; a < 3; a++) {
      for (auto* e : members) e->hf_seed = a;
      run_any(h, true);
      B2M_CK(cudaMemcpyAsync(h->buf.hf_G.p + (size_t)a * N * 3, summed_forces(h), (size_t)N * 3 * sizeof(float),
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
  const double* eps = h->parts.empty() ? h->buf.atom_e.p : part_sum(h, &Bufs::atom_e, h->buf.aesum, h->buf.aetmp, N);
  h->buf.hf_vel.ensure((size_t)n * 3 + 64);
  h->buf.hf_out.ensure(64);
  B2M_CK(cudaMemcpyAsync(h->buf.hf_vel.p, vel, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice, h->st));
  h->buf.hf_out.zero(6, h->st);
  const int grid = std::max(1, std::min(cdiv(N, 256), 4 * h->num_sms));
  launch(k_hf_contract, grid, 256, 0, h->st, N, n, h->g.cart.p, h->hf_c[0], h->hf_c[1], h->hf_c[2], h->uf.image_of.p,
         h->buf.hf_vel.p, F, h->buf.hf_G.p, eps, h->buf.hf_out.p);
  B2M_CK(cudaMemcpyAsync(flux6, h->buf.hf_out.p, 6 * sizeof(double), cudaMemcpyDeviceToHost, h->st));
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

// make() builds the model of one partition and checks its description; it runs for every partition before any device
// is touched
static int create_any(const b2m_model_desc* desc, const int* devices, int ndev, b2m_handle* out,
                      const std::function<std::unique_ptr<Model>()>& make) {
  if (!desc || !devices || !out) return B2M_ERR_INVALID;
  std::vector<b2m_engine*> made;
  try {
    B2M_REQUIRE(ndev >= 1 && ndev <= MAXP, B2M_ERR_PARTITIONS, "ndev must be in [1,16]");
    std::vector<std::unique_ptr<Model>> models;
    for (int p = 0; p < ndev; p++) models.push_back(make());
    int count = 0;
    cudaError_t ce = cudaGetDeviceCount(&count);
    if (ce != cudaSuccess || count <= 0)
      throw Error(B2M_ERR_CUDA, std::string("no CUDA device available (libb200mlip has no CPU fallback): ") +
                                    cudaGetErrorString(ce));
    for (int p = 0; p < ndev; p++) {
      made.push_back(create_one(desc, devices[p], count));
      made.back()->model = std::move(models[p]);
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
    for (auto* m : made) delete m;
    g_create_err = ex.what();
    return ex.code;
  }
  return B2M_OK;
}

int b2m_create(const b2m_model_desc* desc, const int* devices, int ndev, b2m_handle* out) {
  return create_any(desc, devices, ndev, out, [&] { return make_chgnet(*desc); });
}

int b2m_create_tensornet(const b2m_tensornet_desc* tdesc, const int* devices, int ndev, b2m_handle* out) {
  if (!tdesc) return B2M_ERR_INVALID;
  // the shared part of the engine (graph build, scaling, transport) reads the CHGNet-shaped description: no bond graph
  // (use_bond_graph False, three_body_cutoff 0: pes.py:79-80)
  b2m_model_desc d;
  memset(&d, 0, sizeof d);
  d.n_elem = tdesc->n_elem, d.dim = D, d.max_n = NR, d.max_f = 4, d.n_blocks = tdesc->n_blocks, d.cutoff_exponent = 0;
  d.cutoff = tdesc->cutoff, d.three_body_cutoff = 0.0, d.data_mean = tdesc->data_mean, d.data_std = tdesc->data_std;
  return create_any(&d, devices, ndev, out, [&] { return make_tensornet(*tdesc); });
}

int b2m_create_mace(const b2m_mace_desc* mdesc, const int* devices, int ndev, b2m_handle* out) {
  if (!mdesc) return B2M_ERR_INVALID;
  // the shared part of the engine (graph build, transport) reads the CHGNet-shaped description: no bond graph, r_max as
  // the cutoff, no Potential scaling (scale, shift and E0 are part of the model)
  b2m_model_desc d;
  memset(&d, 0, sizeof d);
  d.n_elem = mdesc->n_elem, d.dim = D, d.max_n = NR, d.max_f = 4, d.n_blocks = mdesc->num_interactions;
  d.cutoff = mdesc->r_max, d.three_body_cutoff = 0.0, d.data_mean = 0.0, d.data_std = 1.0;
  return create_any(&d, devices, ndev, out, [&] { return make_mace(*mdesc); });
}

static void destroy_one(b2m_engine* h) {
  cudaSetDevice(h->device);
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
  B2M_REQUIRE(!h->model->own_scaling, B2M_ERR_INVALID, "a MACE model carries its own atomic energies (atomic_energies_fn)");
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
  B2M_REQUIRE(!h->model->own_scaling, B2M_ERR_INVALID, "a MACE model carries its own scale and shift (scale_shift)");
  each_member(h, [&](b2m_engine* e) {
    e->desc.data_mean = data_mean;
    e->desc.data_std = data_std;
  });
  API_END
}

int b2m_finalize_weights(b2m_handle h) {
  API_BEGIN
  each_member(h, finalize_weights);
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

int b2m_set_partition_policy(b2m_handle h, int policy) {
  API_BEGIN
  B2M_REQUIRE(policy == B2M_PARTITION_EQUAL || policy == B2M_PARTITION_BALANCED, B2M_ERR_INVALID,
              "partition policy must be B2M_PARTITION_EQUAL (0) or B2M_PARTITION_BALANCED (1)");
  each_member(h, [&](b2m_engine* e) { e->partition_policy = policy; });
  API_END
}

// natoms atoms of one structure, or (nstruct > 0) the concatenated atoms of nstruct structures with counts[s] atoms each
static void set_structure_one(b2m_engine* h, int64_t natoms, const double* cart, const double* lattice9,
                              const int32_t* species, const int* pbc3, double tol, int nstruct = 0,
                              const int64_t* counts = nullptr) {
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
  h->g.balanced = h->partition_policy == B2M_PARTITION_BALANCED;
  if (nstruct > 0) {
    h->g.walls_from_min = false;
    h->g.build_batch(h->st, nstruct, counts, cart, lattice9, species, pbc3, h->desc.cutoff, h->desc.three_body_cutoff,
                     tol);
  } else if (h->hf_reach > 0) {
    // heat flux: the unfolded cell, built on the device, is the graph's input; no periodicity
    h->uf.build(h->st, natoms, cart, species, lattice9, pbc3, h->hf_reach);
    const int no_pbc[3] = {0, 0, 0};
    h->g.walls_from_min = true;
    h->g.build(h->st, h->uf.N, h->uf.cart.p, lattice9, h->uf.species.p, no_pbc, h->desc.cutoff,
               h->desc.three_body_cutoff, tol, h->rank, h->world);
    h->hf_n = natoms;
    h->buf.hf_w.ensure((size_t)h->uf.N + 64);
    for (int m = 0; m < 3; m++) h->hf_c[m] = 0.5 * (lattice9[m] + lattice9[3 + m] + lattice9[6 + m]);
  } else {
    h->g.walls_from_min = false;
    h->g.build(h->st, natoms, cart, lattice9, species, pbc3, h->desc.cutoff, h->desc.three_body_cutoff, tol, h->rank,
               h->world);
  }
  alloc_workspace(h);
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

int b2m_set_structures(b2m_handle h, int32_t nstruct, const int64_t* natoms, const double* cart,
                       const double* lattice9, const int32_t* species, const int* pbc3, double tol) {
  API_BEGIN
  B2M_REQUIRE(h->parts.empty() && h->world == 1, B2M_ERR_INVALID,
              "a batch runs on one partition: not on a single-process group (ndev > 1) or a rank of a multi-process job");
  B2M_REQUIRE(h->hf_reach == 0, B2M_ERR_STATE, "a batch has no heat flux (b2m_set_heat_flux(h, 0) first)");
  B2M_REQUIRE(nstruct >= 1, B2M_ERR_INVALID, "a batch needs at least one structure");
  B2M_REQUIRE(natoms && cart && lattice9 && species && pbc3, B2M_ERR_INVALID, "null structure argument");
  int64_t total = 0;
  for (int s = 0; s < nstruct; s++) {
    B2M_REQUIRE(natoms[s] > 0, B2M_ERR_INVALID, "structure " + std::to_string(s) + ": no atoms");
    total += natoms[s];
  }
  set_structure_one(h, total, cart, lattice9, species, pbc3, tol, nstruct, natoms);
  API_END
}

int b2m_compute_batch(b2m_handle h, int want_forces, int want_stress, double* energies, float* forces, float* stress9) {
  API_BEGIN
  B2M_REQUIRE(batched(h), B2M_ERR_STATE, "no batch is resident (b2m_set_structures first)");
  const bool grads = want_forces || want_stress;
  run(h, grads);
  fetch_batch(h, grads, energies, want_forces ? forces : nullptr, want_stress ? stress9 : nullptr);
  API_END
}

// the single-structure results (one energy, one stress) of b2m_compute and its relatives do not exist for a batch
static void refuse_batch(b2m_engine* h) {
  B2M_REQUIRE(!batched(h), B2M_ERR_STATE,
              "a batch is resident: b2m_compute_batch evaluates it, b2m_set_structure goes back to one structure");
}

int b2m_compute(b2m_handle h, int want_forces, int want_stress, double* energy, float* forces, float* stress9) {
  API_BEGIN
  refuse_batch(h);
  run_any(h, want_forces || want_stress);
  fetch(h, energy, want_forces ? forces : nullptr, want_stress ? stress9 : nullptr);
  API_END
}

int b2m_compute_resident(b2m_handle h, int want_forces, int want_stress, int reps, double* energy, float* ms) {
  API_BEGIN
  B2M_REQUIRE(reps >= 1, B2M_ERR_INVALID, "reps >= 1");
  refuse_batch(h);
  for (int r = 0; r < reps; r++) run_any(h, want_forces || want_stress);
  fetch(h, energy, nullptr, nullptr);
  if (ms) *ms = (float)h->t_total;
  API_END
}

int b2m_get_results(b2m_handle h, double* energy, float* forces, float* stress9) {
  API_BEGIN
  B2M_REQUIRE(h->have_graph, B2M_ERR_STATE, "no structure");
  refuse_batch(h);
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
  refuse_batch(h);
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
  B2M_REQUIRE(h->model->sitewise, B2M_ERR_INVALID, "the site-wise readout belongs to CHGNet (TensorNet and MACE have none)");
  std::vector<float> full(h->g.N, 0.f);
  auto collect = [&](b2m_engine* e) {  // owned rows of one partition -> global order
    Graph& g = e->g;
    std::vector<float> loc(g.n_own);
    std::vector<int> gid(g.n_own);
    B2M_CK(cudaMemcpyAsync(loc.data(), e->buf.site.p, g.n_own * sizeof(float), cudaMemcpyDeviceToHost, e->st));
    B2M_CK(cudaMemcpyAsync(gid.data(), g.gid.p, g.n_own * sizeof(int), cudaMemcpyDeviceToHost, e->st));
    B2M_CK(cudaStreamSynchronize(e->st));
    for (int i = 0; i < g.n_own; i++) full[gid[i]] = loc[i];
  };
  each_member(h, collect);
  Graph& g = h->g;
  if (h->world > 1 && h->parts.empty()) {
    B2M_CK(cudaMemcpyAsync(h->buf.site_full.p, full.data(), g.N * sizeof(float), cudaMemcpyHostToDevice, h->st));
    NCCL_CK(g_nccl.AllReduce(h->buf.site_full.p, h->buf.site_full.p, (size_t)g.N, ncclFloat32, ncclSum, h->comm, h->st));
    B2M_CK(cudaMemcpyAsync(full.data(), h->buf.site_full.p, g.N * sizeof(float), cudaMemcpyDeviceToHost, h->st));
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
  std::string n(name);
  const float* src = nullptr;
  int64_t r = 0, c = D;
  B2M_REQUIRE(h->model->debug(h, n, src, r, c), B2M_ERR_INVALID, "unknown debug tensor: " + n);
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
    e->atomic_last = 0;
    e->hf_n = 0;
    e->buf = Bufs();
    e->model->release();
    e->uf.~Unfold();
    new (&e->uf) Unfold();
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

