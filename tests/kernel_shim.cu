// kernel_shim.cu -- test-only C entry points into the shipped CHGNet hot-path launchers, the MACE launchers
// (mace_state.cuh) and the TensorNet launchers (kernels.cuh) of libb200mlip.so.
//
// tests/test_gpu_kernel_units.py, tests/test_gpu_mace_units.py and tests/test_gpu_tn_units.py build this file into a
// temporary directory (tests/kernel_units_ref.py: build_shim) and call it through ctypes.  Each entry point fills the
// launcher's argument struct from device pointers (torch tensors), a stream handle and a num_sms value, calls the
// launcher, and returns 0 or the b2m::Error code with its message; the weight-image entry points run the engine's own host formatters (engine.cu) on host buffers, and the MACE
// host entry points the engine's own conv-path list and symmetric-contraction term builder (engine_mace.inl).  The shim
// does no arithmetic of its own.
#include <algorithm>
#include <cstring>
#include <exception>

#include "mace_state.cuh"

namespace {
int fail(int code, const char* what, char* msg, int msglen) {
  if (msg != nullptr && msglen > 0) {
    strncpy(msg, what, (size_t)msglen - 1);
    msg[msglen - 1] = '\0';
  }
  return code;
}
template <class F>
int guarded(char* msg, int msglen, F&& fn) {
  try {
    fn();
    return 0;
  } catch (const b2m::Error& e) {
    return fail(e.code, e.what(), msg, msglen);
  } catch (const std::exception& e) {
    return fail(-1, e.what(), msg, msglen);
  }
}
b2m::RadialParams radial_params(const float* freq, float rc, float norm, int p) {
  b2m::RadialParams rp;
  memcpy(rp.freq, freq, sizeof rp.freq);
  rp.rc = rc;
  rp.norm = norm;
  rp.p = p;
  return rp;
}
std::vector<float> host_vec(const float* p, size_t n) { return std::vector<float>(p, p + n); }
void put(const std::vector<float>& v, float* out) { memcpy(out, v.data(), v.size() * sizeof(float)); }
// MaceRadial from nb, p, r_max, the prefactor and the nb Bessel frequencies w (host); pitch 64 as the engine sets it
b2m::MaceRadial mace_radial(int nb, int p, float r_max, float pref, const float* w) {
  b2m::MaceRadial rp{};
  rp.nb = nb, rp.nbp = 64, rp.p = p, rp.r_max = r_max, rp.pref = pref;
  for (int n = 0; n < 64; n++) rp.w[n] = n < nb ? w[n] : 0.f;
  return rp;
}
// MaceCore from the element table (device float4 [n_elem]) and cf = (za, zc[4], zscale, aq, ap, aa) (host)
b2m::MaceCore mace_core(const float* elem, int zbl, int agnesi, int zp, const float* cf) {
  b2m::MaceCore c{};
  c.elem = reinterpret_cast<const float4*>(elem);
  c.zbl = zbl, c.agnesi = agnesi, c.zp = zp;
  c.za = cf[0];
  for (int k = 0; k < 4; k++) c.zc[k] = cf[1 + k];
  c.zscale = cf[5], c.aq = cf[6], c.ap = cf[7], c.aa = cf[8];
  return c;
}
// TnRadial from nr, the row pitch nrp, width, rc and the nr centres mu (host); centres past nr are 0 as the engine sets them
b2m::TnRadial tn_radial(int nr, int nrp, float width, float rc, const float* mu) {
  b2m::TnRadial rp{};
  rp.nr = nr, rp.nrp = nrp, rp.width = width, rp.rc = rc;
  for (int k = 0; k < 64; k++) rp.mu[k] = k < nr ? mu[k] : 0.f;
  return rp;
}
}  // namespace

extern "C" {

int shim_gemm_wg(void* st, const float* A, int lda, const float* Bcan, float* C, int ldc, int M, int N, int K,
                 const float* bias, const float* R, int ldr, int accum, int epi, float* Cpre, const float* Pre, int ldp,
                 int num_sms, char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    b2m::launch_gemm_wg((cudaStream_t)st, A, lda, Bcan, C, ldc, M, N, K, bias, R, ldr, accum != 0, epi, Cpre, Pre, ldp,
                        num_sms);
  });
}

// bwd = 0: launch_atomconv_fwd (agg +=); bwd = 1: launch_atomconv_bwd (gA / gC +=, gQ =, gd +=)
int shim_atomconv(int bwd, void* st, int64_t E, const int* e_src, const int* e_dst, const int* e_bond,
                  const float* e_vec, const float* Aproj, const float* Cproj, const float* Qproj, const float* radial,
                  const float* W2can, const float* W2Tcan, const float* b2, const float* freq, float rc, float norm,
                  int p, float* agg, const float* gagg, float* gA, float* gC, float* gQ, float* gd, int num_sms,
                  char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    b2m::AtomConvArgs a;
    memset(&a, 0, sizeof a);
    a.E = E;
    a.e_src = e_src, a.e_dst = e_dst, a.e_bond = e_bond, a.e_vec = reinterpret_cast<const float4*>(e_vec);
    a.Aproj = Aproj, a.Cproj = Cproj, a.Qproj = Qproj;
    a.radial = radial, a.W2can = W2can, a.W2Tcan = W2Tcan, a.b2 = b2;
    a.rp = radial_params(freq, rc, norm, p);
    a.agg = agg;
    a.gagg = gagg, a.gA = gA, a.gC = gC, a.gQ = gQ, a.gd = gd;
    if (bwd)
      b2m::launch_atomconv_bwd((cudaStream_t)st, a, num_sms);
    else
      b2m::launch_atomconv_fwd((cudaStream_t)st, a, num_sms);
  });
}

// bwd = 0: launch_line_fwd (hidden: aggB +=; !hidden: ang_out =); bwd = 1: launch_line_bwd (gang, gHa, gHb, gXc +=)
int shim_line(int bwd, int hidden, void* st, int64_t A, const int* a_in, const int* a_out, const int* a_ctr,
              const float* ang, const float* Ha, const float* Hb, const float* Xc, const float* Wgcan,
              const float* WgTcan, const float* W2can, const float* W2Tcan, const float* b2, float* aggB, float* ang_out,
              const float* gaggB, float* gang, float* gHa, float* gHb, float* gXc, int num_sms, char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    b2m::LineArgs a;
    memset(&a, 0, sizeof a);
    a.A = A;
    a.a_in = a_in, a.a_out = a_out, a.a_ctr = a_ctr;
    a.ang = ang, a.Ha = Ha, a.Hb = Hb, a.Xc = Xc;
    a.Wgcan = Wgcan, a.WgTcan = WgTcan, a.W2can = W2can, a.W2Tcan = W2Tcan, a.b2 = b2;
    a.aggB = aggB, a.ang_out = ang_out;
    a.gaggB = gaggB, a.gang = gang, a.gHa = gHa, a.gHb = gHb, a.gXc = gXc;
    if (bwd)
      b2m::launch_line_bwd((cudaStream_t)st, a, hidden != 0, num_sms);
    else
      b2m::launch_line_fwd((cudaStream_t)st, a, hidden != 0, num_sms);
  });
}

// weight images, host buffers in and out (sizes: canon_split 2 N Kpad, permute_k8 N K, second_layer_can and
// line_reverse_can 16384, radial_can ATOM_RAD)
int shim_canon_split(const float* raw, int N, int K, int Kpad, float* out, char* msg, int msglen) {
  return guarded(msg, msglen, [&] { put(b2m::canon_split(host_vec(raw, (size_t)N * K), N, K, Kpad), out); });
}
int shim_permute_k8(const float* raw, int N, int K, float* out, char* msg, int msglen) {
  return guarded(msg, msglen, [&] { put(b2m::permute_k8(host_vec(raw, (size_t)N * K), N, K), out); });
}
int shim_second_layer_can(const float* raw128x64, int transposed, float* out, char* msg, int msglen) {
  return guarded(msg, msglen, [&] { put(b2m::second_layer_can(host_vec(raw128x64, 128 * 64), transposed != 0), out); });
}
int shim_line_reverse_can(const float* raw128x64, float* out, char* msg, int msglen) {
  return guarded(msg, msglen, [&] { put(b2m::line_reverse_can(host_vec(raw128x64, 128 * 64)), out); });
}
int shim_radial_can(const float* M, const float* Wab, float* out, char* msg, int msglen) {
  return guarded(msg, msglen, [&] { put(b2m::radial_can(host_vec(M, 128 * 9), host_vec(Wab, 64 * 9)), out); });
}
int shim_atom_rad() { return b2m::ATOM_RAD; }

// ---------------------------------------------------------------------------------------------- MACE (mace_state.cuh)
int shim_mace_edge_geom(void* st, int64_t E, const float* e_vec, int nb, int p, float r_max, float pref, const float* w,
                        int nsh, float* Y, float* eb, const int* e_src, const int* e_dst, const int* type,
                        const float* elem, int zbl, int agnesi, int zp, const float* cf, char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    b2m::launch_mace_edge_geom((cudaStream_t)st, E, reinterpret_cast<const float4*>(e_vec), mace_radial(nb, p, r_max, pref, w),
                               nsh, Y, eb, e_src, e_dst, type, mace_core(elem, zbl, agnesi, zp, cf));
  });
}
int shim_mace_zbl(void* st, int n_own, const int* row_ptr, const int* e_src, const float* e_vec, const int* type,
                  const float* elem, int zbl, int agnesi, int zp, const float* cf, float* e_lin, char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    b2m::launch_mace_zbl((cudaStream_t)st, n_own, row_ptr, e_src, reinterpret_cast<const float4*>(e_vec), type,
                         mace_core(elem, zbl, agnesi, zp, cf), e_lin);
  });
}
int shim_mace_embed(void* st, int n, int C, const int* type, const float* W, float* h0, char* msg, int msglen) {
  return guarded(msg, msglen, [&] { b2m::launch_mace_embed((cudaStream_t)st, n, C, type, W, h0); });
}
// bwd = 0: launch_mace_msg (A =); bwd = 1: launch_mace_msg_bwd (gR =, gY +=, gu +=)
int shim_mace_msg(int bwd, void* st, int n_own, int C, int L1, const int* row_ptr, const int* e_src, const float* R,
                  const float* Y, const float* u, float* A, const float* gA, float* gR, float* gY, float* gu, char* msg,
                  int msglen) {
  return guarded(msg, msglen, [&] {
    if (bwd)
      b2m::launch_mace_msg_bwd((cudaStream_t)st, n_own, C, L1, row_ptr, e_src, R, Y, u, gA, gR, gY, gu);
    else
      b2m::launch_mace_msg((cudaStream_t)st, n_own, C, L1, row_ptr, e_src, R, Y, u, A);
  });
}
// bwd = 0: launch_mace_msg_eq (Am =); bwd = 1: launch_mace_msg_eq_bwd (R overwritten with gR, gY +=, gu +=)
int shim_mace_msg_eq(int bwd, void* st, int max_ell, int n_own, int C, const int* row_ptr, const int* e_src, float* R,
                     const float* Y, const float* u, float* Am, const float* gAm, float* gY, float* gu, char* msg,
                     int msglen) {
  return guarded(msg, msglen, [&] {
    if (bwd)
      b2m::launch_mace_msg_eq_bwd((cudaStream_t)st, max_ell, n_own, C, row_ptr, e_src, R, Y, u, gAm, gY, gu);
    else
      b2m::launch_mace_msg_eq((cudaStream_t)st, max_ell, n_own, C, row_ptr, e_src, R, Y, u, Am);
  });
}
int shim_mace_elem_mix(void* st, int n, int C, int L1, int nsh, const int* type, const float* W, const float* in,
                       float* out, int accum, char* msg, int msglen) {
  return guarded(msg, msglen,
                 [&] { b2m::launch_mace_elem_mix((cudaStream_t)st, n, C, L1, nsh, type, W, in, out, accum != 0); });
}
int shim_mace_elem_mix_rows(void* st, int n, int C, int ncomp, int ldi, int ldo, const int* type, const float* W,
                            const float* in, float* out, int accum, char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    b2m::launch_mace_elem_mix_rows((cudaStream_t)st, n, C, ncomp, ldi, ldo, type, W, in, out, accum != 0);
  });
}
// eq = 0: launch_mace_symc / _bwd; eq = 1: launch_mace_symc_eq / _bwd.  bwd = 0: out = B; bwd = 1: out = gA (gB read)
int shim_mace_symc(int eq, int bwd, void* st, int n_own, int C, int nsh, int Ktot, const int* type, const float* A,
                   const void* terms, int nterms, const float* w, const float* gB, float* out, char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    const auto* tm = static_cast<const b2m::MaceTerm*>(terms);
    cudaStream_t s = (cudaStream_t)st;
    if (eq && bwd) b2m::launch_mace_symc_eq_bwd(s, n_own, C, nsh, Ktot, type, A, tm, nterms, w, gB, out);
    else if (eq) b2m::launch_mace_symc_eq(s, n_own, C, nsh, Ktot, type, A, tm, nterms, w, out);
    else if (bwd) b2m::launch_mace_symc_bwd(s, n_own, C, nsh, Ktot, type, A, tm, nterms, w, gB, out);
    else b2m::launch_mace_symc(s, n_own, C, nsh, Ktot, type, A, tm, nterms, w, out);
  });
}
int shim_mace_readout_lin(void* st, int n_own, int C, int ld, const float* h, const float* w, float* e_lin, char* msg,
                          int msglen) {
  return guarded(msg, msglen, [&] { b2m::launch_mace_readout_lin((cudaStream_t)st, n_own, C, ld, h, w, e_lin); });
}
int shim_mace_readout_final(void* st, int n_own, int C, int H, const float* h, const float* W1, const float* w2,
                            const float* e_lin, const int* type, const double* E0, double scale, double shift, float* pre,
                            double* energy, const int* gid, double* atom_e, const float* wgt, char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    b2m::launch_mace_readout_final((cudaStream_t)st, n_own, C, H, h, W1, w2, e_lin, type, E0, scale, shift, pre, energy,
                                   gid, atom_e, wgt);
  });
}
int shim_mace_readout_seed(void* st, int n_own, int C, int H, const float* pre, const float* W1, const float* w2,
                           float scale, float* gh, const int* gid, const float* wgt, char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    b2m::launch_mace_readout_seed((cudaStream_t)st, n_own, C, H, pre, W1, w2, scale, gh, gid, wgt);
  });
}
int shim_mace_add_row(void* st, int n_own, int C, int ld, const float* w, float scale, float* gh, const int* gid,
                      const float* wgt, char* msg, int msglen) {
  return guarded(msg, msglen, [&] { b2m::launch_mace_add_row((cudaStream_t)st, n_own, C, ld, w, scale, gh, gid, wgt); });
}
int shim_mace_edge_final(void* st, int64_t E, int nsh, const int* e_src, const int* e_dst, const float* e_vec,
                         const int* gid, const int* type, int nb, int p, float r_max, float pref, const float* w,
                         const float* elem, int zbl, int agnesi, int zp, const float* cf, const float* g_eb,
                         const float* gY, float* forces, double* virial, float* atom_vir, const float* wgt, char* msg,
                         int msglen) {
  return guarded(msg, msglen, [&] {
    b2m::launch_mace_edge_final((cudaStream_t)st, E, nsh, e_src, e_dst, reinterpret_cast<const float4*>(e_vec), gid, type,
                                mace_radial(nb, p, r_max, pref, w), mace_core(elem, zbl, agnesi, zp, cf), g_eb, gY,
                                forces, virial, atom_vir, wgt);
  });
}
// host: the engine's conv_tp path list into out [3 * cap] (l_in, l_sh, l_out per path); *n = its length
int shim_mace_conv_paths(int max_ell, int hidden_l, int* out, int cap, int* n, char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    const auto p = b2m::mace_conv_paths(max_ell, hidden_l);
    *n = (int)p.size();
    for (int k = 0; k < *n && k < cap; k++)
      for (int j = 0; j < 3; j++) out[3 * k + j] = p[k][j];
  });
}
// host: the engine's symmetric-contraction terms of one U (host [ncomp][nsh]^nu [K]) into out (MaceTerm [cap]); *n = count
int shim_mace_sym_terms(const float* U, int nsh, int nu, int ncomp, int K, int kg0, void* out, int cap, int* n,
                        char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    const auto t = b2m::mace_sym_terms(U, nsh, nu, ncomp, K, kg0);
    *n = (int)t.size();
    memcpy(out, t.data(), std::min(t.size(), (size_t)cap) * sizeof(b2m::MaceTerm));
  });
}

// ---------------------------------------------------------------------------------------------- TensorNet (kernels.cuh)
int shim_tn_gemm(void* st, const float* A, int lda, int64_t zA, const float* B0, const float* B1, const float* B2,
                 int bsel, float* C, int ldc, int64_t zC, float* Cpre, const float* Pre, int ldp, const float* bias, int M,
                 int N, int K, int accum, int epi, int nz, char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    b2m::TnGemm g;
    g.A = A, g.lda = lda, g.zA = zA, g.B0 = B0, g.B1 = B1, g.B2 = B2, g.bsel = bsel;
    g.C = C, g.ldc = ldc, g.zC = zC, g.Cpre = Cpre, g.Pre = Pre, g.ldp = ldp, g.bias = bias;
    g.M = M, g.N = N, g.K = K, g.accum = accum, g.epi = epi;
    b2m::launch_tn_gemm((cudaStream_t)st, g, nz);
  });
}
int shim_tn_edge_geom(void* st, int64_t E, const float* e_vec, int nr, int nrp, float width, float rc, const float* mu,
                      float* rbf, float* cut, char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    b2m::launch_tn_edge_geom((cudaStream_t)st, E, reinterpret_cast<const float4*>(e_vec),
                             tn_radial(nr, nrp, width, rc, mu), rbf, cut);
  });
}
// bwd = 0: launch_tn_embed_agg (T0 =, nr0 =) over n_own rows; bwd = 1: launch_tn_embed_agg_bwd over E edges
// (gP =, gC +=, gvh =)
int shim_tn_embed_agg(void* st, int bwd, int n_own, int64_t E, const int* row_ptr, const int* e_src, const int* e_dst,
                      const int* type, const float* U, const float* V, const float* P, const float* cut,
                      const float* e_vec, float* T0, float* nr0, const float* gT0, float* gP, float* gC, float* gvh,
                      char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    const auto* ev = reinterpret_cast<const float4*>(e_vec);
    if (bwd)
      b2m::launch_tn_embed_agg_bwd((cudaStream_t)st, E, e_src, e_dst, type, U, V, P, cut, ev, gT0, gP, gC, gvh);
    else
      b2m::launch_tn_embed_agg((cudaStream_t)st, n_own, row_ptr, e_src, type, U, V, P, cut, ev, T0, nr0);
  });
}
// bwd = 0: y =, stats =; bwd = 1: gx = (gy and stats read)
int shim_tn_layernorm(void* st, int bwd, int rows, int W, const float* x, const float* gamma, const float* beta,
                      float* y, float* stats, const float* gy, float* gx, char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    if (bwd)
      b2m::launch_tn_layernorm_bwd((cudaStream_t)st, rows, W, x, stats, gamma, gy, gx);
    else
      b2m::launch_tn_layernorm((cudaStream_t)st, rows, W, x, gamma, beta, y, stats);
  });
}
// bwd = 0: X0 =; bwd = 1: gT0m =, gs2p =
int shim_tn_embed_out(void* st, int bwd, int n, const float* T0m, const float* s2p, float* X0, const float* gX0,
                      float* gT0m, float* gs2p, char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    if (bwd)
      b2m::launch_tn_embed_out_bwd((cudaStream_t)st, n, T0m, s2p, gX0, gT0m, gs2p);
    else
      b2m::launch_tn_embed_out((cudaStream_t)st, n, T0m, s2p, X0);
  });
}
int shim_tn_norm_bwd_add(void* st, int n, const float* T0, const float* gnr0, float* gT0, char* msg, int msglen) {
  return guarded(msg, msglen, [&] { b2m::launch_tn_norm_bwd_add((cudaStream_t)st, n, T0, gnr0, gT0); });
}
// bwd = 0: Xh =, q =; bwd = 1: g overwritten with the adjoint of X (q read)
int shim_tn_scale(void* st, int bwd, int n, const float* X, float* Xh, float* q, float* g, char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    if (bwd)
      b2m::launch_tn_scale_bwd((cudaStream_t)st, n, X, q, g);
    else
      b2m::launch_tn_scale((cudaStream_t)st, n, X, Xh, q);
  });
}
// bwd = 0: msg =; bwd = 1: g3 =, gC +=, gY += (red.add into source rows)
int shim_tn_msg(void* st, int bwd, int n_own, const int* row_ptr, const int* e_src, const float* f3p, const float* cut,
                const float* Y, float* out, const float* gmsg, float* g3, float* gC, float* gY, char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    if (bwd)
      b2m::launch_tn_msg_bwd((cudaStream_t)st, n_own, row_ptr, e_src, f3p, cut, Y, gmsg, g3, gC, gY);
    else
      b2m::launch_tn_msg((cudaStream_t)st, n_own, row_ptr, e_src, f3p, cut, Y, out);
  });
}
// bwd = 0: Pn =; bwd = 1: gmsg =, gY =
int shim_tn_prod(void* st, int bwd, int n, const float* m, const float* Y, int so3, float* Pn, const float* gPn,
                 float* gmsg, float* gY, char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    if (bwd)
      b2m::launch_tn_prod_bwd((cudaStream_t)st, n, m, Y, so3, gPn, gmsg, gY);
    else
      b2m::launch_tn_prod((cudaStream_t)st, n, m, Y, so3, Pn);
  });
}
// bwd = 0: Xn =; bwd = 1: gdX = (Xh unused)
int shim_tn_update(void* st, int bwd, int n, const float* Xh, const float* dX, float* Xn, const float* gXn, float* gdX,
                   char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    if (bwd)
      b2m::launch_tn_update_bwd((cudaStream_t)st, n, dX, gXn, gdX);
    else
      b2m::launch_tn_update((cudaStream_t)st, n, Xh, dX, Xn);
  });
}
// bwd = 0: inv =; bwd = 1: gX =
int shim_tn_invariants(void* st, int bwd, int n, const float* X, float* inv, const float* ginv, float* gX, char* msg,
                       int msglen) {
  return guarded(msg, msglen, [&] {
    if (bwd)
      b2m::launch_tn_invariants_bwd((cudaStream_t)st, n, X, ginv, gX);
    else
      b2m::launch_tn_invariants((cudaStream_t)st, n, X, inv);
  });
}
// atom_e and wgt null or not pick the instantiation; eref may be null
int shim_tn_readout_final(void* st, int n, int W, const float* hL, const float* wL, float bL, const float* hG,
                          const float* wG, float bG, const int* type, const double* eref, float scale, float* lout,
                          float* gout, float* e_atom, double* energy, const int* gid, double* atom_e,
                          double mean_per_atom, const float* wgt, char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    b2m::launch_tn_readout_final((cudaStream_t)st, n, W, hL, wL, bL, hG, wG, bG, type, eref, scale, lout, gout, e_atom,
                                 energy, gid, atom_e, mean_per_atom, wgt);
  });
}
int shim_tn_readout_seed(void* st, int n, int W, const float* lout, const float* gout, float scale, const float* wL,
                         const float* wG, const float* preL, const float* preG, float* gL, float* gG, const int* gid,
                         const float* wgt, char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    b2m::launch_tn_readout_seed((cudaStream_t)st, n, W, lout, gout, scale, wL, wG, preL, preG, gL, gG, gid, wgt);
  });
}
// gd =, forces +=, virial +=, atom_vir += (null: the plain instantiation)
int shim_tn_edge_final(void* st, int64_t E, const int* e_src, const int* e_dst, const float* e_vec, const int* gid,
                       int nr, int nrp, float width, float rc, const float* mu, const float* g_rbf, const float* gC,
                       const float* gvh, float* gd, float* forces, double* virial, float* atom_vir, char* msg,
                       int msglen) {
  return guarded(msg, msglen, [&] {
    b2m::launch_tn_edge_final((cudaStream_t)st, E, e_src, e_dst, reinterpret_cast<const float4*>(e_vec), gid,
                              tn_radial(nr, nrp, width, rc, mu), g_rbf, gC, gvh, gd, forces, virial, atom_vir);
  });
}

}  // extern "C"
