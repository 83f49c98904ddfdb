// kernel_shim.cu -- test-only C entry points into the shipped CHGNet hot-path launchers of libb200mlip.so.
//
// tests/test_gpu_kernel_units.py builds this file into a temporary directory (tests/kernel_units_ref.py: build_shim)
// and calls it through ctypes.  Each entry point fills the launcher's argument struct from device pointers (torch
// tensors), a stream handle and a num_sms value, calls the launcher, and returns 0 or the b2m::Error code with its
// message; the weight-image entry points run the engine's own host formatters (engine.cu) on host buffers.  The shim
// does no arithmetic of its own.
#include <cstring>
#include <exception>

#include "kernels.cuh"

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

}  // extern "C"
