// relax_shim.cu -- test-only C entry point into the relax launchers of libb200mlip.so (csrc/relax.cu): one step of S
// structures, all active, from an optimizer state, forces and per-structure energy / virial sums given on the host.
//
// tests/test_gpu_relax.py builds this file into a temporary directory (as tests/kernel_units_ref.py builds
// kernel_shim.cu) and compares the step with tests/relax_ref.py.  The shim copies in, calls launch_relax_struct and
// launch_relax_rows, copies out, and returns 0 or the b2m::Error code with its message; it does no arithmetic of its
// own.
#include <cstring>
#include <exception>
#include <vector>

#include "relax.cuh"

namespace {
template <class T>
T* dev(const T* h, size_t n) {
  T* p = nullptr;
  B2M_CK(cudaMalloc(&p, (n + 1) * sizeof(T)));
  if (h) B2M_CK(cudaMemcpy(p, h, n * sizeof(T), cudaMemcpyHostToDevice));
  return p;
}
template <class T>
void back(T* h, const T* d, size_t n) {
  B2M_CK(cudaMemcpy(h, d, n * sizeof(T), cudaMemcpyDeviceToHost));
}
}  // namespace

extern "C" {

// cfg: fmax, maxstep, dtmax, Nmin, finc, fdec, astart, fa, k, p.  Per structure s (in/out): cell0 [9], X [9], vc [9],
// F [9] (expm(X / n) of the current geometry), dt, a, nsteps.  Rows (in/out): v [N][3], r0 [N][3].  forces [N][3],
// bsum [S][10] as k_batch_sums writes them.  Out: stat [S][12], res_f [N][3], res_e [S], res_s [S][9].
int shim_relax_step(int S, const int64_t* natoms, int it, int steps, int relax_cell, const double* cfg, double* cell0,
                    double* X, double* vc, double* F, double* dt, double* a, int* nsteps, const float* forces,
                    const double* bsum, double data_mean, double* v, double* r0, double* stat, float* res_f,
                    double* res_e, double* res_s, char* msg, int msglen) {
  try {
    std::vector<int64_t> off(S + 1, 0), act(S);
    for (int s = 0; s < S; s++) off[s + 1] = off[s] + natoms[s], act[s] = s;
    const int64_t N = off[S];
    std::vector<int> sid(N);
    for (int s = 0; s < S; s++)
      for (int64_t i = off[s]; i < off[s + 1]; i++) sid[i] = s;
    std::vector<b2m::RelaxStruct> rs(S);
    for (int s = 0; s < S; s++) {
      b2m::RelaxStruct& r = rs[s];
      memset(&r, 0, sizeof r);
      memcpy(r.cell0, cell0 + 9 * s, sizeof r.cell0);
      memcpy(r.X, X + 9 * s, sizeof r.X);
      memcpy(r.vc, vc + 9 * s, sizeof r.vc);
      memcpy(r.F, F + 9 * s, sizeof r.F);
      r.dt = dt[s], r.a = a[s], r.nsteps = nsteps[s];
    }
    b2m::RelaxConst c{cfg[0] * cfg[0], cfg[1], cfg[2], cfg[3], cfg[4], cfg[5], cfg[6], cfg[7], cfg[8], cfg[9],
                      relax_cell, steps};
    int64_t* d_off = dev(off.data(), S + 1);
    int64_t* d_act = dev(act.data(), S);
    int* d_sid = dev(sid.data(), N);
    b2m::RelaxStruct* d_rs = dev(rs.data(), S);
    float* d_f = dev(forces, 3 * N);
    double* d_bsum = dev(bsum, 10 * (size_t)S);
    double* d_v = dev(v, 3 * N);
    double* d_r0 = dev(r0, 3 * N);
    double* d_stat = dev<double>(nullptr, b2m::kRelaxStat * (size_t)S);
    float* d_rf = dev<float>(nullptr, 3 * N);
    double* d_re = dev<double>(nullptr, S);
    double* d_rsig = dev<double>(nullptr, 9 * (size_t)S);
    b2m::launch_relax_struct(0, S, it, c, d_act, d_off, d_off, d_f, d_bsum, data_mean, d_v, d_rs, d_stat, d_rf, d_re,
                             d_rsig, nullptr, 0);
    b2m::launch_relax_rows(0, N, c, d_act, d_off, d_off, d_sid, d_f, d_rs, d_v, d_r0);
    B2M_CK(cudaDeviceSynchronize());
    back(rs.data(), d_rs, S);
    back(v, d_v, 3 * N);
    back(r0, d_r0, 3 * N);
    back(stat, d_stat, b2m::kRelaxStat * (size_t)S);
    back(res_f, d_rf, 3 * N);
    back(res_e, d_re, S);
    back(res_s, d_rsig, 9 * (size_t)S);
    for (void* p : {(void*)d_off, (void*)d_act, (void*)d_sid, (void*)d_rs, (void*)d_f, (void*)d_bsum, (void*)d_v,
                    (void*)d_r0, (void*)d_stat, (void*)d_rf, (void*)d_re, (void*)d_rsig})
      cudaFree(p);
    for (int s = 0; s < S; s++) {
      const b2m::RelaxStruct& r = rs[s];
      memcpy(X + 9 * s, r.X, sizeof r.X);
      memcpy(vc + 9 * s, r.vc, sizeof r.vc);
      memcpy(F + 9 * s, r.F, sizeof r.F);
      dt[s] = r.dt, a[s] = r.a, nsteps[s] = r.nsteps;
    }
    return 0;
  } catch (const b2m::Error& e) {
    if (msg && msglen > 0) strncpy(msg, e.what(), msglen - 1), msg[msglen - 1] = '\0';
    return e.code;
  } catch (const std::exception& e) {
    if (msg && msglen > 0) strncpy(msg, e.what(), msglen - 1), msg[msglen - 1] = '\0';
    return -1;
  }
}

}  // extern "C"
