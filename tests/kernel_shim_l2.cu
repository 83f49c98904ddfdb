// kernel_shim_l2.cu -- test-only C entry points into the MACE launchers for 0e+1o+2e node features (mace_state.cuh),
// next to every entry point of kernel_shim.cu, which it includes.
//
// tests/test_gpu_mace_l2_units.py and tests/test_oracle_mace_l2.py build this file into a temporary directory
// (tests/mace_l2_units_ref.py: build_shim_l2) and call it through ctypes, as kernel_shim.cu is called.  The shim does
// no arithmetic of its own.
#include "kernel_shim.cu"

extern "C" {

// bwd = 0: launch_mace_msg_l2 (Am =); bwd = 1: launch_mace_msg_l2_bwd (R overwritten with gR, gY +=, gu +=)
int shim_mace_msg_l2(int bwd, void* st, int max_ell, int n_own, int C, const int* row_ptr, const int* e_src, float* R,
                     const float* Y, const float* u, float* Am, const float* gAm, float* gY, float* gu, char* msg,
                     int msglen) {
  return guarded(msg, msglen, [&] {
    if (bwd)
      b2m::launch_mace_msg_l2_bwd((cudaStream_t)st, max_ell, n_own, C, row_ptr, e_src, R, Y, u, gAm, gY, gu);
    else
      b2m::launch_mace_msg_l2((cudaStream_t)st, max_ell, n_own, C, row_ptr, e_src, R, Y, u, Am);
  });
}
// launch_mace_symc_l2 / _bwd.  bwd = 0: out = B [9][n_own][C]; bwd = 1: out = gA (gB read)
int shim_mace_symc_l2(int bwd, void* st, int n_own, int C, int nsh, int Ktot, const int* type, const float* A,
                      const void* terms, int nterms, const float* w, const float* gB, float* out, char* msg, int msglen) {
  return guarded(msg, msglen, [&] {
    const auto* tm = static_cast<const b2m::MaceTerm*>(terms);
    if (bwd)
      b2m::launch_mace_symc_l2_bwd((cudaStream_t)st, n_own, C, nsh, Ktot, type, A, tm, nterms, w, gB, out);
    else
      b2m::launch_mace_symc_l2((cudaStream_t)st, n_own, C, nsh, Ktot, type, A, tm, nterms, w, out);
  });
}

}  // extern "C"
