// tn_state.cuh -- weights and workspace of the TensorNet path (engine_tn.inl drives kernels_tn.cu with it).
#pragma once
#include <vector>

#include "kernels.cuh"

namespace b2m {

struct TnLayerW {
  // edge MLP nrp -> C -> 2C -> 3C on the wgmma row GEMM (engine.cu tc_mm), forward and reverse (W0 with zero rows for the
  // padding rbf columns; W2T in 64-deep K chunks)
  TcW W0, W0T, W1, W1T, W2, W2T;
  const float *b0, *b1, *b2;
  const float *Wt_t[6], *Wt_r[6];  // linears_tensor 0..5: transposed (forward) and raw (reverse)
};
struct TnChainW {  // one hidden Linear of a readout chain
  const float *Wt, *Wr, *b;
  int in, out;
};

// workspace of the resident structure (b2m_release_workspace replaces it with an empty one)
struct TnWork {
  DBuf<float> rbf, cut, P, T0, nr0, ln0, st0, s1p, s1, s2p, T0m;
  DBuf<float> f1, f2;  // [E][C], [E][2C]: activations of the edge MLP (forward), adjoints of its hidden layers (reverse)
  std::vector<DBuf<float>> X;                                       // nblocks + 1 : [n_loc][10][C]
  std::vector<DBuf<float>> f1p, f2p, f3p, q, Xh, Y, msg, Pn, dX;    // per layer
  DBuf<float> inv, str, r, xr, lout, gout, e_atom;
  std::vector<DBuf<float>> cpre[2], cact[2];
  // reverse pass
  DBuf<float> gX, gY, gmsg, gdX, gPn, gf, g_rbf, gC, gvh, gd, gT0m, gT0, gs2p, gs1p, gln0, gnr0, gr, ginv, gxr,
      gca, gcb;
};

struct TnState : TnWork {
  int units = 64, num_rbf = 32, nblocks = 2, so3 = 0;
  TnRadial rp;
  // ---- weights (device pointers into the engine's weight buffer) ----
  TcW Wd, WdT;                 // three distance projections stacked, nrp -> 3C, and the reverse (64-deep K chunks)
  const float* bd = nullptr;   // [3C]
  const float *U = nullptr, *V = nullptr;                       // emb2 halves applied to the embedding table: [n_elem][C]
  const float *Wte_t[3] = {nullptr, nullptr, nullptr}, *Wte_r[3] = {nullptr, nullptr, nullptr};
  const float *ln0_g = nullptr, *ln0_b = nullptr;
  const float *Ws0_t = nullptr, *bs0 = nullptr, *Ws0_r = nullptr, *Ws1_t = nullptr, *bs1 = nullptr, *Ws1_r = nullptr;
  std::vector<TnLayerW> L;
  const float *lnr_g = nullptr, *lnr_b = nullptr, *Wl_t = nullptr, *bl = nullptr, *Wl_r = nullptr;
  std::vector<TnChainW> chain[2];  // hidden layers of final_layer.gated.{layers, gates}
  const float* wlast[2] = {nullptr, nullptr};
  float blast[2] = {0.f, 0.f};
  int wlast_in = 64;
};

}  // namespace b2m
