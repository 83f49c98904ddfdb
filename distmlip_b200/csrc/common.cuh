// common.cuh -- shared host/device helpers for libb200mlip (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <mutex>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/b200mlip.h"

namespace b2m {

struct Error : public std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

#define B2M_CK(call)                                                                        \
  do {                                                                                      \
    cudaError_t e__ = (call);                                                               \
    if (e__ != cudaSuccess) {                                                               \
      char buf__[512];                                                                      \
      snprintf(buf__, sizeof buf__, "CUDA error %s at %s:%d: %s", cudaGetErrorName(e__),    \
               __FILE__, __LINE__, cudaGetErrorString(e__));                                \
      throw b2m::Error(B2M_ERR_CUDA, buf__);                                                \
    }                                                                                       \
  } while (0)

#define B2M_REQUIRE(cond, code, msg)                         \
  do {                                                       \
    if (!(cond)) throw b2m::Error((code), std::string(msg)); \
  } while (0)

// Grow-only device buffer (resident across MD steps; never shrinks).
template <class T>
struct DBuf {
  T* p = nullptr;
  size_t cap = 0;
  DBuf() = default;
  DBuf(const DBuf&) = delete;
  DBuf& operator=(const DBuf&) = delete;
  DBuf(DBuf&& o) noexcept : p(o.p), cap(o.cap) {
    o.p = nullptr;
    o.cap = 0;
  }
  DBuf& operator=(DBuf&& o) noexcept {  // the buffer held before goes with `o`
    std::swap(p, o.p);
    std::swap(cap, o.cap);
    return *this;
  }
  ~DBuf() {
    if (p) cudaFree(p);
  }
  void ensure(size_t n) {
    if (n <= cap) return;
    if (p) cudaFree(p);
    p = nullptr;
    size_t want = n + n / 8 + 64;
    B2M_CK(cudaMalloc(&p, want * sizeof(T)));
    cap = want;
  }
  void zero(size_t n, cudaStream_t s) { B2M_CK(cudaMemsetAsync(p, 0, n * sizeof(T), s)); }
};

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) applies to the CURRENT device only: guards are per device so that a
// second engine on another GPU of the same process sets them again (ADVICE r1).  The guard holds a lock until the end
// of the `if` statement it is declared in: the partition threads of a single-process group may reach a launcher at
// the same time, and the second one must not launch before the first has finished setting the attribute.
//   if (auto once = attr.first(); once) { cudaFuncSetAttribute(...); }
struct PerDeviceOnce {
  std::mutex m;
  bool done[64] = {};
  struct Guard {
    std::unique_lock<std::mutex> lk;
    bool need;
    explicit operator bool() const { return need; }
  };
  Guard first() {
    Guard g{std::unique_lock<std::mutex>(m), true};
    int d = 0;
    if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= 64) return g;
    g.need = !done[d];
    done[d] = true;
    return g;
  }
};

// Kernels launched by the calling host thread.  Per thread: the partitions of a single-process group run concurrently,
// one host thread each, and run() counts the launches of its own partition as the change across an evaluation.
inline thread_local long long g_launch_count = 0;

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// kern<<<grid, block, smem, st>>>(args...), checked and counted; an empty grid launches nothing
template <class... P, class... A>
void launch(void (*kern)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
  if (grid.x == 0 || grid.y == 0 || grid.z == 0) return;
  kern<<<grid, block, smem, st>>>(std::forward<A>(args)...);
  B2M_CK(cudaGetLastError());
  g_launch_count++;
}

// f(std::bool_constant<b>{}...) for the run-time flags b...: picks a kernel's template instantiation, as in
//   with_flags([&](auto kAtomic) { launch(k<kAtomic>, ...); }, atom_vir != nullptr);
template <class F>
void with_flags(F&& f) {
  f();
}
template <class F, class... B>
void with_flags(F&& f, bool b, B... rest) {
  if (b)
    with_flags([&](auto... c) { f(std::true_type{}, c...); }, rest...);
  else
    with_flags([&](auto... c) { f(std::false_type{}, c...); }, rest...);
}

// ---------------------------------------------------------------- model constants
constexpr int D = 64;    // feature width (atom = bond = angle)
constexpr int D2 = 128;  // both GatedMLP branches stacked
constexpr int NR = 9;    // radial basis size (max_n)
constexpr int NF = 9;    // Fourier features (2*max_f+1)
constexpr int MAXP = 16; // max partitions (slab width rule caps it anyway)

}  // namespace b2m
