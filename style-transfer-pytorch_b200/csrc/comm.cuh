// Device-side primitives of the peer-memory exchange (comm.cu, and the cross-rank reductions of the banded L-BFGS step
// in lbfgs.cu): system-scope release / acquire of the iteration stamps, the bounded wait for a peer's stamp, and loads
// of peer data that bypass a possibly stale L1 line.
#pragma once

#include "kernels.h"

namespace stb {
namespace {

__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
// peer data: the local L1 may hold a stale copy of a remote line (peer accesses bypass the local L2 but not L1)
__device__ __forceinline__ float4 ld_peer(const float4* p) { return __ldcv(p); }
__device__ __forceinline__ float ld_peer(const float* p) { return __ldcv(p); }
__device__ __forceinline__ double ld_peer(const double* p) { return __ldcv(p); }

// spin until *flag >= want; past timeout_ns the wanted stamp goes to *err and the kernel traps (the launch fails with a
// CUDA error) instead of hanging
__device__ void wait_stamp(const unsigned long long* flag, unsigned long long want, unsigned long long* err,
                           unsigned long long timeout_ns) {
  if (ld_acquire_sys(flag) >= want) return;
  const unsigned long long t0 = globaltimer_ns();
  unsigned spins = 0;
  while (ld_acquire_sys(flag) < want) {
    if ((++spins & 0xFF) == 0 && globaltimer_ns() - t0 > timeout_ns) {
      *err = want;
      __threadfence_system();
      __trap();
    }
  }
}

}  // namespace
}  // namespace stb
