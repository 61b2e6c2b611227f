// Device-side primitives of the peer-memory exchange (comm.cu, and the cross-rank reductions of the banded L-BFGS step
// in lbfgs.cu): system-scope release / acquire of the iteration stamps, the bounded wait for a peer's stamp, and loads
// of peer data that bypass a possibly stale L1 line.  Also the one home of what every banded row kernel (comm.cu,
// lbfgs.cu, api.cu) must agree on bit for bit: the row vector, the walk over a band's rows, the seam sum of the image
// gradient and the outbox layout.
#pragma once

#include <type_traits>

#include "kernels.h"

namespace stb {

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
static __device__ void wait_stamp(const unsigned long long* flag, unsigned long long want, unsigned long long* err,
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

// V consecutive floats of a row: V = 4 is one 16-byte access (the rows of an image whose width is a multiple of 4, and
// the L-BFGS state vectors, are 16-byte aligned), V = 1 a scalar (odd pyramid widths such as 181 or 543)
template <int V> struct Vec { float v[V]; };
template <int V> using VecWord = std::conditional_t<V == 4, float4, float>;
__device__ __forceinline__ Vec<4> to_vec(const float4& t) { return {{t.x, t.y, t.z, t.w}}; }
__device__ __forceinline__ Vec<1> to_vec(float t) { return {{t}}; }
// the V floats at p + j
template <int V> __device__ __forceinline__ Vec<V> ld(const float* p, long j) {
  return to_vec(*reinterpret_cast<const VecWord<V>*>(p + j));
}
template <int V> __device__ __forceinline__ Vec<V> ld_peer(const float* p, long j) {
  return to_vec(ld_peer(reinterpret_cast<const VecWord<V>*>(p + j)));
}
template <int V> __device__ __forceinline__ void st(float* p, long j, const Vec<V>& a) {
  if constexpr (V == 4) *reinterpret_cast<float4*>(p + j) = make_float4(a.v[0], a.v[1], a.v[2], a.v[3]);
  else p[j] = a.v[0];
}

// calls f(std::integral_constant<int, V>(), n) with the row vector width V of rows of W floats and the number n of
// V-vectors in `rows` such rows (what grid_for sizes a row kernel by)
template <typename F> void with_row_vec(int W, long rows, F&& f) {
  if (W % 4 == 0) f(std::integral_constant<int, 4>(), rows * (W / 4));
  else f(std::integral_constant<int, 1>(), rows * W);
}

// Element i of a walk over rows [row0, row0 + rows) of a [3][h][W] tensor, V floats per element: channel ch, row r of
// the window, first column x, and off, the float offset of the element in the tensor.  32-bit indices: the callers
// refuse bands of 2^31 floats or more.
struct RowPos {
  int ch, r, x;
  long off;
};
template <int V> __device__ __forceinline__ RowPos row_pos(int i, int rows, int W, int h, int row0) {
  const int wv = W / V;
  const int per = rows * wv;
  RowPos p;
  p.ch = (unsigned)i / (unsigned)per;   // unsigned: lets the compiler keep both divisors' reciprocals out of the loop
  const int e = i - p.ch * per;
  p.r = e / wv;
  p.x = (e - p.r * wv) * V;
  p.off = ((long)p.ch * h + row0 + p.r) * W + p.x;
  return p;
}

// Outbox k (0: the first COMM_APRON own rows, 1: the last ones -- the neighbours' next halo) of rank m's mailbox is
// [3][COMM_APRON][W] floats; the address of its row r, channel ch, column x.
__device__ __forceinline__ float* outbox_at(const CommDev& c, int m, int k, int ch, int r, int x) {
  return reinterpret_cast<float*>(c.mbox[m] + c.off_outbox[k]) + ((long)ch * COMM_APRON + r) * c.W + x;
}
// own row r of this band, updated: into the outboxes when it is one of the first / last COMM_APRON own rows
template <int V>
__device__ __forceinline__ void outbox_store(const CommDev& c, int ch, int r, int x, const Vec<V>& v) {
  if (r < COMM_APRON) st<V>(outbox_at(c, c.rank, 0, ch, r, x), 0, v);
  if (r >= c.own_rows - COMM_APRON) st<V>(outbox_at(c, c.rank, 1, ch, r - (c.own_rows - COMM_APRON), x), 0, v);
}

// d loss / d (own row r of this band) at channel ch, column x: the band's local gradient [3][h_local][W] in its
// mailbox, then (add_seams) plus the upper neighbour's bottom-apron rows (its local rows from up_apron_row0) on the
// first COMM_APRON own rows, then plus the lower neighbour's top-apron rows (its local rows [0, COMM_APRON)) on the last
// ones.  Every consumer of the seams sums in this one order, so they all get the same bits.
template <int V>
__device__ __forceinline__ void seam_gradient(const CommDev& c, int ch, int r, int x, bool add_seams,
                                              Vec<V>& out) {
  const float* grad = reinterpret_cast<const float*>(c.mbox[c.rank] + c.off_grad);
  out = ld<V>(grad, ((long)ch * c.h_local + c.own0 + r) * c.W + x);
  if (add_seams && c.rank > 0 && r < COMM_APRON) {
    const float* up = reinterpret_cast<const float*>(c.mbox[c.rank - 1] + c.off_grad);
    const Vec<V> a = ld_peer<V>(up, ((long)ch * c.up_h_local + c.up_apron_row0 + r) * c.W + x);
#pragma unroll
    for (int k = 0; k < V; ++k) out.v[k] += a.v[k];
  }
  if (add_seams && c.rank + 1 < c.world && r >= c.own_rows - COMM_APRON) {
    const float* dn = reinterpret_cast<const float*>(c.mbox[c.rank + 1] + c.off_grad);
    const Vec<V> a = ld_peer<V>(dn, ((long)ch * c.dn_h_local + (r - (c.own_rows - COMM_APRON))) * c.W + x);
#pragma unroll
    for (int k = 0; k < V; ++k) out.v[k] += a.v[k];
  }
}

}  // namespace stb
