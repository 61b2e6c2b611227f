// Peer-memory exchange of the spatially tiled (multi-GPU) iteration: SURVEY.md section 8e, DESIGN.md section 6.
//
// One process per GPU.  Every rank owns a MAILBOX (one cudaMalloc block, exported with CUDA IPC and mapped by all
// peers over NVLink / NVSwitch); a rank only ever WRITES its own mailbox and READS the peers' -- "pull" everywhere:
//
//   flags[]       monotonically increasing iteration stamps {stats, grad, halo} of the owner
//   stats[2]      the owner's band-local statistics block (Gram sums, channel sums, content SSE, TV sum; 2.4 MB),
//                 double buffered by iteration parity
//   grad          d loss / d (local image) of the owner, [3][h_local][W] fp32: its apron rows are the contributions
//                 the neighbouring bands add to their own rows (the "single reduce at the seams" of the north star)
//   outbox[2]     the owner's first / last APRON updated image rows, i.e. the neighbours' next halo
//
// An iteration is ONE CUDA graph per rank (api.cu: stb_iterate_banded); the exchanges are kernels inside it:
//   comm_phase_kernel   1 warp: publishes an iteration stamp (release, system scope) and/or waits for the peers'
//                       stamps (acquire loads of the peer flags over NVLink).  Kept apart from the data kernels so
//                       that a waiting rank occupies one warp, not the GPU.
//   halo_pull_kernel    neighbours' outboxes -> halo rows of the local image
//   stats_publish / stats_allreduce_kernel
//                       all-reduce of the statistics block as "everybody sums everybody's slot in rank order":
//                       deterministic, and bit-identical on every rank, so the replicated W2 chain stays in lock step
//   adam_seam_kernel    seam reduce of the image gradient (own + neighbours' apron rows) fused with Adam + clamp + EMA
//                       (torch/optim/adam.py:413-546, ST:483-486) and with the fill of the outboxes
//   lbfgs_seam_gather   the same seam reduce for the banded L-BFGS step (lbfgs.cu), into its compact gradient
// A wait that is not satisfied within CommDev::timeout_ns (30 s; STB_COMM_TIMEOUT_S) traps (the launch fails with a CUDA error) instead of hanging.
#include <cstring>

#include "comm.cuh"
#include "kernels.h"
#include "ptx.cuh"

namespace stb {

namespace {

// Row-wise kernels run on float4 when the image width is a multiple of 4 (rows are then 16-byte aligned) and on
// scalars otherwise (odd pyramid widths such as 181 or 543).
template <int V> struct Vec;
template <> struct Vec<4> { typedef float4 T; };
template <> struct Vec<1> { typedef float T; };
__device__ __forceinline__ void unpack(const float4& v, float (&a)[4]) { a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w; }
__device__ __forceinline__ void unpack(const float& v, float (&a)[1]) { a[0] = v; }
__device__ __forceinline__ void pack(float4& v, const float (&a)[4]) { v = make_float4(a[0], a[1], a[2], a[3]); }
__device__ __forceinline__ void pack(float& v, const float (&a)[1]) { v = a[0]; }

// phase 0 BEGIN : t = ++iter;                     wait halo  stamps of the neighbours >= t - 1
// phase 1 STATS : publish stats stamp = t;        wait stats stamps of ALL ranks      >= t
// phase 2 GRAD  : publish grad  stamp = t;        wait grad  stamps of the neighbours >= t
// phase 3 END   : publish halo  stamp = t
__global__ void comm_phase_kernel(CommDev c, int phase) {
  unsigned long long* own = reinterpret_cast<unsigned long long*>(c.mbox[c.rank]);
  unsigned long long t = own[COMM_ITER];
  if (phase == 0) {
    t += 1;
    __syncwarp();
    if (threadIdx.x == 0) own[COMM_ITER] = t;
  }
  const int lane = threadIdx.x;
  if (lane == 0 && phase >= 1) {
    __threadfence_system();  // everything earlier kernels of this stream wrote is visible before the stamp
    st_release_sys(own + (phase == 1 ? COMM_FLAG_STATS : phase == 2 ? COMM_FLAG_GRAD : COMM_FLAG_HALO), t);
  }
  if (phase == 3 || lane >= c.world || lane == c.rank) return;
  const bool neighbour = lane == c.rank - 1 || lane == c.rank + 1;
  const unsigned long long* peer = reinterpret_cast<const unsigned long long*>(c.mbox[lane]);
  if (phase == 0 && neighbour) wait_stamp(peer + COMM_FLAG_HALO, t - 1, own + COMM_ERR, c.timeout_ns);
  if (phase == 1) wait_stamp(peer + COMM_FLAG_STATS, t, own + COMM_ERR, c.timeout_ns);
  if (phase == 2 && neighbour) wait_stamp(peer + COMM_FLAG_GRAD, t, own + COMM_ERR, c.timeout_ns);
}

// halo rows of the local image <- the neighbours' outboxes (skipped in the first iteration after a reset: the halo
// then still holds the rows the host sliced out of the full image)
template <int V>
__global__ void __launch_bounds__(256) halo_pull_kernel(CommDev c, float* __restrict__ img) {
  typedef typename Vec<V>::T T;
  const unsigned long long t = reinterpret_cast<const unsigned long long*>(c.mbox[c.rank])[COMM_ITER];
  if (t <= 1) return;
  const int w4 = c.W / V;
  const long per_side = 3l * COMM_APRON * w4;
  const int sides = (c.rank > 0 ? 1 : 0) + (c.rank + 1 < c.world ? 1 : 0);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < per_side * sides; i += (long)gridDim.x * blockDim.x) {
    int side = (int)(i / per_side);           // 0: from the upper neighbour, 1: from the lower one
    const long e = i - side * per_side;
    if (c.rank == 0) side = 1;
    const int ch = (int)(e / ((long)COMM_APRON * w4));
    const long r4 = e - (long)ch * COMM_APRON * w4;
    const int row = (int)(r4 / w4), x4 = (int)(r4 - (long)row * w4);
    // upper neighbour's LAST own rows = its outbox 1; lower neighbour's FIRST own rows = its outbox 0
    const uint8_t* peer = c.mbox[side == 0 ? c.rank - 1 : c.rank + 1];
    const T* src = reinterpret_cast<const T*>(peer + c.off_outbox[side == 0 ? 1 : 0]) +
                   ((long)ch * COMM_APRON + row) * w4 + x4;
    const int dst_row = side == 0 ? row : c.own0 + c.own_rows + row;
    reinterpret_cast<T*>(img)[((long)ch * c.h_local + dst_row) * w4 + x4] = ld_peer(src);
  }
}

__global__ void __launch_bounds__(256) stats_publish_kernel(CommDev c, const float* __restrict__ stats, long n4) {
  const unsigned long long t = reinterpret_cast<const unsigned long long*>(c.mbox[c.rank])[COMM_ITER];
  float4* dst = reinterpret_cast<float4*>(c.mbox[c.rank] + c.off_stats[t & 1]);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x)
    dst[i] = reinterpret_cast<const float4*>(stats)[i];
}

// stats[e] = sum over ranks (in rank order, own slot included) of slot_r[e]
__global__ void __launch_bounds__(256) stats_allreduce_kernel(CommDev c, float* __restrict__ stats, long n4) {
  const unsigned long long t = reinterpret_cast<const unsigned long long*>(c.mbox[c.rank])[COMM_ITER];
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
    for (int r0 = 0; r0 < c.world; r0 += 4) {   // up to four loads in flight per thread (NVLink latency ~2 us)
      float4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (r0 + u < c.world)
          v[u] = ld_peer(reinterpret_cast<const float4*>(c.mbox[r0 + u] + c.off_stats[t & 1]) + i);
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (r0 + u < c.world) { acc.x += v[u].x; acc.y += v[u].y; acc.z += v[u].z; acc.w += v[u].w; }
    }
    reinterpret_cast<float4*>(stats)[i] = acc;
  }
}

// own rows: g = grad_local (+ upper neighbour's bottom-apron rows) (+ lower neighbour's top-apron rows); Adam; clamp;
// EMA; the first / last APRON updated rows also go to the outboxes (the neighbours' next halo)
// Per-layer halo exchange (DESIGN.md section 6, "halo mode"): the band computed only its own rows of a tensor; the one
// row above / below them that the next 3x3 kernel reads is the neighbour's boundary own row, pulled here.  One kernel =
// publish my progress stamp (everything before it on this stream is done: kernel boundary + system fence), wait for the
// neighbours' same stamp, copy.  Few small CTAs: a waiting rank leaves the GPU to whoever shares it.
__global__ void __launch_bounds__(256) halo_rows_kernel(CommDev c, HaloRowArgs a) {
  // launched with programmatic stream serialization: the grid may become resident while the producing kernel drains;
  // nothing of it is touched (and nothing is published) before that kernel has completed
  asm volatile("griddepcontrol.wait;" ::: "memory");
  // letting the NEXT kernel (a PDL-launched conv) become resident now is only safe when this rank has the GPU to itself:
  // its CTAs would sit on every SM waiting for this kernel, which waits for a rank that may need those SMs (CommDev::pdl)
  if (c.pdl) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  unsigned long long* own = reinterpret_cast<unsigned long long*>(c.mbox[c.rank]);
  const unsigned long long want = own[COMM_ITER] * 256ull + (unsigned long long)a.seq;
  if (threadIdx.x == 0) {
    if (blockIdx.x == 0) {
      __threadfence_system();
      st_release_sys(own + COMM_PROG, want);
    }
    if (a.src_up != nullptr)
      wait_stamp(reinterpret_cast<const unsigned long long*>(c.mbox[c.rank - 1]) + COMM_PROG, want, own + COMM_ERR,
                 c.timeout_ns);
    if (a.src_dn != nullptr)
      wait_stamp(reinterpret_cast<const unsigned long long*>(c.mbox[c.rank + 1]) + COMM_PROG, want, own + COMM_ERR,
                 c.timeout_ns);
  }
  __syncthreads();
  const long n16 = (long)(a.row_bytes >> 4);
  const int sides = (a.src_up != nullptr ? 1 : 0) + (a.src_dn != nullptr ? 1 : 0);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n16 * sides; i += (long)gridDim.x * blockDim.x) {
    int side = (int)(i / n16);
    const long e = i - side * n16;
    if (a.src_up == nullptr) side = 1;
    const float4* src = reinterpret_cast<const float4*>(side == 0 ? a.src_up : a.src_dn) + e;
    float4* dst = reinterpret_cast<float4*>(side == 0 ? a.dst_up : a.dst_dn) + e;
    *dst = ld_peer(src);
  }
}

template <int V>
__global__ void __launch_bounds__(256)
adam_seam_kernel(CommDev c, float* __restrict__ img, float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
                 float* __restrict__ ema, const AdamScalars* __restrict__ d_adam, int add_seams) {
  typedef typename Vec<V>::T T;
  const AdamScalars ac = *d_adam;
  const int w4 = c.W / V;
  const long per = (long)c.own_rows * w4;
  const T* grad = reinterpret_cast<const T*>(c.mbox[c.rank] + c.off_grad);
  // add_seams = 0 (per-layer-halo mode): the local gradient of the own rows is already complete
  const bool has_up = c.rank > 0 && add_seams, has_dn = c.rank + 1 < c.world && add_seams;
  const T* gup = has_up ? reinterpret_cast<const T*>(c.mbox[c.rank - 1] + c.off_grad) : nullptr;
  const T* gdn = has_dn ? reinterpret_cast<const T*>(c.mbox[c.rank + 1] + c.off_grad) : nullptr;
  T* out_first = reinterpret_cast<T*>(c.mbox[c.rank] + c.off_outbox[0]);
  T* out_last = reinterpret_cast<T*>(c.mbox[c.rank] + c.off_outbox[1]);
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < 3 * per; i += (long)gridDim.x * blockDim.x) {
    const int ch = (int)(i / per);
    const long r4 = i - (long)ch * per;
    const int r = (int)(r4 / w4), x4 = (int)(r4 - (long)r * w4);
    const long idx = ((long)ch * c.h_local + c.own0 + r) * w4 + x4;
    float gg[V], aa[V], mm[V], vv[V], pp[V], ee[V];
    unpack(grad[idx], gg);
    if (has_up && r < COMM_APRON) {   // the upper band's bottom apron starts at its local row own0 + own_rows
      unpack(ld_peer(gup + ((long)ch * c.up_h_local + c.up_apron_row0 + r) * w4 + x4), aa);
#pragma unroll
      for (int k = 0; k < V; ++k) gg[k] += aa[k];
    }
    if (has_dn && r >= c.own_rows - COMM_APRON) {   // the lower band's top apron is its local rows [0, APRON)
      unpack(ld_peer(gdn + ((long)ch * c.dn_h_local + (r - (c.own_rows - COMM_APRON))) * w4 + x4), aa);
#pragma unroll
      for (int k = 0; k < V; ++k) gg[k] += aa[k];
    }
    unpack(reinterpret_cast<T*>(exp_avg)[idx], mm);
    unpack(reinterpret_cast<T*>(exp_avg_sq)[idx], vv);
    unpack(reinterpret_cast<T*>(img)[idx], pp);
    unpack(reinterpret_cast<T*>(ema)[idx], ee);
#pragma unroll
    for (int k = 0; k < V; ++k) {
      mm[k] = mm[k] + (gg[k] - mm[k]) * ac.one_minus_b1;
      vv[k] = vv[k] * ac.b2 + ac.one_minus_b2 * gg[k] * gg[k];
      const float denom = sqrtf(vv[k]) * ac.inv_sqrt_bc2 + ac.eps;
      pp[k] = fminf(fmaxf(pp[k] - ac.step_size * (mm[k] / denom), 0.f), 1.f);
      ee[k] = ee[k] * ac.ema_decay + ac.one_minus_decay * pp[k];
    }
    T pn;
    pack(pn, pp);
    pack(reinterpret_cast<T*>(exp_avg)[idx], mm);
    pack(reinterpret_cast<T*>(exp_avg_sq)[idx], vv);
    reinterpret_cast<T*>(img)[idx] = pn;
    pack(reinterpret_cast<T*>(ema)[idx], ee);
    if (r < COMM_APRON) out_first[((long)ch * COMM_APRON + r) * w4 + x4] = pn;
    if (r >= c.own_rows - COMM_APRON)
      out_last[((long)ch * COMM_APRON + (r - (c.own_rows - COMM_APRON))) * w4 + x4] = pn;
  }
}

// banded L-BFGS: g[3][own_rows][W] (compact) = the own rows of the local gradient (+ the neighbours' apron rows), summed
// in the order of adam_seam_kernel: own, upper, lower
template <int V>
__global__ void __launch_bounds__(256) lbfgs_seam_gather_kernel(CommDev c, float* __restrict__ g, int add_seams) {
  typedef typename Vec<V>::T T;
  const int w4 = c.W / V;
  const long per = (long)c.own_rows * w4;
  const T* grad = reinterpret_cast<const T*>(c.mbox[c.rank] + c.off_grad);
  const bool has_up = c.rank > 0 && add_seams, has_dn = c.rank + 1 < c.world && add_seams;
  const T* gup = has_up ? reinterpret_cast<const T*>(c.mbox[c.rank - 1] + c.off_grad) : nullptr;
  const T* gdn = has_dn ? reinterpret_cast<const T*>(c.mbox[c.rank + 1] + c.off_grad) : nullptr;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < 3 * per; i += (long)gridDim.x * blockDim.x) {
    const int ch = (int)(i / per);
    const long r4 = i - (long)ch * per;
    const int r = (int)(r4 / w4), x4 = (int)(r4 - (long)r * w4);
    float gg[V], aa[V];
    unpack(grad[((long)ch * c.h_local + c.own0 + r) * w4 + x4], gg);
    if (has_up && r < COMM_APRON) {
      unpack(ld_peer(gup + ((long)ch * c.up_h_local + c.up_apron_row0 + r) * w4 + x4), aa);
#pragma unroll
      for (int k = 0; k < V; ++k) gg[k] += aa[k];
    }
    if (has_dn && r >= c.own_rows - COMM_APRON) {
      unpack(ld_peer(gdn + ((long)ch * c.dn_h_local + (r - (c.own_rows - COMM_APRON))) * w4 + x4), aa);
#pragma unroll
      for (int k = 0; k < V; ++k) gg[k] += aa[k];
    }
    pack(reinterpret_cast<T*>(g)[i], gg);
  }
}

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

int grid_for(long n) {
  long b = (n + 255) / 256;
  const long cap = 8l * num_sms();
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace

// ------------------------------------------------------------------------------------------------ host side
size_t comm_mailbox_bytes(size_t stats_floats, int max_h_local, int max_W, size_t off[5]) {
  size_t o = 4096;  // flags
  off[0] = o; o = align_up(o + stats_floats * 4, 1024);
  off[1] = o; o = align_up(o + stats_floats * 4, 1024);
  off[2] = o; o = align_up(o + (size_t)3 * max_h_local * max_W * 4, 1024);                 // grad
  off[3] = o; o = align_up(o + (size_t)3 * COMM_APRON * max_W * 4, 1024);                  // outbox 0 (first rows)
  off[4] = o; o = align_up(o + (size_t)3 * COMM_APRON * max_W * 4, 1024);                  // outbox 1 (last rows)
  return o;
}

int comm_preload() {
  cudaFuncAttributes fa;
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, comm_phase_kernel));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, halo_pull_kernel<4>));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, halo_pull_kernel<1>));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, stats_publish_kernel));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, stats_allreduce_kernel));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, adam_seam_kernel<4>));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, adam_seam_kernel<1>));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, halo_rows_kernel));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, lbfgs_seam_gather_kernel<4>));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, lbfgs_seam_gather_kernel<1>));
  return preload_lbfgs_kernels();
}

int launch_comm_phase(const CommDev& c, int phase, cudaStream_t s) {
  comm_phase_kernel<<<1, 32, 0, s>>>(c, phase);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

int launch_halo_pull(const CommDev& c, float* img, cudaStream_t s) {
  if (c.world <= 1) return STB_OK;
  if (c.W % 4 == 0) halo_pull_kernel<4><<<grid_for(6l * COMM_APRON * (c.W / 4)), 256, 0, s>>>(c, img);
  else halo_pull_kernel<1><<<grid_for(6l * COMM_APRON * c.W), 256, 0, s>>>(c, img);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

int launch_stats_allreduce(const CommDev& c, float* stats, size_t n_floats, cudaStream_t s) {
  STB_CHECK(n_floats % 4 == 0, STB_ERR_INVALID, "stats block must be a multiple of 4 floats");
  const long n4 = (long)(n_floats / 4);
  stats_publish_kernel<<<grid_for(n4), 256, 0, s>>>(c, stats, n4);
  STB_TRY(launch_comm_phase(c, 1, s));
  stats_allreduce_kernel<<<grid_for(n4), 256, 0, s>>>(c, stats, n4);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

int launch_halo_rows(const CommDev& c, const HaloRowArgs& a, cudaStream_t s) {
  STB_CHECK(a.row_bytes % 16 == 0, STB_ERR_INVALID, "halo row of %zu bytes", a.row_bytes);   // 0: stamps only
  if (a.src_up == nullptr && a.src_dn == nullptr) return STB_OK;
  long blocks = (long)(a.row_bytes / 16) * 2 / 256 + 1;
  if (blocks > 16) blocks = 16;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)blocks);
  cfg.blockDim = dim3(256);
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = c.pdl ? 1 : 0;
  STB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, halo_rows_kernel, c, a));
  return STB_OK;
}

int launch_adam_seam(const CommDev& c, float* img, float* exp_avg, float* exp_avg_sq, float* ema,
                     const AdamScalars* d_adam, int add_seams, cudaStream_t s) {
  if (c.W % 4 == 0)
    adam_seam_kernel<4><<<grid_for(3l * c.own_rows * (c.W / 4)), 256, 0, s>>>(c, img, exp_avg, exp_avg_sq, ema, d_adam,
                                                                             add_seams);
  else
    adam_seam_kernel<1><<<grid_for(3l * c.own_rows * c.W), 256, 0, s>>>(c, img, exp_avg, exp_avg_sq, ema, d_adam,
                                                                        add_seams);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

int launch_lbfgs_seam_gather(const CommDev& c, float* g, int add_seams, cudaStream_t s) {
  if (c.W % 4 == 0)
    lbfgs_seam_gather_kernel<4><<<grid_for(3l * c.own_rows * (c.W / 4)), 256, 0, s>>>(c, g, add_seams);
  else
    lbfgs_seam_gather_kernel<1><<<grid_for(3l * c.own_rows * c.W), 256, 0, s>>>(c, g, add_seams);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

}  // namespace stb
