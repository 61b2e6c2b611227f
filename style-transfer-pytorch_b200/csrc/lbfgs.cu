// L-BFGS step on the device: torch.optim.LBFGS.step (torch/optim/lbfgs.py, lr = 1, max_iter = 1, history_size =
// STB_LBFGS_HISTORY, tolerance_grad = 1e-7, tolerance_change = 1e-9, no line search; ST:464-465) followed by the EMA of
// the iterate (ST:250-253).  There is no clamp on this path (ST:482-485).
//
// The whole optimiser state lives in one caller-owned device block (a torch tensor):
//   header | fp64 partial sums | g | g_prev | d | S[11] | Y[11]
// S / Y form a ring of STB_LBFGS_HISTORY + 1 slots: pass 0 writes the candidate pair (y, s) into the spare slot, so a
// pair that the y.s test rejects never overwrites a live one.
//
// The launch sequence is fixed (it is captured into the iteration's CUDA graph); every branch of torch's step is a
// flag in the header that each kernel reads:
//   pass 0          max|g|, sum|g|, y.s, y.y; y = g - g_prev and s = d * t into the spare slot
//   decide          (one block) opt_cond, first iteration, push/reject the pair, ro, H_diag, t
//   21 rounds       the two-loop recursion, one pass over memory per dependent dot product.  The active part of the
//                   2 * count + 1 operations runs in the LAST rounds, earlier rounds return at once, so the final pass
//                   always finds g.d in the same partial buffer.
//   final           g.d test, x += t * d, EMA, g_prev = g
// The banded step of a tiled iteration (launch_lbfgs_step_banded) runs the same kernels on a rank's own rows, with a
// one-block cross-rank reduction (lbfgs_xreduce_kernel) after pass 0 and after every round: the consumers then read one
// partial, the global value, which every rank summed in rank order and therefore holds bit for bit.
// Dot products are reduced deterministically: fixed grid for a given n, one fp64 partial per block, and every block
// of the consuming kernel sums the partials in the same fixed order (graph replay == eager, bit for bit).  Scalars
// are rounded to fp32 where torch holds fp32 tensors (ys, ro, H_diag, al, be, t, gtd and the comparisons).
#include <type_traits>

#include "comm.cuh"
#include "kernels.h"

namespace stb {
namespace {

constexpr int LB_HIST = STB_LBFGS_HISTORY;
constexpr int LB_SLOTS = LB_HIST + 1;
constexpr int LB_ROUNDS = 2 * LB_HIST + 1;
constexpr int LB_THREADS = 256;
constexpr int LB_MAX_BLOCKS = 512;
constexpr size_t LB_HEADER_BYTES = 4096;
constexpr size_t LB_PART_BYTES = (4 + 2) * LB_MAX_BLOCKS * sizeof(double);

struct LbHeader {
  int n_iter;     // torch's state["n_iter"]
  int count;      // pairs held (<= LB_HIST)
  int head;       // ring slot of the oldest pair
  int skip;       // this step hit opt_cond (max|g| <= tolerance_grad): nothing but the EMA changes
  int took_step;  // the last non-skipped step moved x (g.d <= -tolerance_change)
  int pad[3];
  float t;        // step length of the current direction d
  float H_diag;
  float gtd;
  float pad2;
  float ro[LB_SLOTS];  // per ring slot
  float al[LB_SLOTS];
};
static_assert(sizeof(LbHeader) <= LB_HEADER_BYTES, "header");

struct LbState {  // the caller's block, carved up (passed by value to the kernels)
  LbHeader* hdr;
  double* part0;  // [4][LB_MAX_BLOCKS]: max|g|, sum|g|, y.s, y.y of pass 0
  double* part;   // [2][LB_MAX_BLOCKS]: ping-pong partials of the rounds (round r writes buffer r & 1)
  float *g, *g_prev, *d, *S, *Y;
  long n;
  long stride;    // floats between two vectors (S and Y hold LB_SLOTS vectors each)
};

inline long vec_stride(long n) { return (n + 63) / 64 * 64; }   // 256-byte aligned vectors

LbState carve(void* state, long n) {
  LbState st;
  uint8_t* p = static_cast<uint8_t*>(state);
  st.hdr = reinterpret_cast<LbHeader*>(p);
  st.part0 = reinterpret_cast<double*>(p + LB_HEADER_BYTES);
  st.part = st.part0 + 4 * LB_MAX_BLOCKS;
  st.n = n;
  st.stride = vec_stride(n);
  float* v = reinterpret_cast<float*>(p + LB_HEADER_BYTES + LB_PART_BYTES);
  st.g = v;
  st.g_prev = v + st.stride;
  st.d = v + 2 * st.stride;
  st.S = v + 3 * st.stride;
  st.Y = st.S + LB_SLOTS * st.stride;
  return st;
}

int lb_blocks(long n) {
  const long b = (n + 4 * LB_THREADS - 1) / (4 * LB_THREADS);
  return (int)(b < 1 ? 1 : (b > LB_MAX_BLOCKS ? LB_MAX_BLOCKS : b));
}

// max that propagates NaN like torch's abs().max(): a NaN gradient must fail opt_cond (NaN <= 1e-7 is false) and keep
// stepping as torch does, not reduce to 0 and freeze the iterate (fmax drops NaN)
__device__ __forceinline__ double nan_max(double a, double b) { return (b > a || b != b) ? b : a; }

// ---- deterministic block reductions in fp64 (fixed shuffle tree, fixed warp order); the result is broadcast
template <bool kMax>
__device__ __forceinline__ double block_reduce(double v, double* sm) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double w = __shfl_xor_sync(0xffffffffu, v, o);
    v = kMax ? nan_max(v, w) : v + w;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();  // sm may still be read by a previous reduction
  if (lane == 0) sm[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = lane < (int)(blockDim.x >> 5) ? sm[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double w = __shfl_xor_sync(0xffffffffu, v, o);
      v = kMax ? nan_max(v, w) : v + w;
    }
    if (lane == 0) sm[32] = v;
  }
  __syncthreads();
  return sm[32];
}

// sum of the nb partials of the previous kernel, in a fixed order (every block computes the same value)
template <bool kMax = false>
__device__ __forceinline__ double reduce_partials(const double* p, int nb, double* sm) {
  double v = 0.0;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) v = kMax ? nan_max(v, p[i]) : v + p[i];
  return block_reduce<kMax>(v, sm);
}

// L consecutive floats at j (L = 4: one 16-byte access; the vectors and the caller's tensors are 16-byte aligned)
template <int L> struct Vec { float v[L]; };
template <int L>
__device__ __forceinline__ Vec<L> ld(const float* p, long j) {
  Vec<L> r;
  if constexpr (L == 4) {
    const float4 t = *reinterpret_cast<const float4*>(p + j);
    r.v[0] = t.x; r.v[1] = t.y; r.v[2] = t.z; r.v[3] = t.w;
  } else {
    r.v[0] = p[j];
  }
  return r;
}
template <int L>
__device__ __forceinline__ void st(float* p, long j, const Vec<L>& r) {
  if constexpr (L == 4) *reinterpret_cast<float4*>(p + j) = make_float4(r.v[0], r.v[1], r.v[2], r.v[3]);
  else p[j] = r.v[0];
}

// calls body(Vec-width constant, j) over [0, n): 4-wide chunks in a grid-stride loop, then the < 4 scalar tail
template <typename Body>
__device__ __forceinline__ void for_each(long n, Body&& body) {
  const long n4 = n >> 2;
  const long stride = (long)gridDim.x * blockDim.x;
  const long tid = (long)blockIdx.x * blockDim.x + threadIdx.x;
  for (long c = tid; c < n4; c += stride) body(std::integral_constant<int, 4>(), 4 * c);
  for (long j = 4 * n4 + tid; j < n; j += stride) body(std::integral_constant<int, 1>(), j);
}

__device__ __forceinline__ int ring_slot(const LbHeader& h, int i) { return (h.head + i) % LB_SLOTS; }

// pass 0: one read of g, g_prev, d.  y and s of the candidate pair go to the spare slot (not written before the first
// iteration, where torch has no previous direction).
__global__ void __launch_bounds__(LB_THREADS) lbfgs_pass0_kernel(LbState s) {
  __shared__ double sm[33];
  const LbHeader h = *s.hdr;
  const bool pair = h.n_iter > 0;
  const float t = h.t;
  const long spare = (long)((h.head + h.count) % LB_SLOTS) * s.stride;
  float* Ys = s.Y + spare;
  float* Ss = s.S + spare;
  double amax = 0.0, asum = 0.0, ys = 0.0, yy = 0.0;
  for_each(s.n, [&](auto lanes, long j) {
    constexpr int L = decltype(lanes)::value;
    const Vec<L> g = ld<L>(s.g, j);
#pragma unroll
    for (int k = 0; k < L; ++k) {
      amax = nan_max(amax, (double)fabsf(g.v[k]));
      asum += (double)fabsf(g.v[k]);
    }
    if (pair) {
      const Vec<L> gp = ld<L>(s.g_prev, j), d = ld<L>(s.d, j);
      Vec<L> y, sv;
#pragma unroll
      for (int k = 0; k < L; ++k) {
        y.v[k] = g.v[k] - gp.v[k];
        sv.v[k] = d.v[k] * t;
        ys += (double)y.v[k] * (double)sv.v[k];
        yy += (double)y.v[k] * (double)y.v[k];
      }
      st<L>(Ys, j, y);
      st<L>(Ss, j, sv);
    }
  });
  const int b = blockIdx.x;
  amax = block_reduce<true>(amax, sm);
  asum = block_reduce<false>(asum, sm);
  ys = block_reduce<false>(ys, sm);
  yy = block_reduce<false>(yy, sm);
  if (threadIdx.x == 0) {
    s.part0[0 * LB_MAX_BLOCKS + b] = amax;
    s.part0[1 * LB_MAX_BLOCKS + b] = asum;
    s.part0[2 * LB_MAX_BLOCKS + b] = ys;
    s.part0[3 * LB_MAX_BLOCKS + b] = yy;
  }
}

// decide: torch's scalar control flow for this step (one block)
__global__ void __launch_bounds__(LB_THREADS) lbfgs_decide_kernel(LbState s, int nb) {
  __shared__ double sm[33];
  const double amax = reduce_partials<true>(s.part0 + 0 * LB_MAX_BLOCKS, nb, sm);
  const double asum = reduce_partials(s.part0 + 1 * LB_MAX_BLOCKS, nb, sm);
  const double ys = reduce_partials(s.part0 + 2 * LB_MAX_BLOCKS, nb, sm);
  const double yy = reduce_partials(s.part0 + 3 * LB_MAX_BLOCKS, nb, sm);
  if (threadIdx.x != 0) return;
  LbHeader& h = *s.hdr;
  if ((float)amax <= 1e-7f) {  // opt_cond: return before n_iter advances, the state stays as it is
    h.skip = 1;
    return;
  }
  h.skip = 0;
  h.n_iter += 1;
  if (h.n_iter == 1) {
    h.count = 0;
    h.head = 0;
    h.H_diag = 1.f;
    const float inv = 1.f / (float)asum;   // t = min(1, 1 / sum|g|) * lr
    h.t = inv < 1.f ? inv : 1.f;
  } else {
    const float ysf = (float)ys;
    if (ysf > 1e-10f) {  // accept the pair in the spare slot; drop the oldest one when the history is full
      const int spare = (h.head + h.count) % LB_SLOTS;
      h.ro[spare] = 1.f / ysf;
      h.H_diag = ysf / (float)yy;
      if (h.count == LB_HIST) h.head = (h.head + 1) % LB_SLOTS;
      else h.count += 1;
    }
    h.t = 1.f;
  }
}

// round r of the two-loop recursion (the previous round left np partials).  With c pairs the active operations o = 0 .. 2c run in rounds
// r = LB_ROUNDS - (2c + 1) + o:
//   o = 0        v = -g                          (torch: q = -g)
//   1 <= o <= c  v -= al_i y_i, i = c - o        (al_i = (s_i . q) ro_i, the dot of the previous round)
//   o = c        v *= H_diag                     (r = q H_diag)
//   o > c        v += (al_i - be_i) s_i, i = o-c-1 (be_i = (y_i . r) ro_i)
// v is stored into d (q and r share it, as in torch) and the dot the next operation needs is accumulated:
// s_{c-1-o} . v while o < c, y_{o-c} . v while o < 2c, and g . d (gtd) at o = 2c.
__global__ void __launch_bounds__(LB_THREADS) lbfgs_round_kernel(LbState s, int round, int np) {
  __shared__ double sm[33];
  const LbHeader& h = *s.hdr;
  if (h.skip) return;
  const int c = h.count;
  const int o = round - (LB_ROUNDS - (2 * c + 1));
  if (o < 0) return;
  float coef = 0.f;
  const float* upd = nullptr;
  if (o >= 1) {
    const float dot = (float)reduce_partials(s.part + ((round - 1) & 1) * LB_MAX_BLOCKS, np, sm);
    if (o <= c) {
      const int slot = ring_slot(h, c - o);
      const float al = dot * h.ro[slot];
      if (blockIdx.x == 0 && threadIdx.x == 0) s.hdr->al[slot] = al;
      coef = -al;
      upd = s.Y + (long)slot * s.stride;
    } else {
      const int slot = ring_slot(h, o - c - 1);
      const float be = dot * h.ro[slot];
      coef = h.al[slot] - be;
      upd = s.S + (long)slot * s.stride;
    }
  }
  const float hd = o == c ? h.H_diag : 1.f;
  const bool scale = o == c;
  const float* src = o == 0 ? s.g : s.d;
  const float sign = o == 0 ? -1.f : 1.f;
  const float* dv = o < c ? s.S + (long)ring_slot(h, c - 1 - o) * s.stride
                          : (o < 2 * c ? s.Y + (long)ring_slot(h, o - c) * s.stride : s.g);
  double acc = 0.0;
  for_each(s.n, [&](auto lanes, long j) {
    constexpr int L = decltype(lanes)::value;
    Vec<L> v = ld<L>(src, j);
    const Vec<L> w = ld<L>(dv, j);
    Vec<L> u;
    if (upd) u = ld<L>(upd, j);
#pragma unroll
    for (int k = 0; k < L; ++k) {
      float x = sign * v.v[k];
      if (upd) x = x + coef * u.v[k];
      if (scale) x = x * hd;
      v.v[k] = x;
      acc += (double)x * (double)w.v[k];
    }
    st<L>(s.d, j, v);
  });
  acc = block_reduce<false>(acc, sm);
  if (threadIdx.x == 0) s.part[(round & 1) * LB_MAX_BLOCKS + blockIdx.x] = acc;
}

// g.d test of the final pass over the np partials of the last round: whether x moves (false on an opt_cond step)
__device__ __forceinline__ bool final_take(const LbState& s, int np, double* sm) {
  if (s.hdr->skip) return false;
  const float gtd = (float)reduce_partials(s.part + ((LB_ROUNDS - 1) & 1) * LB_MAX_BLOCKS, np, sm);
  const bool take = !(gtd > -1e-9f);
  if (blockIdx.x == 0 && threadIdx.x == 0) { s.hdr->gtd = gtd; s.hdr->took_step = take; }
  return take;
}

// the per-element work of the final pass, shared by the untiled and the banded kernel: x += t d (no clamp) when the
// step is taken, EMA of x, g_prev = g.  x / ema at jx, the state vectors at j; xv receives the new x.
template <int L>
__device__ __forceinline__ void final_elems(const LbState& s, bool take, bool skip, float t, float decay, float* x,
                                            float* ema, long jx, long j, Vec<L>& xv) {
  const float om = 1.f - decay;
  xv = ld<L>(x, jx);
  if (take) {
    const Vec<L> d = ld<L>(s.d, j);
#pragma unroll
    for (int k = 0; k < L; ++k) xv.v[k] = xv.v[k] + t * d.v[k];
    st<L>(x, jx, xv);
  }
  Vec<L> e = ld<L>(ema, jx);
#pragma unroll
  for (int k = 0; k < L; ++k) e.v[k] = e.v[k] * decay + om * xv.v[k];
  st<L>(ema, jx, e);
  if (!skip) st<L>(s.g_prev, j, ld<L>(s.g, j));
}

// final pass: g.d test, x += t d (no clamp), EMA of x, g_prev = g
__global__ void __launch_bounds__(LB_THREADS) lbfgs_final_kernel(LbState s, float* __restrict__ x,
                                                                 float* __restrict__ ema, float decay, int np) {
  __shared__ double sm[33];
  const bool skip = s.hdr->skip != 0;
  const bool take = final_take(s, np, sm);
  const float t = s.hdr->t;
  for_each(s.n, [&](auto lanes, long j) {
    constexpr int L = decltype(lanes)::value;
    Vec<L> xv;
    final_elems<L>(s, take, skip, t, decay, x, ema, j, j, xv);
  });
}

// ---- banded step (tiled iteration): the state vectors are compact [3][own_rows][W]; x and ema are the local
// [3][h_local][W] image.  V = 4 when W % 4 == 0 (rows are 16-byte aligned), else 1 (odd pyramid widths such as 181).

// Cross-rank reduction, one block.  nvals (<= 4) values; value k has nb block partials at part + k * LB_MAX_BLOCKS
// (value 0 is a NaN-propagating max when max0).  This rank's sums, taken in reduce_partials' order, go to its mailbox
// slot [iteration parity][seq] and are published by the stamp iter * 32 + seq (system-scope release).  Lane r of warp 0
// waits for rank r's stamp (acquire, wait_stamp's timeout) and loads rank r's values; thread 0 combines the ranks in
// rank order -- the same order on every rank, so every rank gets the same bits -- and stores the global values at
// part[k * LB_MAX_BLOCKS], where the next kernel reads them as its only partial.  Peer waits happen here and never in
// the full-grid kernels: ranks that share a GPU must not hold its SMs while they wait.
__global__ void __launch_bounds__(LB_THREADS) lbfgs_xreduce_kernel(CommDev c, double* part, int nvals, int nb,
                                                                   int max0, int seq) {
  __shared__ double sm[33];
  __shared__ double vals[COMM_MAX_RANKS][4];
  double mine[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (k < nvals)
      mine[k] = k == 0 && max0 ? reduce_partials<true>(part + k * LB_MAX_BLOCKS, nb, sm)
                               : reduce_partials(part + k * LB_MAX_BLOCKS, nb, sm);
  unsigned long long* own = reinterpret_cast<unsigned long long*>(c.mbox[c.rank]);
  const unsigned long long it = own[COMM_ITER];
  const int slot = COMM_XVAL + ((int)(it & 1) * LBFGS_XREDUCES + seq) * 4;
  const unsigned long long want = it * 32ull + (unsigned long long)seq;
  if (threadIdx.x == 0) {
    double* mv = reinterpret_cast<double*>(own + slot);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (k < nvals) { mv[k] = mine[k]; vals[c.rank][k] = mine[k]; }
    __threadfence_system();
    st_release_sys(own + COMM_FLAG_XRED, want);
  }
  const int lane = threadIdx.x;
  if (lane < c.world && lane != c.rank) {
    const unsigned long long* peer = reinterpret_cast<const unsigned long long*>(c.mbox[lane]);
    wait_stamp(peer + COMM_FLAG_XRED, want, own + COMM_ERR, c.timeout_ns);
    const double* pv = reinterpret_cast<const double*>(peer + slot);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (k < nvals) vals[lane][k] = ld_peer(pv + k);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (k < nvals) {
        double v = vals[0][k];
        for (int r = 1; r < c.world; ++r) v = k == 0 && max0 ? nan_max(v, vals[r][k]) : v + vals[r][k];
        part[k * LB_MAX_BLOCKS] = v;
      }
  }
}
static_assert(COMM_XVAL + 2 * LBFGS_XREDUCES * 4 <= 4096 / 8, "cross-rank values must fit the mailbox head");
static_assert(LBFGS_XREDUCES < 32, "stamp = iteration * 32 + seq");

// final pass of the banded step on the own rows of the local image; the first / last COMM_APRON rows also go to the
// outboxes (the neighbours' next halo), as adam_seam_kernel does
template <int V>
__global__ void __launch_bounds__(LB_THREADS) lbfgs_final_banded_kernel(LbState s, CommDev c, float* __restrict__ x,
                                                                        float* __restrict__ ema, float decay) {
  __shared__ double sm[33];
  const bool skip = s.hdr->skip != 0;
  const bool take = final_take(s, 1, sm);
  const float t = s.hdr->t;
  const int wv = c.W / V;
  const int per = c.own_rows * wv;   // 3 * per < 2^31 (launch_lbfgs_step_banded)
  float* out_first = reinterpret_cast<float*>(c.mbox[c.rank] + c.off_outbox[0]);
  float* out_last = reinterpret_cast<float*>(c.mbox[c.rank] + c.off_outbox[1]);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 3 * per; i += gridDim.x * blockDim.x) {
    const int ch = i / per;
    const int r4 = i - ch * per;
    const int r = r4 / wv;
    const long xo = (long)(r4 - r * wv) * V;
    Vec<V> xv;
    final_elems<V>(s, take, skip, t, decay, x, ema, ((long)ch * c.h_local + c.own0 + r) * c.W + xo, (long)i * V, xv);
    if (r < COMM_APRON) st<V>(out_first, ((long)ch * COMM_APRON + r) * c.W + xo, xv);
    if (r >= c.own_rows - COMM_APRON)
      st<V>(out_last, ((long)ch * COMM_APRON + (r - (c.own_rows - COMM_APRON))) * c.W + xo, xv);
  }
}

}  // namespace

size_t lbfgs_state_bytes(long n) {
  return LB_HEADER_BYTES + LB_PART_BYTES + (size_t)(3 + 2 * LB_SLOTS) * (size_t)vec_stride(n) * sizeof(float);
}

float* lbfgs_grad_buffer(void* state, long n) { return carve(state, n).g; }

int launch_lbfgs_reset(void* state, cudaStream_t s) {
  STB_CUDA_CHECK(cudaMemsetAsync(state, 0, LB_HEADER_BYTES, s));
  return STB_OK;
}

int launch_lbfgs_step(void* state, long n, float* x, float* ema, float ema_decay, cudaStream_t s) {
  const LbState st = carve(state, n);
  const int nb = lb_blocks(n);
  lbfgs_pass0_kernel<<<nb, LB_THREADS, 0, s>>>(st);
  lbfgs_decide_kernel<<<1, LB_THREADS, 0, s>>>(st, nb);
  for (int r = 0; r < LB_ROUNDS; ++r) lbfgs_round_kernel<<<nb, LB_THREADS, 0, s>>>(st, r, nb);
  lbfgs_final_kernel<<<nb, LB_THREADS, 0, s>>>(st, x, ema, ema_decay, nb);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

int launch_lbfgs_step_banded(void* state, const CommDev& c, float* x, float* ema, float ema_decay, int add_seams,
                             cudaStream_t s) {
  const long n = 3l * c.own_rows * c.W;
  STB_CHECK(n < (1l << 31), STB_ERR_INVALID, "band of %d x %d pixels is too large", c.own_rows, c.W);
  const LbState st = carve(state, n);
  const int nb = lb_blocks(n);
  STB_TRY(launch_lbfgs_seam_gather(c, st.g, add_seams, s));
  lbfgs_pass0_kernel<<<nb, LB_THREADS, 0, s>>>(st);
  lbfgs_xreduce_kernel<<<1, LB_THREADS, 0, s>>>(c, st.part0, 4, nb, 1, 0);
  lbfgs_decide_kernel<<<1, LB_THREADS, 0, s>>>(st, 1);
  for (int r = 0; r < LB_ROUNDS; ++r) {
    lbfgs_round_kernel<<<nb, LB_THREADS, 0, s>>>(st, r, 1);
    lbfgs_xreduce_kernel<<<1, LB_THREADS, 0, s>>>(c, st.part + (r & 1) * LB_MAX_BLOCKS, 1, nb, 0, r + 1);
  }
  if (c.W % 4 == 0) lbfgs_final_banded_kernel<4><<<nb, LB_THREADS, 0, s>>>(st, c, x, ema, ema_decay);
  else lbfgs_final_banded_kernel<1><<<nb, LB_THREADS, 0, s>>>(st, c, x, ema, ema_decay);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

int preload_lbfgs_kernels() {
  cudaFuncAttributes fa;
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, lbfgs_pass0_kernel));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, lbfgs_decide_kernel));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, lbfgs_round_kernel));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, lbfgs_xreduce_kernel));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, lbfgs_final_banded_kernel<4>));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, lbfgs_final_banded_kernel<1>));
  return STB_OK;
}

int lbfgs_read_info(const void* state, int* pairs, float* t, cudaStream_t s) {
  LbHeader h;
  STB_CUDA_CHECK(cudaMemcpyAsync(&h, state, sizeof(h), cudaMemcpyDeviceToHost, s));
  STB_CUDA_CHECK(cudaStreamSynchronize(s));
  if (pairs) *pairs = h.count;
  if (t) *t = h.t;
  return STB_OK;
}

}  // namespace stb
