// Wasserstein-2 style loss on the five tap covariances, forward and backward, at fp32 accuracy on wgmma:
//   StyleLossW2.__init__/forward      style_transfer/style_transfer.py:149-181 of the reference  (ST)
//   sqrtm_ns (12 Newton-Schulz its)   style_transfer/sqrtm.py:9-25 of the reference              (SQ)
//   _MatrixSquareRootNSLyap.backward  SQ:36-47 (iterative Lyapunov solve, 12 its)
// plus the closed-form backward of ST:163-181 down to  G = d loss / d srm  and  d loss / d mean.
//
// The loss is a cancellation (tr(St + S - 2 sqrt(.)), SURVEY.md section 7.2): plain TF32/bf16 operands are not
// accurate enough.  Every C x C matrix of the chain therefore lives as TWO fp32 planes, x = hi + lo, where hi has its
// low 13 mantissa bits cleared (exactly representable in TF32) and lo = x - hi; a product is evaluated as
//     a*b ~= lo_a*hi_b + hi_a*lo_b + hi_a*hi_b        (3 x wgmma tf32, fp32 accumulate in registers),
// the dropped lo*lo term being 2^-22 relative.  The split of a result is done by the producing GEMM's epilogue, so a
// GEMM only ever streams ready-made planes through TMA.
//
// All five layers advance in lock-step: one "round" = one grouped launch whose CTAs are 128 x 64 output tiles of
// every layer's GEMM (75 or 150 tiles, largest matrices first).  Both wgmma operands are K-major SW128 tiles:
// A[m][k] from the row-major planes of A, B[n][k] from the planes of B^T -- every matrix that is later used as a
// right factor is therefore written TWICE by its producer: the planes of D (TMA store of the staged tile) and the
// planes of D^T (scalar stores).
//
// The products are formed in exactly the reference's order, Y <- Y T, Z <- T Z, and NOTHING is symmetrised, although
// every matrix here is symmetric in exact arithmetic.  Two shortcuts were tried and measured to break parity on real
// (ill-conditioned, eps = 1e-4) covariances, where the coupled Newton-Schulz iteration amplifies a perturbation of
// the small-eigenvalue directions by 1.5^12:
//   * reading a computed product as its own transpose turns the error recursion E' = E/2 into
//     E' = E - A^(1/2) E A^(-1/2) / 2: NaN at 2048^2;
//   * computing only the upper triangle and mirroring it bit-for-bit (38 % fewer tiles) is stable but biases the
//     style terms by -1e-3 ... -3e-3 at 512^2 and above (the CPU emulation of that schedule in fp32 shows the same),
//     i.e. above the 1e-3 loss bar.  The full products stay within 3e-4 of the fp64 chain.
// Tensor maps are encoded once per workspace binding.
#include <cuda_fp16.h>

#include <algorithm>
#include <cstdlib>
#include <map>
#include <set>
#include <utility>
#include <vector>

#include "kernels.h"
#include "ptx.cuh"

namespace stb {

namespace {

constexpr int TM = 128, TN = 64, TKF = 32;      // tile rows / cols, k floats per stage (128 B swizzle row)
constexpr int T_STAGES = 4;
constexpr int A_PLANE_BYTES = TM * 128;          // 16 KiB
constexpr int B_PLANE_BYTES = TN * 128;          // 8 KiB
constexpr int T_STAGE_BYTES = 2 * A_PLANE_BYTES + 2 * B_PLANE_BYTES;  // A_hi, A_lo, B_hi, B_lo = 48 KiB
constexpr int T_OFF_BAR = T_STAGES * T_STAGE_BYTES;
constexpr int T_OFF_RED = T_OFF_BAR + 2 * T_STAGES * 8;
constexpr int T_SMEM_BYTES = T_OFF_RED + 64 + 1024;
constexpr int T_EPI_THREADS = 256;                 // two consumer warpgroups: rows 0..63 and 64..127 of the tile
constexpr int T_THREADS = T_EPI_THREADS + 32;      // + the TMA producer warp
constexpr int NRED = 128;  // max reduction partials per layer
constexpr int NB = 128;    // helper-kernel CTAs per layer: they are latency-bound element-wise passes (32 CTAs: 48 us)
static_assert(NB <= NRED, "the covariance kernel writes one partial per CTA");

// x = hi + lo with both parts rounded to nearest TF32 (the tensor core would otherwise truncate them: a biased
// error that the loss' cancellation amplifies); x - hi is exact in fp32.
__device__ __forceinline__ float rna_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
__device__ __forceinline__ void split_tf32(float v, float& h, float& l) {
  h = rna_tf32(v);
  l = rna_tf32(v - h);
}
__device__ __forceinline__ void store_split(float* m, size_t nn, size_t e, float v) {
  float h, l;
  split_tf32(v, h, l);
  m[e] = h;
  m[nn + e] = l;
}
__device__ __forceinline__ float load2(const float* m, size_t nn, size_t e) { return m[e] + m[nn + e]; }

// fp16 plane pairs (the Newton-Schulz / Lyapunov iterates): x = hi + lo' * 2^-11 with hi = fp16(x) and
// lo' = fp16((x - hi) * 2^11) -- 22 significant bits like the TF32 pair, in HALF the bytes, and kind::f16 MMAs.  The
// residual is stored scaled so that it lives in the same exponent range as x (no fp16 underflow); the products
// lo'_a hi_b + hi_a lo'_b go to their own accumulator, which the epilogue scales by 2^-11.  Every matrix kept this way
// is normalised (|entries| <~ 1e2), far inside the fp16 range; the un-normalised ones (cov, P, X, M, U, Gc and the
// final q) stay TF32 pairs.
constexpr float H_LO_SCALE = 2048.f, H_LO_INV = 1.f / 2048.f;
__device__ __forceinline__ void split_half(float v, __half& h, __half& l) {
  h = __float2half_rn(v);
  l = __float2half_rn((v - __half2float(h)) * H_LO_SCALE);
}
__device__ __forceinline__ void store_split_h(float* m, size_t nn, size_t e, float v) {
  __half* mh = reinterpret_cast<__half*>(m);
  __half h, l;
  split_half(v, h, l);
  mh[e] = h;
  mh[nn + e] = l;
}
__device__ __forceinline__ float load2_h(const float* m, size_t nn, size_t e) {
  const __half* mh = reinterpret_cast<const __half*>(m);
  return __half2float(mh[e]) + __half2float(mh[nn + e]) * H_LO_INV;
}

// D = alpha * A * B + gamma * I on one 128 x 64 tile.  A matrix is 4 planes of n*n floats: hi, lo, hi^T, lo^T.
// smem per stage: A planes [128 rows][32 k] and B^T planes [64 rows (n)][32 k], all K-major SW128.
constexpr int STG_OFF = 0;                          // 4 store tiles (2 column halves x hi/lo) of 16 KiB, SW128, in
static_assert(4 * A_PLANE_BYTES <= T_STAGES * T_STAGE_BYTES, "epilogue smem");  // the drained pipeline buffers

__device__ __forceinline__ unsigned ld_acquire_gpu_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// The whole chain of rounds [r0, r1) in ONE persistent, cooperatively launched kernel: one CTA per SM, tile t of a
// round goes to CTA t % gridDim.x, a grid-wide barrier separates two rounds.  Replaces 24-26 dependent launches per
// phase: barrier init and the launch / drain latency of a grid are paid once, a round boundary costs one atomic + one
// acquire spin instead of a launch gap.  The arithmetic of a tile is unchanged.
//
// Roles: warp 8 TMA producer (four planes per stage), warps 0-7 two consumer warpgroups (tile rows 64 g .. 64 g + 63).
// A consumer issues per stage 4 k-steps x 3 split products, one k-step per MMA group: the cross terms lo*hi and hi*lo
// into one accumulator over the whole K range, the hi*hi product into a fresh accumulator that is added into the
// running sum in round-to-nearest fp32 once the group completes.  The tensor core
// aligns every product to the accumulator and truncates, so a chain of hi*hi products loses ~2^-25 per step of the
// sum, systematically, which the Newton-Schulz iteration turns into a bias of the style terms on the ill-conditioned
// covariances (measured: 1.5e-3 on the 64-channel term with chains of four).
__global__ void __launch_bounds__(T_THREADS, 1)
w2_chain_kernel(const W2Round* __restrict__ rounds, int r0, int r1, unsigned* __restrict__ grid_counter,
                unsigned long long* __restrict__ trace) {
  // trace (STB_W2_TRACE=1, diagnostics): CTA 0 stamps %globaltimer at 8 points of every round --
  // 0 round start, 1 first stage landed, 2 accumulators complete, 3 tile staged + TMA stores issued, 4 stores complete,
  // 5 arrived at the grid barrier, 6 barrier passed
  auto stamp = [&](int round, int k) {
    if (trace != nullptr && blockIdx.x == 0) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
      trace[round * 8 + k] = t;
    }
  };
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + T_OFF_BAR);
  uint64_t* empty = full + T_STAGES;
  float* s_red = reinterpret_cast<float*>(smem + T_OFF_RED);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (warp == 8 && lane == 0) {
    // empty: one arrival per consumer warp once its wgmma reads of the stage are complete
    for (int i = 0; i < T_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  // pipeline ring state, persistent across tiles and rounds (the producer and the consumers advance identically)
  int s = 0;
  uint32_t ph = 0;
  unsigned barriers_done = 0;

  // The tile -> CTA map is static, so everything a CTA needs for its first tile of the NEXT round (problem record,
  // tensor-map descriptors) is fetched BEFORE the grid barrier: after it the producer can issue its TMA loads at once
  // instead of first walking rounds[] -> tiles[] -> probs[] -> descriptor through dependent L2 reads.
  uint32_t pre_t = 0;
  int pre_n_tiles = 0;
  TcProb pre_pr = {};
  auto prefetch_round = [&](int round) {
    const W2Round& nx = rounds[round];
    pre_n_tiles = nx.n_tiles;
    if ((int)blockIdx.x < pre_n_tiles) {
      pre_t = nx.tiles[blockIdx.x];
      pre_pr = nx.probs[pre_t >> 16];
      if (threadIdx.x == 0) {
        tma_prefetch_desc(pre_pr.amap); tma_prefetch_desc(pre_pr.amap + 1);
        tma_prefetch_desc(pre_pr.bmap); tma_prefetch_desc(pre_pr.bmap + 1);
        tma_prefetch_desc(pre_pr.dmap); tma_prefetch_desc(pre_pr.dmap + 1);
      }
    }
  };
  prefetch_round(r0);

  for (int round = r0; round < r1; ++round) {
    const W2Round& rp = rounds[round];
    const int n_tiles = pre_n_tiles;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      const bool first = tile == (int)blockIdx.x;
      const uint32_t t = first ? pre_t : rp.tiles[tile];
      const TcProb pr = first ? pre_pr : rp.probs[t >> 16];
      const int ti = (t >> 8) & 0xFF, tj = t & 0xFF;
      const int n = pr.n;
      const int k_elems = pr.in_half ? 2 * TKF : TKF;          // elements per 128-byte stage row
      const int n_k = n / k_elems;

      if (warp == 8) {
        // ---- TMA producer: four planes per stage
        const bool leader = elect_one();   // every lane walks the ring state, the elected one issues
        if (leader && first) stamp(round, 0);
        for (int k = 0; k < n_k; ++k) {
          if (leader) {
            mbar_wait(&empty[s], ph ^ 1);
            mbar_expect_tx(&full[s], T_STAGE_BYTES);
            uint8_t* st = smem + s * T_STAGE_BYTES;
            tma_load_2d(st, pr.amap, &full[s], k * k_elems, ti * TM);
            tma_load_2d(st + A_PLANE_BYTES, pr.amap + 1, &full[s], k * k_elems, ti * TM);
            tma_load_2d(st + 2 * A_PLANE_BYTES, pr.bmap, &full[s], k * k_elems, tj * TN);  // rows of B^T
            tma_load_2d(st + 2 * A_PLANE_BYTES + B_PLANE_BYTES, pr.bmap + 1, &full[s], k * k_elems, tj * TN);
          }
          if (++s == T_STAGES) { s = 0; ph ^= 1; }
        }
        __syncwarp();
      } else {
        // ---- consumers: MMA (warpgroup g = rows 64 g .. 64 g + 63 of the tile), then the epilogue
        const int g = warp >> 2, wq = warp & 3;
        const bool half_in = pr.in_half != 0;
        float hh[32], cross[32], tot[32];
#pragma unroll
        for (int e = 0; e < 32; ++e) tot[e] = 0.f;
        for (int k = 0; k < n_k; ++k) {
          mbar_wait(&full[s], ph);
          if (threadIdx.x == 0 && first && k == 0) stamp(round, 1);
          const uint32_t base = smem_u32(smem + s * T_STAGE_BYTES);
          const uint64_t a_h = gmma_desc_k(base + g * 64 * 128), a_l = gmma_desc_k(base + A_PLANE_BYTES + g * 64 * 128);
          const uint64_t b_h = gmma_desc_k(base + 2 * A_PLANE_BYTES);
          const uint64_t b_l = gmma_desc_k(base + 2 * A_PLANE_BYTES + B_PLANE_BYTES);
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {  // 8 floats / 16 halfs = 32 bytes per K step -> +2 in the descriptor
            wgmma_fence();
            if (!half_in) {
              wgmma_tf32(cross, a_l + 2 * kk, b_h + 2 * kk, k > 0 || kk > 0);
              wgmma_tf32(hh, a_h + 2 * kk, b_h + 2 * kk, 0);
              wgmma_tf32(cross, a_h + 2 * kk, b_l + 2 * kk, 1);
            } else {
              wgmma_f16<0, 0>(cross, a_l + 2 * kk, b_h + 2 * kk, k > 0 || kk > 0);
              wgmma_f16<0, 0>(hh, a_h + 2 * kk, b_h + 2 * kk, 0);
              wgmma_f16<0, 0>(cross, a_h + 2 * kk, b_l + 2 * kk, 1);
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_acc(hh);
#pragma unroll
            for (int e = 0; e < 32; ++e) tot[e] += hh[e];
          }
          if (lane == 0) mbar_arrive(&empty[s]);
          if (++s == T_STAGES) { s = 0; ph ^= 1; }
        }
        wgmma_fence_acc(cross);
        // every consumer is done reading the pipeline buffers, which the epilogue reuses as staging
        named_bar_sync(2, T_EPI_THREADS);
        const bool issuer = threadIdx.x == 0;   // the one thread that issues the TMA stores / writes the partials
        if (issuer && first) stamp(round, 2);
        const size_t nn = (size_t)n * n;
        uint8_t* stg = smem + STG_OFF;
        const float cross_scale = pr.in_half ? H_LO_INV : 1.f;   // fp16 pairs keep the residual plane times 2^11
        const bool half_out = pr.out_half != 0;
        __half* Dh = reinterpret_cast<__half*>(pr.D);
        const int cq = 2 * (lane & 3);
        float ssq = 0.f, tr = 0.f;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int r = 64 * g + 16 * wq + (lane >> 2) + 8 * hr;   // tile row
          const int gi = ti * TM + r;
          const bool valid = gi < n;
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const int c = 8 * q + cq;                              // tile column (and c + 1)
            float o[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int idx = 4 * q + 2 * hr + e;
              o[e] = (tot[idx] + cross[idx] * cross_scale) * pr.alpha;
              if (gi == tj * TN + c + e) { o[e] += pr.gamma; tr += o[e]; }
              if (valid) ssq = fmaf(o[e], o[e], ssq);
            }
            const int gj = tj * TN + c;
            if (!half_out) {
              // planes of column half h = c / 32: [128 rows][32 floats], 128-byte swizzle as the TMA store expects
              const int h = c >> 5, cc = c & 31;
              uint8_t* row_hi = stg + (h * 2) * A_PLANE_BYTES + r * 128;
              uint8_t* row_lo = row_hi + A_PLANE_BYTES;
              const int off = (((cc >> 2) ^ (r & 7)) << 4) + (cc & 3) * 4;
              float vh[2], vl[2];
              split_tf32(o[0], vh[0], vl[0]);
              split_tf32(o[1], vh[1], vl[1]);
              *reinterpret_cast<float2*>(row_hi + off) = make_float2(vh[0], vh[1]);
              *reinterpret_cast<float2*>(row_lo + off) = make_float2(vl[0], vl[1]);
              if (pr.write_t && valid) {  // D^T planes
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const size_t at = 2 * nn + (size_t)(gj + e) * n + gi;
                  pr.D[at] = vh[e];
                  pr.D[nn + at] = vl[e];
                }
              }
            } else {
              // fp16 pair: one 128 x 64 tile per plane (row = 64 halfs = 128 bytes), hi plane at stg, lo plane after it
              uint8_t* row_hi = stg + r * 128;
              uint8_t* row_lo = row_hi + A_PLANE_BYTES;
              const int off = ((q ^ (r & 7)) << 4) + cq * 2;
              __half hh[2], ll[2];
              split_half(o[0], hh[0], ll[0]);
              split_half(o[1], hh[1], ll[1]);
              *reinterpret_cast<__half2*>(row_hi + off) = __halves2half2(hh[0], hh[1]);
              *reinterpret_cast<__half2*>(row_lo + off) = __halves2half2(ll[0], ll[1]);
              if (pr.write_t && valid) {  // D^T planes
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const size_t at = 2 * nn + (size_t)(gj + e) * n + gi;
                  Dh[at] = hh[e];
                  Dh[nn + at] = ll[e];
                }
              }
            }
          }
        }
        fence_proxy_async_smem();
        // the D^T planes were written through the generic proxy; the next round reads them through TMA (async proxy)
        asm volatile("fence.proxy.async;" ::: "memory");
        named_bar_sync(1, T_EPI_THREADS);
        if (issuer) {
          const CUtensorMap* dm = pr.dmap;
          if (!half_out) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              tma_store_2d(dm, stg + (h * 2) * A_PLANE_BYTES, tj * TN + h * 32, ti * TM);
              tma_store_2d(dm + 1, stg + (h * 2 + 1) * A_PLANE_BYTES, tj * TN + h * 32, ti * TM);
            }
          } else {
            tma_store_2d(dm, stg, tj * TN, ti * TM);
            tma_store_2d(dm + 1, stg + A_PLANE_BYTES, tj * TN, ti * TM);
          }
          tma_store_commit();
          if (first) stamp(round, 3);
        }
        if (pr.red_out != nullptr) {
          ssq = warp_sum(ssq);
          tr = warp_sum(tr);
          if (lane == 0) { s_red[warp * 2] = ssq; s_red[warp * 2 + 1] = tr; }
          named_bar_sync(1, T_EPI_THREADS);
          if (issuer) {
            const int ntj = n / TN;
            pr.red_out[(ti * ntj + tj) * 2] = ((s_red[0] + s_red[2]) + (s_red[4] + s_red[6])) +
                                              ((s_red[8] + s_red[10]) + (s_red[12] + s_red[14]));
            pr.red_out[(ti * ntj + tj) * 2 + 1] = ((s_red[1] + s_red[3]) + (s_red[5] + s_red[7])) +
                                                  ((s_red[9] + s_red[11]) + (s_red[13] + s_red[15]));
          }
        }
        if (issuer) {
          tma_store_wait_all0();   // stores complete (not only read): the staging smem is free, the data is out
          if (first) stamp(round, 4);
        }
      }
      // ---- end of tile: staging smem free, every role done
      __syncthreads();
    }
    // ---- grid-wide barrier between two rounds (the last round of the launch ends with the kernel)
    if (round + 1 < r1) {
      prefetch_round(round + 1);
      __syncthreads();
      if (threadIdx.x == 0) {
        ++barriers_done;
        const unsigned target = barriers_done * gridDim.x;
        stamp(round, 5);
        asm volatile("fence.proxy.async;" ::: "memory");
        __threadfence();
        atomicAdd(grid_counter, 1u);
        if (ld_acquire_gpu_u32(grid_counter) < target) {
          const long long t0 = clock64();
          while (ld_acquire_gpu_u32(grid_counter) < target)
            if (clock64() - t0 > (8ll << 30)) __trap();   // ~4 s at 2 GHz: a lost CTA must not hang the stream
        }
        __threadfence();
        asm volatile("fence.proxy.async;" ::: "memory");
        stamp(round, 6);
      }
      __syncthreads();
    }
  }
}

// ---- helpers: grid (5 layers, NB CTAs), 256 threads; reductions via fixed-order partials (deterministic)
__device__ __forceinline__ float block_sum_256(float v, float* s_red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) t += s_red[i];
  return t;
}
// Sum of the (<= NRED) reduction partials {a_i, b_i}, by the whole 256-thread block in a fixed tree (every CTA of a
// layer gets the same bits).  Was a serial loop in every thread: 32-128 dependent-issue global loads at the head of
// each element-wise helper, ~20 us of the 40-50 us those kernels took.
__device__ __forceinline__ void sum_partials(const float* red, int count, float& a, float& b, float* s_red16) {
  float va = 0.f, vb = 0.f;
  if ((int)threadIdx.x < count) { va = red[2 * threadIdx.x]; vb = red[2 * threadIdx.x + 1]; }
  va = warp_sum(va);
  vb = warp_sum(vb);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) { s_red16[threadIdx.x >> 5] = va; s_red16[8 + (threadIdx.x >> 5)] = vb; }
  __syncthreads();
  a = 0.f; b = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) { a += s_red16[i]; b += s_red16[8 + i]; }
}
__device__ __forceinline__ int gemm_tiles(int n) { return ((n + TM - 1) / TM) * (n / TN); }

// covariance from (reduced) raw sums:  mu = sums/N; cov = S_raw/N - mu mu^T + eps I     (ST:171-173, 177)
// target mode: cov_t from (mean_t, srm_t), plus sum-of-squares partials of cov_t for the NS normalisation.
__global__ void __launch_bounds__(256) w2_cov_kernel(const W2Layer* __restrict__ layers, int from_target) {
  __shared__ float s_red[8];
  const W2Layer L = layers[blockIdx.x];
  const int n = L.n;
  const size_t nn = (size_t)n * n;
  const float inv_n = from_target ? 1.f : 1.f / L.npix;
  const float* S = from_target ? L.srm_t : L.S_raw;
  const float* sm = from_target ? L.mean_t : L.sums;
  float* cov = from_target ? L.cov_t : L.cov;
  float ssq = 0.f;
  for (int e = blockIdx.y * 256 + threadIdx.x; e < n * n; e += NB * 256) {
    const int i = e / n, j = e - i * n;
    const int lo = min(i, j), hi = max(i, j);  // read the upper triangle of S: cov must be symmetric bit-for-bit
    float v = S[(size_t)lo * n + hi] * inv_n - (sm[lo] * inv_n) * (sm[hi] * inv_n);
    if (i == j) v += L.eps;
    store_split(cov, nn, e, v);
    store_split(cov + 2 * nn, nn, e, v);  // cov^T = cov bit-for-bit (upper triangle of S read for both)
    ssq = fmaf(v, v, ssq);
  }
  ssq = block_sum_256(ssq, s_red);
  if (threadIdx.x == 0) { L.red[blockIdx.y * 2] = ssq; L.red[blockIdx.y * 2 + 1] = 0.f; }
  if (blockIdx.y == 0) {
    float tr = 0.f, md = 0.f;
    for (int i = threadIdx.x; i < n; i += 256) {
      const float m = sm[i] * inv_n;
      tr += S[(size_t)i * n + i] * inv_n - m * m + L.eps;
      if (!from_target) {
        L.mu[i] = m;
        const float d = m - L.mean_t[i];
        md += d * d;
      }
    }
    tr = block_sum_256(tr, s_red);
    md = block_sum_256(md, s_red);
    if (threadIdx.x == 0) {
      if (from_target) L.scal[W2S_TR_COV_T] = tr;
      else { L.scal[W2S_TR_COV] = tr; L.scal[W2S_MEAN_DIFF] = md / n; }
    }
  }
}

// Y = M / ||M||_F, Z = I        (SQ:15-19).  ||M||^2 arrives as partials (cov kernel: NB; GEMM tiles otherwise)
__global__ void __launch_bounds__(256) w2_ns_init_kernel(const W2Layer* __restrict__ layers, int from_target) {
  __shared__ float s_red16[16];
  const W2Layer L = layers[blockIdx.x];
  const int n = L.n;
  const size_t nn = (size_t)n * n;
  const float* M = from_target ? L.cov_t : L.M;
  float ss, dummy;
  sum_partials(L.red, from_target ? NB : gemm_tiles(n), ss, dummy, s_red16);
  const float norm = sqrtf(ss);
  for (int e = blockIdx.y * 256 + threadIdx.x; e < n * n; e += NB * 256) {
    const int i = e / n, j = e - i * n;
    // Y, Z are fp16 plane pairs: planes hi, lo', hi^T, lo'^T of n*n HALFS each
    store_split_h(L.Y[0], nn, e, load2(M, nn, e) / norm);
    store_split_h(L.Y[0], nn, 2 * nn + e, load2(M + 2 * nn, nn, e) / norm);  // Y^T from the planes of M^T (cov_t: symmetric)
    const __half z0 = __float2half_rn((i == j) ? 1.f : 0.f), zero = __float2half_rn(0.f);
    __half* Zh = reinterpret_cast<__half*>(L.Z[0]);
    Zh[e] = z0; Zh[nn + e] = zero; Zh[2 * nn + e] = z0; Zh[3 * nn + e] = zero;
  }
  if (blockIdx.y == 0 && threadIdx.x == 0) L.scal[W2S_NORM_A] = norm;
}

// target: P = Y sqrt(norm)                                              (ST:159, SQ:25)
__global__ void __launch_bounds__(256) w2_target_finish_kernel(const W2Layer* __restrict__ layers) {
  const W2Layer L = layers[blockIdx.x];
  const int n = L.n;
  const size_t nn = (size_t)n * n;
  const float s = sqrtf(L.scal[W2S_NORM_A]);
  for (int e = blockIdx.y * 256 + threadIdx.x; e < n * n; e += NB * 256) {
    store_split(L.P, nn, e, load2_h(L.Y[0], nn, e) * s);
    store_split(L.P + 2 * nn, nn, e, load2_h(L.Y[0], nn, 2 * nn + e) * s);  // P^T from the planes of Y^T
  }
}

// forward finish: R = Y sqrt(normA); loss; seeds of the Lyapunov backward    (SQ:25, ST:178-181, SQ:37-41).
// ||Y||^2 and tr(Y) arrive as per-tile partials written by the last NS round.
__global__ void __launch_bounds__(256) w2_fwd_finish_kernel(const W2Layer* __restrict__ layers, float* loss_terms) {
  __shared__ float s_red16[16];
  const W2Layer L = layers[blockIdx.x];
  const int n = L.n;
  const size_t nn = (size_t)n * n;
  float ss, tr;
  sum_partials(L.red, gemm_tiles(n), ss, tr, s_red16);
  const float sq = sqrtf(L.scal[W2S_NORM_A]);
  const float norm_y = sqrtf(ss);
  const float norm_r = sq * norm_y;                     // ||R||_F
  const float tr_r = tr * sq;
  const float seed = -2.f * L.weight / (n * norm_r);    // grad_output / ||z|| with grad_output = -2 w / C * I
  // q only ever enters linearly (q' = q E / 2, U = P^T q, Gc = U P^T / 2): the iteration runs on q * 2^k with
  // |seed| * 2^k in [0.5, 1), which keeps the fp16 pair of a 1e-5-sized seed out of the subnormals; 2^-k goes into the
  // alpha of the Gc GEMM (exact powers of two: no rounding changes)
  const float qscale = (fabsf(seed) > 0.f && isfinite(seed)) ? exp2f(-floorf(log2f(fabsf(seed))) - 1.f) : 1.f;
  for (int e = blockIdx.y * 256 + threadIdx.x; e < n * n; e += NB * 256) {
    const int i = e / n, j = e - i * n;
    store_split_h(L.A[0], nn, e, load2_h(L.Y[0], nn, e) / norm_y);   // a = z / ||z||
    store_split_h(L.A[0], nn, 2 * nn + e, load2_h(L.Y[0], nn, 2 * nn + e) / norm_y);
    const float q0 = (i == j) ? seed * qscale : 0.f;
    store_split_h(L.Q[0], nn, e, q0);
    store_split_h(L.Q[0], nn, 2 * nn + e, q0);
  }
  if (blockIdx.y == 0 && threadIdx.x == 0) {
    L.scal[W2S_QSCALE] = qscale;
    *L.gc_alpha = 0.5f / qscale;
    const float cov_diff = (L.scal[W2S_TR_COV_T] + L.scal[W2S_TR_COV] - 2.f * tr_r) / n;
    const float l = (L.scal[W2S_MEAN_DIFF] + cov_diff) * L.weight;
    L.scal[W2S_LOSS] = l;
    loss_terms[blockIdx.x] = l;
  }
}

// backward finish 1: Gs = Gc + Gc^T; bf16 Gs/N ([C][C]) for the tap-gradient GEMM
__global__ void __launch_bounds__(256) w2_bwd_finish_kernel(const W2Layer* __restrict__ layers) {
  const W2Layer L = layers[blockIdx.x];
  const int n = L.n;
  const size_t nn = (size_t)n * n;
  const float inv_n = 1.f / L.npix;
  for (int e = blockIdx.y * 256 + threadIdx.x; e < n * n; e += NB * 256) {
    const int i = e / n, j = e - i * n;
    const float gs = load2(L.Gc, nn, e) + load2(L.Gc, nn, (size_t)j * n + i);
    L.Gs[e] = gs;
    L.gs_bf16[e] = __float2bfloat16(gs * inv_n);
  }
}
// backward finish 2: gmu = 2w(mu - mu_t)/C - Gs mu  (one warp per row), emitted divided by N
__global__ void __launch_bounds__(256) w2_gmu_kernel(const W2Layer* __restrict__ layers) {
  const W2Layer L = layers[blockIdx.x];
  const int n = L.n;
  const int lane = threadIdx.x & 31;
  const float inv_n = 1.f / L.npix;
  for (int i = blockIdx.y * 8 + (threadIdx.x >> 5); i < n; i += NB * 8) {
    float s = 0.f;
    for (int j = lane; j < n; j += 32) s = fmaf(L.Gs[(size_t)i * n + j], L.mu[j], s);
    s = warp_sum(s);
    if (lane == 0) L.gmu_bias[i] = (2.f * L.weight * (L.mu[i] - L.mean_t[i]) / n - s) * inv_n;
  }
}

__global__ void sum_planes_kernel(float* __restrict__ dst, const float* __restrict__ pair, size_t nn) {
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < nn; e += (size_t)gridDim.x * blockDim.x)
    dst[e] = pair[e] + pair[nn + e];
}

}  // namespace

int preload_w2_kernels() {
  cudaFuncAttributes fa;
#define STB_PRELOAD(k) STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(k)))
  STB_PRELOAD(w2_chain_kernel); STB_PRELOAD(w2_cov_kernel); STB_PRELOAD(w2_ns_init_kernel);
  STB_PRELOAD(w2_target_finish_kernel); STB_PRELOAD(w2_fwd_finish_kernel); STB_PRELOAD(w2_bwd_finish_kernel);
  STB_PRELOAD(w2_gmu_kernel); STB_PRELOAD(sum_planes_kernel);
#undef STB_PRELOAD
  return STB_OK;
}

int W2Engine::read_matrix(float* dst, const float* pair, int n, cudaStream_t s) {
  sum_planes_kernel<<<64, 256, 0, s>>>(dst, pair, (size_t)n * n);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

// ================================================================================================ host engine
size_t W2Engine::layer_floats(int n) {
  // 4 planes (hi, lo, hi^T, lo^T): cov, M, X, Y[2], Z[2], T, A[2], Q[2], E, U, Gc, P, cov_t, Qf (18); single: Gs, srm_t, X1
  // (the fp16 pairs Y, Z, T, A, Q, E use half of their slot)
  return (size_t)(18 * 4 + 3) * n * n + 8 * (size_t)n + 64 + 2 * NRED + 1024;
}

size_t W2Engine::workspace_bytes() {
  // the largest configuration: all six style taps of the reference model, 1, 6, 11, 20, 22 and 29
  size_t fl = 0;
  const int ns[W2_MAX_LAYERS] = {64, 128, 256, 512, 512, 512};
  for (int l = 0; l < W2_MAX_LAYERS; ++l) fl += layer_floats(ns[l]) + (size_t)ns[l] * ns[l] / 2 + 64;  // + bf16 Gs
  // + device copies of the layer table, tensor maps, problems and tiles
  return fl * 4 + (size_t(1) << 20);
}

namespace {
struct Builder {
  std::vector<W2Round>* rounds = nullptr;
  std::vector<CUtensorMap> maps;
  std::map<const float*, int> map_index;
  std::set<const float*> half_mats;   // matrices kept as fp16 plane pairs (4 planes of n*n halfs at the slot's start)
  CUtensorMap* d_maps = nullptr;
  int rc = 0;
  bool is_half(const float* m) const { return half_mats.count(m) != 0; }
  int maps_for(const float* m, int n) {
    auto it = map_index.find(m);
    if (it != map_index.end()) return it->second;
    const int idx = (int)maps.size();
    maps.resize(idx + 4);
    const size_t nn = (size_t)n * n;
    int r;
    if (is_half(m)) {
      const __half* h = reinterpret_cast<const __half*>(m);
      r = make_tmap_f16_2d(&maps[idx + 0], h, n, n, 2 * TKF, TM);               // 64 halfs = 128 bytes per box row
      if (!r) r = make_tmap_f16_2d(&maps[idx + 1], h + nn, n, n, 2 * TKF, TM);
      if (!r) r = make_tmap_f16_2d(&maps[idx + 2], h + 2 * nn, n, n, 2 * TKF, TN);
      if (!r) r = make_tmap_f16_2d(&maps[idx + 3], h + 3 * nn, n, n, 2 * TKF, TN);
    } else {
      r = make_tmap_f32_2d(&maps[idx + 0], m, n, n, TKF, TM);               // 128-row boxes: A loads, D stores
      if (!r) r = make_tmap_f32_2d(&maps[idx + 1], m + nn, n, n, TKF, TM);
      if (!r) r = make_tmap_f32_2d(&maps[idx + 2], m + 2 * nn, n, n, TKF, TN);  // 64-row boxes on the planes of the
      if (!r) r = make_tmap_f32_2d(&maps[idx + 3], m + 3 * nn, n, n, TKF, TN);  // transpose: B loads
    }
    if (r) rc = r;
    map_index[m] = idx;
    return idx;
  }
  void begin_round() { rounds->emplace_back(); rounds->back().n_tiles = 0; rounds->back().n_probs = 0; }
  // D = alpha op(A) B' + gamma I.  a_t: op(A) = A^T (its planes sit 2*n*n floats after A's).  b_t: B' = B^T, whose
  // K-major rows are B's own planes 0,1 -- registered under the key B - 2*n*n so that "+2" lands on them.
  // write_t: also emit the planes of D^T (D is later used as a right factor).
  void add(int n, float* D, const float* A, const float* B, float alpha, float gamma = 0.f, float* red_out = nullptr,
           int write_t = 1, int a_t = 0, int b_t = 0) {
    W2Round& R = rounds->back();
    if (R.n_probs >= W2_MAX_PROBS) { rc = STB_ERR_STATE; return; }
    const size_t nn = (size_t)n * n;
    TcProb& p = R.probs[R.n_probs];
    p.amap = d_maps + maps_for(a_t ? A + 2 * nn : A, n);
    p.bmap = d_maps + maps_for(b_t ? B - 2 * nn : B, n) + 2;
    p.dmap = d_maps + maps_for(D, n);
    p.D = D; p.red_out = red_out; p.n = n; p.alpha = alpha; p.gamma = gamma; p.write_t = write_t;
    p.in_half = is_half(A) ? 1 : 0;
    p.out_half = is_half(D) ? 1 : 0;
    if (is_half(A) != is_half(B) || ((a_t || b_t) && is_half(A))) { rc = STB_ERR_STATE; return; }
    for (int i = 0; i < (n + TM - 1) / TM; ++i)
      for (int j = 0; j < n / TN; ++j) {
        if (R.n_tiles >= W2_MAX_TILES) { rc = STB_ERR_STATE; return; }
        R.tiles[R.n_tiles++] = (uint32_t)R.n_probs << 16 | (uint32_t)i << 8 | (uint32_t)j;
      }
    ++R.n_probs;
  }
};
constexpr int MAX_MAPS = W2_MAX_LAYERS * 32 * 4;
}  // namespace

int W2Engine::init(void* ws, size_t bytes, int nl, const int* n_per_layer) {
  STB_CHECK(bytes >= workspace_bytes(), STB_ERR_WORKSPACE, "W2 workspace too small");
  STB_CHECK(nl >= 0 && nl <= W2_MAX_LAYERS, STB_ERR_INVALID, "W2: %d layers (at most %d)", nl, W2_MAX_LAYERS);
  for (int l = 0; l < nl; ++l)
    STB_CHECK(n_per_layer[l] == 64 || n_per_layer[l] == 128 || n_per_layer[l] == 256 || n_per_layer[l] == 512,
              STB_ERR_INVALID, "W2: %d channels (64, 128, 256 or 512)", n_per_layer[l]);
  n_layers = nl;
  uint8_t* base = static_cast<uint8_t*>(ws);
  size_t off = 0;
  auto take = [&](size_t nbytes) { void* p = base + off; off += (nbytes + 255) & ~size_t(255); return p; };
  for (int l = 0; l < nl; ++l) {
    W2Layer& L = host_layers[l];
    const int n = n_per_layer[l];
    const size_t nn = (size_t)n * n * 4, pp = 4 * nn;  // single plane / (hi, lo, hi^T, lo^T)
    L.n = n;
    L.eps = 1e-4f;
    L.cov = (float*)take(pp); L.M = (float*)take(pp); L.X = (float*)take(pp);
    L.Y[0] = (float*)take(pp); L.Y[1] = (float*)take(pp); L.Z[0] = (float*)take(pp); L.Z[1] = (float*)take(pp);
    L.T = (float*)take(pp); L.A[0] = (float*)take(pp); L.A[1] = (float*)take(pp);
    L.Q[0] = (float*)take(pp); L.Q[1] = (float*)take(pp); L.E = (float*)take(pp);
    L.U = (float*)take(pp); L.Gc = (float*)take(pp); L.P = (float*)take(pp); L.cov_t = (float*)take(pp);
    L.Qf = (float*)take(pp);
    L.Gs = (float*)take(nn); L.srm_t = (float*)take(nn); L.X1 = (float*)take(nn); L.X23 = nullptr;
    L.S_raw = nullptr; L.sums = nullptr;  // bound per plan (stats buffer)
    L.mu = (float*)take(n * 4); L.mean_t = (float*)take(n * 4); L.gmu_bias = (float*)take(n * 4);
    L.scal = (float*)take(64 * 4);
    L.red = (float*)take(2 * NRED * 4);
    L.gs_bf16 = (bf16*)take((size_t)n * n * 2);
    L.weight = 0.f; L.npix = 1.f;
  }
  d_layers = (W2Layer*)take(sizeof(W2Layer) * W2_MAX_LAYERS);
  d_maps = (CUtensorMap*)take(sizeof(CUtensorMap) * MAX_MAPS);
  d_grid_counter = (unsigned*)take(256);
  d_trace = (unsigned long long*)take(W2_TRACE_WORDS * 8);

  // ---- build the round lists once (pointers are stable)
  Builder b;
  b.d_maps = d_maps;
  b.rounds = &rounds;
  rounds.clear();
  for (int l = 0; l < nl; ++l) {  // the normalised iterates of both iterations live as fp16 plane pairs
    W2Layer& L = host_layers[l];
    for (float* m : {L.Y[0], L.Y[1], L.Z[0], L.Z[1], L.T, L.A[0], L.A[1], L.Q[0], L.Q[1], L.E}) b.half_mats.insert(m);
  }
  auto begin_round = [&]() { b.begin_round(); };
  auto end_round = [&]() {};
  auto ns_rounds = [&]() {  // 12 x { T = 1.5 I - 0.5 Z Y ; Y' = Y T, Z' = T Z }, result ends in Y[0]
    for (int it = 0; it < 12; ++it) {
      const int s = it & 1, d = s ^ 1;
      begin_round();
      for (int l = nl - 1; l >= 0; --l) { W2Layer& L = host_layers[l]; b.add(L.n, L.T, L.Z[s], L.Y[s], -0.5f, 1.5f); }
      end_round();
      begin_round();
      for (int l = nl - 1; l >= 0; --l) {  // largest matrices first: the tiles beyond one per SM are short ones
        W2Layer& L = host_layers[l];
        b.add(L.n, L.Y[d], L.Y[s], L.T, 1.f, 0.f, it == 11 ? L.red : nullptr);
        if (it < 11) b.add(L.n, L.Z[d], L.T, L.Z[s], 1.f);  // Z is dead after the last Y
      }
      end_round();
    }
  };
  // (a) target chain: NS on cov_t
  r_target_begin = (int)rounds.size();
  ns_rounds();
  r_target_end = (int)rounds.size();
  // (b) iterate forward: X = P cov; M = X P; NS
  r_fwd_begin = (int)rounds.size();
  begin_round();
  for (int l = nl - 1; l >= 0; --l) { W2Layer& L = host_layers[l]; b.add(L.n, L.X, L.P, L.cov, 1.f, 0.f, nullptr, 0); }
  end_round();
  begin_round();
  for (int l = nl - 1; l >= 0; --l) { W2Layer& L = host_layers[l]; b.add(L.n, L.M, L.X, L.P, 1.f, 0.f, L.red, 1); }  // M^T planes: ns_init reads them coalesced
  end_round();
  r_fwd_ns_begin = (int)rounds.size();
  ns_rounds();
  r_fwd_end = (int)rounds.size();
  // (c) backward, SQ:42-46:  E = 3I - a a;  q' = (q E - a^T (a^T q - q a)) / 2;  a' = a E / 2.
  // On this path grad_output is always a multiple of I (d/dR of -2 w tr(R)/C), `a` is symmetric and every q is a
  // polynomial in `a`, so the commutator a^T q - q a is identically zero in exact arithmetic (the reference
  // evaluates its rounding noise, ~1e-7 relative); the schedule below drops it:  q' = q E / 2.
  r_bwd_begin = (int)rounds.size();
  for (int it = 0; it < 12; ++it) {
    const int s = it & 1, d = s ^ 1;
    begin_round();
    for (int l = nl - 1; l >= 0; --l) { W2Layer& L = host_layers[l]; b.add(L.n, L.E, L.A[s], L.A[s], -1.f, 3.f); }
    end_round();
    begin_round();
    for (int l = nl - 1; l >= 0; --l) {
      W2Layer& L = host_layers[l];
      b.add(L.n, it == 11 ? L.Qf : L.Q[d], L.Q[s], L.E, 0.5f);   // the final q leaves the iteration as a TF32 pair
      if (it < 11) b.add(L.n, L.A[d], L.A[s], L.E, 0.5f);
    }
    end_round();
  }
  // after 12 its q (times the layer's power-of-two q scale) is in Qf.  U = P^T q ; Gc = alpha U P^T + (w/C) I with
  // alpha = 0.5 / qscale patched on the device by w2_fwd_finish_kernel, gamma per layer in upload_layers
  begin_round();
  for (int l = nl - 1; l >= 0; --l) { W2Layer& L = host_layers[l]; b.add(L.n, L.U, L.P, L.Qf, 1.f, 0.f, nullptr, 0, 1, 0); }
  end_round();
  begin_round();
  gc_round = (int)rounds.size() - 1;
  for (int l = nl - 1; l >= 0; --l) { W2Layer& L = host_layers[l]; b.add(L.n, L.Gc, L.U, L.P, 0.5f, 0.f, nullptr, 0, 0, 1); }
  end_round();
  r_bwd_end = (int)rounds.size();
  STB_CHECK(b.rc == 0, STB_ERR_CUDA, "W2 round construction failed (%d): %s", b.rc, last_error_string().c_str());
  STB_CHECK((int)b.maps.size() <= MAX_MAPS, STB_ERR_WORKSPACE, "W2 tensor map table overflow (%zu)", b.maps.size());

  d_rounds = (W2Round*)take(sizeof(W2Round) * std::max<size_t>(rounds.size(), 1));
  STB_CHECK(off <= bytes, STB_ERR_WORKSPACE, "W2 workspace overflow (%zu > %zu)", off, bytes);
  STB_CUDA_CHECK(cudaMemcpy(d_rounds, rounds.data(), sizeof(W2Round) * rounds.size(), cudaMemcpyHostToDevice));
  // the rounds list the layers deepest first: layer l is problem nl - 1 - l of the Gc round
  for (int l = 0; l < nl; ++l) host_layers[l].gc_alpha = &d_rounds[gc_round].probs[nl - 1 - l].alpha;
  if (nl == 0) return STB_OK;
  STB_CUDA_CHECK(cudaMemcpy(d_maps, b.maps.data(), sizeof(CUtensorMap) * b.maps.size(), cudaMemcpyHostToDevice));
  STB_CUDA_CHECK(cudaMemcpy(d_layers, host_layers, sizeof(W2Layer) * nl, cudaMemcpyHostToDevice));
  return STB_OK;
}

int W2Engine::upload_layers(cudaStream_t s) {
  // layer weights enter the Gc round through gamma = w / C (rounds travel as kernel parameters)
  if (n_layers == 0) return STB_OK;
  for (int l = 0; l < n_layers; ++l)
    rounds[gc_round].probs[n_layers - 1 - l].gamma = host_layers[l].weight / host_layers[l].n;
  STB_CUDA_CHECK(cudaMemcpyAsync(d_rounds + gc_round, &rounds[gc_round], sizeof(W2Round), cudaMemcpyHostToDevice, s));
  STB_CUDA_CHECK(cudaMemcpyAsync(d_layers, host_layers, sizeof(W2Layer) * n_layers, cudaMemcpyHostToDevice, s));
  return STB_OK;
}

int W2Engine::run_rounds(int r0, int r1, cudaStream_t s) {
  if (r1 <= r0) return STB_OK;
  STB_TRY(ensure_dynamic_smem(reinterpret_cast<const void*>(w2_chain_kernel), T_SMEM_BYTES));
  // STB_W2_CHAIN=0: one launch per round (no grid barrier, no cooperative launch) -- diagnostic / fallback
  static const bool chain = [] { const char* e = getenv("STB_W2_CHAIN"); return !(e && e[0] == '0'); }();
  const int sms = num_sms();
  if (!chain) {
    for (int r = r0; r < r1; ++r) {
      const int grid = rounds[r].n_tiles < sms ? rounds[r].n_tiles : sms;
      w2_chain_kernel<<<grid, T_THREADS, T_SMEM_BYTES, s>>>(d_rounds, r, r + 1, d_grid_counter, nullptr);
    }
    STB_CUDA_CHECK(cudaGetLastError());
    return STB_OK;
  }
  int max_tiles = 1;
  for (int r = r0; r < r1; ++r) max_tiles = rounds[r].n_tiles > max_tiles ? rounds[r].n_tiles : max_tiles;
  STB_CUDA_CHECK(cudaMemsetAsync(d_grid_counter, 0, sizeof(unsigned), s));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(max_tiles < sms ? max_tiles : sms);   // one CTA per SM: all co-resident (cooperative launch)
  cfg.blockDim = dim3(T_THREADS);
  cfg.dynamicSmemBytes = T_SMEM_BYTES;
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeCooperative;
  at[0].val.cooperative = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  const W2Round* dr = d_rounds;
  unsigned* ctr = d_grid_counter;
  static const bool tracing = [] { const char* e = getenv("STB_W2_TRACE"); return e && e[0] == '1'; }();
  unsigned long long* tr = tracing ? d_trace : nullptr;
  STB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, w2_chain_kernel, dr, r0, r1, ctr, tr));
  return STB_OK;
}

int W2Engine::build_targets(cudaStream_t s) {
  // srm_t / mean_t already hold the blended target moments (ST:443-450)
  if (n_layers == 0) return STB_OK;
  const dim3 grid(n_layers, NB);
  w2_cov_kernel<<<grid, 256, 0, s>>>(d_layers, 1);
  w2_ns_init_kernel<<<grid, 256, 0, s>>>(d_layers, 1);
  STB_TRY(run_rounds(r_target_begin, r_target_end, s));
  w2_target_finish_kernel<<<grid, 256, 0, s>>>(d_layers);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

int W2Engine::forward_backward(float* loss_terms, cudaStream_t s) {
  if (n_layers == 0) return STB_OK;
  const dim3 grid(n_layers, NB);
  w2_cov_kernel<<<grid, 256, 0, s>>>(d_layers, 0);
  STB_TRY(run_rounds(r_fwd_begin, r_fwd_ns_begin, s));
  w2_ns_init_kernel<<<grid, 256, 0, s>>>(d_layers, 0);
  STB_TRY(run_rounds(r_fwd_ns_begin, r_fwd_end, s));
  w2_fwd_finish_kernel<<<grid, 256, 0, s>>>(d_layers, loss_terms);
  STB_TRY(run_rounds(r_bwd_begin, r_bwd_end, s));
  w2_bwd_finish_kernel<<<grid, 256, 0, s>>>(d_layers);
  w2_gmu_kernel<<<grid, 256, 0, s>>>(d_layers);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

}  // namespace stb
