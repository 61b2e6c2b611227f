// Second raw moment and channel sums of a pixel-major (NHWC bf16) activation on wgmma:
//     S_raw[i][j] = sum_p F[p][i] * F[p][j]        sums[i] = sum_p F[p][i]
// i.e. the un-normalised `einsum('...chw,...dhw->...cd')` and `mean([-2,-1])` of StyleLossW2.get_target
// (style_transfer/style_transfer.py:163-168 of the reference).  K is the pixel axis (up to 4.2 M), so the GEMM is
// split-K: CTA (tile, split) accumulates a 128 x BN fp32 tile over its pixel range and writes a partial; gram_reduce
// sums the partials in a fixed order (deterministic).
//
// Accuracy: the tensor core adds into its fp32 accumulator with TRUNCATION, and here every product is >= 0 (post-ReLU
// features), so a long chain of k-steps loses ~n * 2^-24.5 of the sum -- systematically, and the covariance
// (S/N - mu mu^T) and the W2 cancellation amplify that ~200x.  The MMA accumulator is therefore restarted every 32
// k-steps and DRAINED into a second set of fp32 registers (round-to-nearest adds).  C >= 256 runs as 128 x 128 tiles
// of the UPPER triangle (GCfg<128, true>: separate A atoms, 64-pixel stages); the lower triangle is mirrored by the
// reduction.
//
// Both operands are the SAME pixel-major smem tiles read "MN-major" (channel contiguous, SW128): no transpose is
// ever materialised.  Channel sums ride along as one extra N=16 MMA per k-step against a constant tile of ones.
// Roles: two consumer warpgroups (rows i0 .. i0+63 and i0+64 .. i0+127 of the tile), one TMA producer warp.
#include <cstdlib>

#include "kernels.h"
#include "ptx.cuh"

namespace stb {

namespace {

constexpr int G_STAGES = 4;
constexpr int G_THREADS = 256 + 32;
constexpr int PK_MAX = 256;

// PK = pixels per pipeline stage.  The narrow layers are pure HBM streams (C = 64: 8 KiB per 64 pixels), so they get
// deep stages (32 KiB each, 128 KiB in flight per SM); C >= 256 needs the room for the separate A atoms.
// SEP: the A block (rows i0..i0+127) is not part of the B block (columns j0..j0+BN-1) for off-diagonal tiles: separate
// A atoms in every stage (C >= 256, tiles of the upper triangle).
template <int BN, bool SEP = false>
struct GCfg {
  static constexpr int PK = BN == 64 ? 256 : (BN == 128 ? (SEP ? 64 : 128) : 64);
  static constexpr int ATOM_BYTES = PK * 128;   // 64 channels x PK pixels, bf16
  static constexpr int B_ATOMS = BN / 64;
  static constexpr int A_ATOMS = SEP ? 2 : 0;   // C <= 128: the A block is always contained in the B block
  static constexpr int STAGE_BYTES = (B_ATOMS + A_ATOMS) * ATOM_BYTES;
  // + one atom of slack: with C = 64 the (discarded) rows 64..127 of the second warpgroup read one atom past the stage
  static constexpr int OFF_ONES = G_STAGES * STAGE_BYTES + ATOM_BYTES;
  static constexpr int OFF_BAR = OFF_ONES + 2048;
  static constexpr int SMEM_BYTES = OFF_BAR + 2 * G_STAGES * 8 + 1024;
  static constexpr int CHUNK_STAGES = 32 / (PK / 16);   // stages per 32-k-step chunk
};

struct GParams {
  long P;              // number of pixels
  int C;
  int n_tj;            // column tiles
  int upper;           // 1: blockIdx.x enumerates the tiles (ti <= tj) of the upper triangle, row by row
  long chunk_per_split;  // pixels per split (multiple of PK)
  float* partials;     // [n_splits][C][C]
  float* sum_partials; // [n_splits][C]
};

template <int BN, bool SEP>
__global__ void __launch_bounds__(G_THREADS, 1)
gram_kernel(const __grid_constant__ CUtensorMap tmF, const GParams p) {
  using C = GCfg<BN, SEP>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + C::OFF_BAR);
  uint64_t* empty = full + G_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int ti = blockIdx.x / p.n_tj, tj = blockIdx.x % p.n_tj;
  if (p.upper) {  // tile index -> (ti, tj) with ti <= tj
    int rem = blockIdx.x;
    ti = 0;
    while (rem >= p.n_tj - ti) { rem -= p.n_tj - ti; ++ti; }
    tj = ti + rem;
  }
  const int split = blockIdx.y;
  const int i0 = ti * 128, j0 = tj * BN;
  const int m_valid = min(128, p.C - i0);
  const bool contained = (i0 >= j0) && (i0 + m_valid <= j0 + BN);
  const long p_begin = (long)split * p.chunk_per_split;
  const long p_end = min(p.P, p_begin + p.chunk_per_split);
  constexpr int PK = C::PK;
  constexpr int ATOM_BYTES = C::ATOM_BYTES;
  const int n_k = (int)((p_end - p_begin + PK - 1) / PK);

  // constant ones tile (bf16 1.0 = 0x3F80)
  for (int i = threadIdx.x; i < 2048 / 4; i += G_THREADS)
    reinterpret_cast<uint32_t*>(smem + C::OFF_ONES)[i] = 0x3F803F80u;
  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmF);
    // empty: one arrival per consumer warp once its wgmma reads of the stage are complete
    for (int i = 0; i < G_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
    fence_barrier_init();
  }
  fence_proxy_async_smem();  // ones tile is read by the tensor core (async proxy)
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      const uint32_t tx_bytes = (C::B_ATOMS + (contained ? 0 : C::A_ATOMS)) * ATOM_BYTES;
      int s = 0;
      uint32_t ph = 0;
      for (int k = 0; k < n_k; ++k) {
        mbar_wait(&empty[s], ph ^ 1);
        mbar_expect_tx(&full[s], tx_bytes);
        uint8_t* st = smem + s * C::STAGE_BYTES;
        const int pix = (int)(p_begin + (long)k * PK);
        for (int b = 0; b < C::B_ATOMS; ++b) tma_load_3d(st + b * ATOM_BYTES, &tmF, &full[s], j0 + b * 64, pix, 0);
        if (!contained)
          for (int a = 0; a < C::A_ATOMS; ++a)
            tma_load_3d(st + (C::B_ATOMS + a) * ATOM_BYTES, &tmF, &full[s], i0 + a * 64, pix, 0);
        if (++s == G_STAGES) { s = 0; ph ^= 1; }
      }
    }
    __syncwarp();
  } else {
    // ---- consumer warpgroup wg: Gram rows i0 + 64 wg .. i0 + 64 wg + 63 (discarded beyond m_valid).  The MMAs are
    // issued unconditionally (channel sums included, kept on diagonal tiles only): a wgmma under a branch the compiler
    // cannot prove uniform is serialised.
    const int wg = warp >> 2, wq = warp & 3;
    const bool diag = tj == ti;
    const uint64_t ones = gmma_desc_k(smem_u32(smem + C::OFF_ONES));   // K-major, every element 1
    float acc[BN / 2], tot[BN / 2], sacc[8], stot[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) tot[i] = 0.f;
    int s = 0;
    uint32_t ph = 0;
    for (int k = 0; k < n_k;) {
      // one chunk of (at most) 32 k-steps into a fresh accumulator; stage k-1 is released once only stage k's MMA
      // group is still in flight
      int prev = -1;
      for (int kc = 0; kc < C::CHUNK_STAGES && k < n_k; ++kc, ++k) {
        mbar_wait(&full[s], ph);
        const uint32_t b_addr = smem_u32(smem + s * C::STAGE_BYTES);
        const uint32_t a_addr =
            (contained ? b_addr + ((i0 - j0) >> 6) * ATOM_BYTES : b_addr + C::B_ATOMS * ATOM_BYTES) + wg * ATOM_BYTES;
        // MN-major SW128: LBO = stride between 64-channel atoms, SBO = 8 pixels; a 16-pixel K step is +2048 bytes
        const uint64_t ad = gmma_desc(a_addr, ATOM_BYTES, 1024), bd = gmma_desc(b_addr, ATOM_BYTES, 1024);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < PK / 16; ++ks) {
          const uint32_t sc = kc > 0 || ks > 0;
          wgmma_bf16<1, 1>(acc, ad + ks * 128, bd + ks * 128, sc);
          wgmma_bf16<1, 0>(sacc, ad + ks * 128, ones, sc);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        prev = s;
        if (++s == G_STAGES) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(&empty[prev]);
      wgmma_fence_acc(acc);
      wgmma_fence_acc(sacc);
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) tot[i] += acc[i];
      stot[0] += sacc[0];
      stot[1] += sacc[2];
    }
    if (n_k > 0) {
      const int cq = 2 * (lane & 3);
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int r = 64 * wg + 16 * wq + (lane >> 2) + 8 * half;
        if (r < m_valid) {
          float* dst = p.partials + ((size_t)split * p.C + (i0 + r)) * p.C + j0 + cq;
#pragma unroll
          for (int q = 0; q < BN / 8; ++q)
            *reinterpret_cast<float2*>(dst + 8 * q) = make_float2(tot[4 * q + 2 * half], tot[4 * q + 2 * half + 1]);
          if (diag && cq == 0) p.sum_partials[(size_t)split * p.C + i0 + r] = stot[half];
        }
      }
    }
  }
}

// sum partials in a fixed order: out[i] = sum_s part[s][i]; deterministic run to run.  One launch covers the Gram
// partials (n0 elements) and the channel-sum partials (n1 elements, element index continues after n0).  A block owns
// 64 elements; its 256 threads are 4 split-lanes x 64 elements: lane g adds the splits s = g, g+4, ... (4 interleaved
// accumulators for memory-level parallelism), then the four lane sums are combined in order through shared memory.
// (With one thread per element the C = 64 layer -- one split per SM, 4160 elements -- ran on 17 CTAs.)
// mirror_c > 0: part0 is a [mirror_c][mirror_c] matrix of which only the 128 x 128 tiles of the upper triangle were
// written; elements of the lower triangle read the transposed position (the Gram matrix is symmetric).
__global__ void __launch_bounds__(256)
gram_reduce_kernel(const float* __restrict__ part0, float* __restrict__ out0, long n0,
                   const float* __restrict__ part1, float* __restrict__ out1, long n1, int n_splits, int mirror_c) {
  __shared__ float s_part[4][64];
  const int g = threadIdx.x >> 6, el = threadIdx.x & 63;
  for (long base = (long)blockIdx.x * 64; base < n0 + n1; base += (long)gridDim.x * 64) {
    const long e = base + el;
    const bool in = e < n0 + n1, first = e < n0;
    const float* part = first ? part0 : part1;
    const long n = first ? n0 : n1, i = first ? e : e - n0;
    long src = i;
    if (first && mirror_c > 0) {
      const int r = (int)(i / mirror_c), c = (int)(i - (long)r * mirror_c);
      if ((r >> 7) > (c >> 7)) src = (long)c * mirror_c + r;
    }
    float a[4] = {0.f, 0.f, 0.f, 0.f};
    if (in) {
      int k = g;
      for (; k + 12 < n_splits; k += 16) {
#pragma unroll
        for (int u = 0; u < 4; ++u) a[u] += __ldg(part + (size_t)(k + 4 * u) * n + src);
      }
      for (; k < n_splits; k += 4) a[0] += __ldg(part + (size_t)k * n + src);
    }
    s_part[g][el] = (a[0] + a[1]) + (a[2] + a[3]);
    __syncthreads();
    if (g == 0 && in) (first ? out0 : out1)[i] = (s_part[0][el] + s_part[1][el]) + (s_part[2][el] + s_part[3][el]);
    __syncthreads();
  }
}

template <int BN, bool SEP>
int launch_gram_cfg(const CUtensorMap& tm, const GParams& gp, int n_tiles, int n_splits, cudaStream_t stream) {
  using C = GCfg<BN, SEP>;
  auto kern = gram_kernel<BN, SEP>;
  STB_TRY(ensure_dynamic_smem(reinterpret_cast<const void*>(kern), C::SMEM_BYTES));
  kern<<<dim3(n_tiles, n_splits), G_THREADS, C::SMEM_BYTES, stream>>>(tm, gp);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

}  // namespace

int preload_gram_kernels() {
  cudaFuncAttributes fa;
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(gram_kernel<64, false>)));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(gram_kernel<128, false>)));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(gram_kernel<128, true>)));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(gram_reduce_kernel)));
  return STB_OK;
}

// C <= 128: one tile row, BN = C.  C >= 256: 128 x 128 tiles of the upper triangle, 64-pixel stages.
static int gram_bn(int C) { return C >= 128 ? 128 : C; }
static bool gram_sep(int C) { return C >= 256; }
static int gram_pk(int C) { return C == 64 ? 256 : (C == 128 ? 128 : 64); }
static int gram_tiles(int C) {
  if (!gram_sep(C)) return 1;
  const int t = C / 128;
  return t * (t + 1) / 2;
}

static long gram_want_splits(int C) {
  const int n_tiles = gram_tiles(C);
  long want = (num_sms() + n_tiles - 1) / n_tiles;  // one CTA per SM
  {  // diagnostic knob: a different split count = a different (equally valid) fp32 summation order of the Gram
    static const int div = [] { const char* e = getenv("STB_GRAM_SPLIT_DIV"); return e ? atoi(e) : 1; }();
    if (div > 1) want = (want + div - 1) / div;
  }
  if (want < 1) want = 1;
  if (want > 1024) want = 1024;
  return want;
}

int gram_num_splits(long P, int C) {
  const int PK = gram_pk(C);
  long chunks = (P + PK - 1) / PK;
  long want = gram_want_splits(C);
  if (want > chunks) want = chunks;
  if (want < 1) want = 1;
  // make every split non-empty
  long per = (chunks + want - 1) / want;
  long n = (chunks + per - 1) / per;
  return (int)n;
}

size_t gram_partials_floats(long P, int C) { return (size_t)gram_num_splits(P, C) * ((size_t)C * C + C); }

// Upper bound of gram_partials_floats over EVERY pixel count: gram_num_splits is not monotonic in P (a band of own rows
// can need more splits than the taller local image the plan was sized for), so the workspace reserves this bound.
size_t gram_max_partials_floats(int C) { return (size_t)gram_want_splits(C) * ((size_t)C * C + C); }

int launch_gram(const bf16* F, long P, int C, float* partials_ws, size_t partials_capacity_floats, float* S_raw,
                float* sums, cudaStream_t stream) {
  STB_CHECK(C % 64 == 0 && C <= 512 && P > 0, STB_ERR_INVALID, "gram: C=%d P=%ld", C, P);
  STB_CHECK(gram_partials_floats(P, C) <= partials_capacity_floats, STB_ERR_WORKSPACE,
            "gram: split-K partials need %zu floats, %zu reserved (P=%ld, C=%d)", gram_partials_floats(P, C),
            partials_capacity_floats, P, C);
  const int BN = gram_bn(C);
  const bool sep = gram_sep(C);
  const int n_splits = gram_num_splits(P, C);
  const int PK = gram_pk(C);
  const long chunks = (P + PK - 1) / PK;
  const long per = (chunks + n_splits - 1) / n_splits;
  GParams gp;
  gp.P = P; gp.C = C; gp.n_tj = C / BN; gp.upper = sep ? 1 : 0; gp.chunk_per_split = per * PK;
  gp.partials = partials_ws;
  gp.sum_partials = partials_ws + (size_t)n_splits * C * C;
  CUtensorMap tm;
  STB_TRY(make_tmap_bf16_3d(&tm, F, C, (uint64_t)P, 1, C * 2ull, (uint64_t)P * C * 2ull, 64, PK, 1));
  static_assert(PK_MAX <= 256, "TMA box dimension limit");
  if (sep) STB_TRY((launch_gram_cfg<128, true>(tm, gp, gram_tiles(C), n_splits, stream)));
  else if (BN == 128) STB_TRY((launch_gram_cfg<128, false>(tm, gp, 1, n_splits, stream)));
  else STB_TRY((launch_gram_cfg<64, false>(tm, gp, 1, n_splits, stream)));
  const long nn = (long)C * C;
  long g = (nn + C + 63) / 64;
  if (g > 16l * num_sms()) g = 16l * num_sms();
  gram_reduce_kernel<<<(int)g, 256, 0, stream>>>(gp.partials, S_raw, nn, gp.sum_partials, sums, C, n_splits,
                                                sep ? C : 0);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

}  // namespace stb
