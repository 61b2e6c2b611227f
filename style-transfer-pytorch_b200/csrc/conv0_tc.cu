// conv0 forward (Normalize + replicate-pad 3x3 conv 3 -> 64 + bias + ReLU) as ONE wgmma kernel:
//   VGGFeatures.forward, first module    style_transfer/style_transfer.py:39,52-59,85-89 of the reference  (ST)
//   transforms.Normalize                 ST:30-31
// K = 27 is too short for a tensor-core GEMM and fp32 pixels do not fit bf16, so every pixel's K row is the im2col of
// the normalised, replicate-padded image in split form: k < 27 the bf16 "hi" part of tap (c*3+ky)*3+kx, 27 <= k < 54
// the bf16 residual x - hi ("lo": together 16 mantissa bits), the rest zero; the weights are laid out the same way
// (pack_weights_conv0_fwd).  Unlike the earlier two-pass version (im2col kernel -> 537 MB operand in HBM -> 1x1
// pixel-GEMM) the operand rows are produced straight into the SW128 shared-memory tile the MMA reads: the only HBM
// traffic left is the 12 B/pixel image read and the 128 B/pixel activation write, which is the bound.
//
// Persistent CTAs (two per SM: the roles are latency- not throughput-bound).  Work item = 4 image rows x 128 pixels (4 M-tiles sharing one 6 x 130 x 3 halo):
//   warps 4-11 producers: halo via cp.async (next item prefetched during the current one), one thread per pixel
//              builds the 128-byte K row, fence.proxy.async, arrive on the tile's "full" mbarrier (ring of 2 tiles)
//   warps 0-3  one warpgroup: 2 x 4 x wgmma (M64 N64 K16) per tile into registers, one M64 half at a time -> + bias, ReLU -> bf16 ->
//              swizzled staging -> TMA store (OOB pixels clipped)
#include "kernels.h"
#include "ptx.cuh"

namespace stb {

namespace {

constexpr int C0_PX = 128, C0_ROWS = 4;
constexpr int C0_RING = 2;                          // A tiles in flight
constexpr int C0_PROD = 256, C0_EPI = 128;
constexpr int C0_THREADS = C0_EPI + C0_PROD;        // 384
constexpr int HALO_W = 132, HALO_ROWS = C0_ROWS + 2;
constexpr int HALO_FLOATS = 3 * HALO_ROWS * HALO_W;
constexpr int A_TILE = C0_PX * 128;                 // 16 KiB
constexpr int OFF_A = 0;
constexpr int OFF_B = OFF_A + C0_RING * A_TILE;     // 8 KiB weights [64 n][64 k]
constexpr int OFF_STG = OFF_B + 64 * 128;           // 2 x 16 KiB store staging
constexpr int OFF_HALO = OFF_STG + 2 * A_TILE;
constexpr int OFF_BIAS = OFF_HALO + 2 * HALO_FLOATS * 4;
constexpr int OFF_BAR = OFF_BIAS + 64 * 4;
constexpr int C0_SMEM = OFF_BAR + 2 * C0_RING * 8 + 1024;
static_assert(OFF_HALO % 16 == 0 && OFF_BAR % 8 == 0, "alignment");

__constant__ float c0_mean[3] = {0.485f, 0.456f, 0.406f};

__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ int clampi0(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

__global__ void __launch_bounds__(C0_THREADS, 2)
conv0_fwd_kernel(const float* __restrict__ img, const bf16* __restrict__ w0p, const float* __restrict__ bias,
                 const __grid_constant__ CUtensorMap tm_out, int H, int W) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* a_full = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* a_empty = a_full + C0_RING;
  float* s_bias = reinterpret_cast<float*>(smem + OFF_BIAS);
  float* s_halo = reinterpret_cast<float*>(smem + OFF_HALO);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int items_x = (W + C0_PX - 1) / C0_PX;
  const int n_items = ((H + C0_ROWS - 1) / C0_ROWS) * items_x;

  if (threadIdx.x == 0) {
    for (int i = 0; i < C0_RING; ++i) {
      mbar_init(&a_full[i], C0_PX);
      mbar_init(&a_empty[i], 4);   // one arrival per MMA warp once its wgmma reads are complete
    }
    fence_barrier_init();
    tma_prefetch_desc(&tm_out);
  }
  // weights -> SW128 K-major tile, bias
  for (int i = threadIdx.x; i < 512; i += C0_THREADS) {
    const int n = i >> 3, j = i & 7;
    *reinterpret_cast<uint4*>(smem + OFF_B + n * 128 + ((j ^ (n & 7)) << 4)) =
        *reinterpret_cast<const uint4*>(w0p + n * 64 + j * 8);
  }
  if (threadIdx.x < 64) s_bias[threadIdx.x] = bias[threadIdx.x];
  fence_proxy_async_smem();
  __syncthreads();

  if (warp < 4) {
    // ------------------------------------------------------------------ MMA + epilogue warpgroup
    const int te = threadIdx.x;
    const int cq = 2 * (lane & 3);
    const uint64_t bd = gmma_desc_k(smem_u32(smem + OFF_B));
    uint32_t tc = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
      const int y0 = (item / items_x) * C0_ROWS, x0 = (item % items_x) * C0_PX;
      const int nt = min(C0_ROWS, H - y0);
      for (int r = 0; r < nt; ++r, ++tc) {
        const int slot = tc & (C0_RING - 1);
        mbar_wait(&a_full[slot], (tc / C0_RING) & 1);
        const uint32_t a_tile = smem_u32(smem + OFF_A + slot * A_TILE);
        uint8_t* stg = smem + OFF_STG + (tc & 1) * A_TILE;
        if (te == 0) tma_store_wait_read<1>();  // the store issued two tiles ago has drained this buffer
        named_bar_sync(3, C0_EPI);
#pragma unroll
        for (int h = 0; h < 2; ++h) {   // pixels 64 h .. 64 h + 63, one after the other (32 accumulator registers)
          float acc[32];
          const uint64_t ad = gmma_desc_k(a_tile + h * 64 * 128);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_bf16<0, 0>(acc, ad + 2 * k, bd + 2 * k, k > 0);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_acc(acc);
          if (h == 1 && lane == 0) mbar_arrive(&a_empty[slot]);
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const int p = 64 * h + 16 * warp + (lane >> 2) + 8 * half;  // pixel of the tile
#pragma unroll
            for (int q = 0; q < 8; ++q) {
              const int n = 8 * q + cq;
              const float a = acc[4 * q + 2 * half] + s_bias[n];
              const float b = acc[4 * q + 2 * half + 1] + s_bias[n + 1];
              *reinterpret_cast<uint32_t*>(stg + p * 128 + ((q ^ (p & 7)) << 4) + cq * 2) =
                  pack_bf16x2(fmaxf(a, 0.f), fmaxf(b, 0.f));
            }
          }
        }
        fence_proxy_async_smem();
        named_bar_sync(3, C0_EPI);
        if (te == 0) {
          tma_store_3d(&tm_out, stg, 0, x0, y0 + r);
          tma_store_commit();
        }
      }
    }
    if (te == 0) tma_store_wait_all0();
  } else {
    // ------------------------------------------------------------------ producers
    const int tp = threadIdx.x - C0_EPI;
    const int half = tp >> 7, x = tp & (C0_PX - 1);
    const float inv_std[3] = {(float)(1.0 / 0.229), (float)(1.0 / 0.224), (float)(1.0 / 0.225)};
    auto prefetch = [&](int item, int buf) {
      const int y0 = (item / items_x) * C0_ROWS, x0 = (item % items_x) * C0_PX;
      float* dst = s_halo + buf * HALO_FLOATS;
      for (int e = tp; e < 3 * HALO_ROWS * (C0_PX + 2); e += C0_PROD) {
        const int c = e / (HALO_ROWS * (C0_PX + 2));
        const int rem = e - c * (HALO_ROWS * (C0_PX + 2));
        const int ry = rem / (C0_PX + 2), hx = rem - ry * (C0_PX + 2);
        const int gy = clampi0(y0 - 1 + ry, 0, H - 1), gx = clampi0(x0 - 1 + hx, 0, W - 1);
        cp_async4(dst + (c * HALO_ROWS + ry) * HALO_W + hx, img + ((size_t)c * H + gy) * W + gx);
      }
      cp_async_commit();
    };
    uint32_t tc = 0;
    int it = 0;
    if ((int)blockIdx.x < n_items) prefetch(blockIdx.x, 0);
    for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++it) {
      const int y0 = (item / items_x) * C0_ROWS;
      const int nt = min(C0_ROWS, H - y0);
      cp_async_wait_all();
      named_bar_sync(2, C0_PROD);  // this item's halo visible; everyone is done with the other buffer
      if (item + (int)gridDim.x < n_items) prefetch(item + gridDim.x, (it + 1) & 1);
      const float* hal = s_halo + (it & 1) * HALO_FLOATS;
      for (int r = half; r < nt; r += 2) {
        const uint32_t t = tc + r;
        const int slot = t & (C0_RING - 1);
        mbar_wait(&a_empty[slot], ((t / C0_RING) & 1) ^ 1);
        float v[27];
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
          for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j)
              v[(c * 3 + i) * 3 + j] = (hal[(c * HALO_ROWS + r + i) * HALO_W + x + j] - c0_mean[c]) * inv_std[c];
        // k < 27: the value itself (the pack rounds it to its bf16 "hi"); 27 <= k < 54: the residual v - hi
        auto kval = [&](int k) -> float {
          if (k < 27) return v[k];
          if (k < 54) return v[k - 27] - __bfloat162float(__float2bfloat16(v[k - 27]));
          return 0.f;
        };
        uint8_t* row = smem + OFF_A + slot * A_TILE + x * 128;
#pragma unroll
        for (int ch = 0; ch < 8; ++ch) {  // k layout: [hi0..hi26, lo0..lo26, 0 x 10]
          uint32_t wv[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) wv[q] = pack_bf16x2(kval(8 * ch + 2 * q), kval(8 * ch + 2 * q + 1));
          *reinterpret_cast<uint4*>(row + ((ch ^ (x & 7)) << 4)) = make_uint4(wv[0], wv[1], wv[2], wv[3]);
        }
        fence_proxy_async_smem();
        mbar_arrive(&a_full[slot]);
      }
      tc += nt;
    }
  }
}


// =====================================================================================================================
// conv0 backward for the interior pixels + the optimiser step, as a 1x1 GEMM followed by a 3x3 "col2im" in shared
// memory (autograd of ST:85-89 w.r.t. the image, then ST:481-486):
//     D[p][(ky,kx,c)] = sum_co g0[p][co] * w0[co][c][ky][kx]            wgmma, M = 128 pixels, N = 32 (27 used), K = 64
//     grad[c][y][x]   = sum_{ky,kx} D[(y-ky+1, x-kx+1)][(ky,kx,c)]      27 shared-memory reads per pixel
// A direct dgrad GEMM (K = 9 x 64, N = 3 padded to 16) re-reads every g0 pixel from shared memory nine times and was
// shared-memory-bandwidth bound at 2.5x the HBM time; here every g0 row is loaded and multiplied exactly once.
// Work item = a vertical strip: 126 output columns (128 D columns incl. the one-pixel halo) x 32 output rows (34 D
// rows).  Roles: warp 4 TMA producer (ring of 2 stages of one 128-pixel g0 row each, zero-filled outside the image = the
// conv's zero padding; two CTAs per SM), warps 0-3 one warpgroup: wgmma of the row into registers -> D ring (4 rows,
// k-major planes) -> gather for the output row one above -> Normalize backward + TV gradient + Adam + clamp + EMA with
// fully coalesced accesses to the fp32 planes, whose loads are issued one row ahead.
constexpr int BW_OUT = 126, BW_ROWS = 32, BW_RING = 2;
constexpr int BW_THREADS = 128 + 32;
constexpr int D_PITCH = 132, D_SLOT = 27 * D_PITCH;   // floats
constexpr int BW_OFF_A = 0;
constexpr int BW_OFF_B = BW_OFF_A + BW_RING * A_TILE;  // 32 x 128 B weights
constexpr int BW_OFF_D = BW_OFF_B + 32 * 128;
constexpr int BW_OFF_BAR = BW_OFF_D + 4 * D_SLOT * 4;
constexpr int BW_SMEM = BW_OFF_BAR + 2 * BW_RING * 8 + 1024;
static_assert(BW_OFF_BAR % 8 == 0, "alignment");

struct ImgState {
  float tv[3], m[3], v[3], p[3], e[3];
};

__global__ void __launch_bounds__(BW_THREADS, 2)
conv0_bwd_kernel(const __grid_constant__ CUtensorMap tm_g0, const bf16* __restrict__ w0q,
                 const float* __restrict__ gtv, float* __restrict__ img, float* __restrict__ exp_avg,
                 float* __restrict__ exp_avg_sq, float* __restrict__ ema, float* __restrict__ grad_out,
                 const AdamScalars* __restrict__ adam, int apply_update, int H, int W) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* a_full = reinterpret_cast<uint64_t*>(smem + BW_OFF_BAR);
  uint64_t* a_empty = a_full + BW_RING;
  float* s_d = reinterpret_cast<float*>(smem + BW_OFF_D);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int strips = (W + BW_OUT - 1) / BW_OUT;
  const int n_items = strips * ((H + BW_ROWS - 1) / BW_ROWS);

  if (threadIdx.x == 0) {
    for (int i = 0; i < BW_RING; ++i) {
      mbar_init(&a_full[i], 1);
      mbar_init(&a_empty[i], 4);   // one arrival per MMA warp once its wgmma reads are complete
    }
    fence_barrier_init();
    tma_prefetch_desc(&tm_g0);
  }
  for (int i = threadIdx.x; i < 256; i += BW_THREADS) {  // weights [32 n][64 co] -> SW128 K-major tile
    const int n = i >> 3, j = i & 7;
    *reinterpret_cast<uint4*>(smem + BW_OFF_B + n * 128 + ((j ^ (n & 7)) << 4)) =
        *reinterpret_cast<const uint4*>(w0q + n * 64 + j * 8);
  }
  fence_proxy_async_smem();
  __syncthreads();

  if (warp == 4) {
    if (elect_one()) {
      uint32_t tc = 0;
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int xs = (item % strips) * BW_OUT, ys = (item / strips) * BW_ROWS;
        const int nd = min(BW_ROWS, H - ys) + 2;
        for (int j = 0; j < nd; ++j, ++tc) {
          const int slot = tc & (BW_RING - 1);
          mbar_wait(&a_empty[slot], ((tc / BW_RING) & 1) ^ 1);
          mbar_expect_tx(&a_full[slot], A_TILE);
          tma_load_3d(smem + BW_OFF_A + slot * A_TILE, &tm_g0, &a_full[slot], 0, xs - 1, ys - 1 + j);
        }
      }
    }
    __syncwarp();
  } else {
    const int t = threadIdx.x;     // D column of the strip in the gather; output column for 1 <= t <= 126
    const int cq = 2 * (lane & 3);
    const uint64_t bd = gmma_desc_k(smem_u32(smem + BW_OFF_B));
    AdamScalars ac{};
    if (apply_update) ac = *adam;
    const float inv_std[3] = {(float)(1.0 / 0.229), (float)(1.0 / 0.224), (float)(1.0 / 0.225)};
    uint32_t tc = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
      const int xs = (item % strips) * BW_OUT, ys = (item / strips) * BW_ROWS;
      const int nd = min(BW_ROWS, H - ys) + 2;
      const int x = xs - 1 + t;
      const bool col_ok = t >= 1 && t <= BW_OUT && x >= 1 && x < W - 1;
      ImgState cur{}, nxt{};
      auto load_state = [&](int yo, ImgState& S) {
        const bool ok = col_ok && yo >= 1 && yo < H - 1;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const size_t idx = (static_cast<size_t>(c) * H + yo) * W + x;
          S.tv[c] = (ok && gtv) ? __ldg(gtv + idx) : 0.f;
          const bool ld = ok && apply_update;
          S.m[c] = ld ? exp_avg[idx] : 0.f;
          S.v[c] = ld ? exp_avg_sq[idx] : 0.f;
          S.p[c] = ld ? img[idx] : 0.f;
          S.e[c] = ld ? ema[idx] : 0.f;
        }
      };
      for (int j = 0; j < nd; ++j, ++tc) {
        if (j + 1 >= 2 && j + 1 < nd) load_state(ys + j - 1, nxt);  // state of the NEXT iteration's output row
        const int slot = tc & (BW_RING - 1);
        mbar_wait(&a_full[slot], (tc / BW_RING) & 1);
        float acc[2][16];
        const uint32_t a_tile = smem_u32(smem + BW_OFF_A + slot * A_TILE);
        wgmma_fence();
#pragma unroll
        for (int h = 0; h < 2; ++h) {   // D columns 64 h .. 64 h + 63
          const uint64_t ad = gmma_desc_k(a_tile + h * 64 * 128);
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_bf16<0, 0>(acc[h], ad + 2 * k, bd + 2 * k, k > 0);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(acc[0]);
        wgmma_fence_acc(acc[1]);
        if (lane == 0) mbar_arrive(&a_empty[slot]);
        float* drow = s_d + (j & 3) * D_SLOT;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const int col = 64 * h + 16 * warp + (lane >> 2) + 8 * half;
#pragma unroll
            for (int q = 0; q < 4; ++q)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int k = 8 * q + cq + e;
                if (k < 27) drow[k * D_PITCH + col] = acc[h][4 * q + 2 * half + e];
              }
          }
        named_bar_sync(1, 128);
        if (j >= 2) {
          const int yo = ys + j - 2;
          if (col_ok && yo >= 1 && yo < H - 1) {
            float g[3] = {0.f, 0.f, 0.f};
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
              const float* dr = s_d + ((j - ky) & 3) * D_SLOT;
#pragma unroll
              for (int kx = 0; kx < 3; ++kx)
#pragma unroll
                for (int c = 0; c < 3; ++c) g[c] += dr[((ky * 3 + kx) * 3 + c) * D_PITCH + t - kx + 1];
            }
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              const size_t idx = (static_cast<size_t>(c) * H + yo) * W + x;
              const float gg = g[c] * inv_std[c] + cur.tv[c];
              if (grad_out) grad_out[idx] = gg;
              if (apply_update) {
                float mm = cur.m[c], vv = cur.v[c], pp = cur.p[c], ee = cur.e[c];
                adam_element(ac, gg, mm, vv, pp, ee);
                exp_avg[idx] = mm; exp_avg_sq[idx] = vv; img[idx] = pp; ema[idx] = ee;
              }
            }
          }
        }
        cur = nxt;
      }
      named_bar_sync(1, 128);  // the next item restarts the D ring at slot 0
    }
  }
}

__global__ void pack_w0_bwd_q_kernel(const float* __restrict__ w0, bf16* __restrict__ out) {
  // out[n][co], n = (ky*3+kx)*3+c < 27 -> w0[co][c][ky][kx]; rows 27..31 zero
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 32 * 64) {
    const int n = i >> 6, co = i & 63;
    float v = 0.f;
    if (n < 27) {
      const int c = n % 3, kk = n / 3;
      v = w0[(co * 3 + c) * 9 + kk];
    }
    out[i] = __float2bfloat16(v);
  }
}

}  // namespace

int launch_conv0_fwd(const float* img, const bf16* w0_packed, const float* bias, bf16* out, int H, int W,
                     cudaStream_t s) {
  STB_TRY(ensure_dynamic_smem(reinterpret_cast<const void*>(conv0_fwd_kernel), C0_SMEM));
  CUtensorMap tm;
  STB_TRY(make_tmap_bf16_3d(&tm, out, 64, W, H, 128ull, (uint64_t)W * 128ull, 64, W < C0_PX ? W : C0_PX, 1));
  const int n_items = ((H + C0_ROWS - 1) / C0_ROWS) * ((W + C0_PX - 1) / C0_PX);
  const int grid = n_items < 2 * num_sms() ? n_items : 2 * num_sms();  // two CTAs per SM (92 KiB smem each)
  conv0_fwd_kernel<<<grid, C0_THREADS, C0_SMEM, s>>>(img, w0_packed, bias, tm, H, W);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

}  // namespace stb

namespace stb {

int preload_conv0_kernels() {
  cudaFuncAttributes fa;
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(conv0_fwd_kernel)));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(conv0_bwd_kernel)));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(pack_w0_bwd_q_kernel)));
  return STB_OK;
}

int pack_weights_conv0_bwd(const float* w0, bf16* out, cudaStream_t s) {
  pack_w0_bwd_q_kernel<<<8, 256, 0, s>>>(w0, out);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

int launch_conv0_bwd_interior(const bf16* g0, const bf16* w0q, const float* gtv, float* img, float* exp_avg,
                              float* exp_avg_sq, float* ema, float* grad_out, int H, int W, const AdamScalars* d_adam,
                              int apply_update, cudaStream_t s) {
  if (H < 3 || W < 3) return STB_OK;  // no interior pixels
  STB_TRY(ensure_dynamic_smem(reinterpret_cast<const void*>(conv0_bwd_kernel), BW_SMEM));
  CUtensorMap tm;
  STB_TRY(make_tmap_bf16_3d(&tm, g0, 64, W, H, 128ull, (uint64_t)W * 128ull, 64, C0_PX, 1));
  const int n_items = ((W + BW_OUT - 1) / BW_OUT) * ((H + BW_ROWS - 1) / BW_ROWS);
  const int cap = 2 * num_sms();
  conv0_bwd_kernel<<<n_items < cap ? n_items : cap, BW_THREADS, BW_SMEM, s>>>(tm, w0q, gtv, img, exp_avg, exp_avg_sq,
                                                                            ema, grad_out, d_adam, apply_update, H, W);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

}  // namespace stb
