// HBM-bound kernels on either side of the tensor-core trunk:
//   im2col0        : Normalize (ST:30-31,85) + replicate-pad (ST:39,52-59) im2col of the image, hi/lo bf16 split, so
//                    that conv0 itself runs as a 1x1 pixel-GEMM on the tensor cores (conv_tc.cu)
//   tv             : nine-point TV loss and its gradient on the raw image (ST:184-195)
//   conv0_bwd_adam : border part of the conv0 dgrad (adjoint of replicate pad; the interior comes from the tensor
//                    cores) + Normalize backward + TV gradient -> Adam step (torch/optim/adam.py:413-546
//                    single-tensor math) -> clamp_(0,1) (ST:483-485) -> EMA (ST:250-253)
//   pool2x2 fwd/bwd: MaxPool2d(2) / Scale(AvgPool2d(2),2.0) / Scale(LPPool2d(2,2),0.78)  (ST:21-22,41-46)
//   content_sse    : sum((F22 - T)^2)  (ST:119-126)
#include "kernels.h"
#include "ptx.cuh"

namespace stb {

namespace {

__constant__ float c_std[3] = {0.229f, 0.224f, 0.225f};

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// ------------------------------------------------------------------------------------------------ conv0 fwd + TV
// grid: (ceil(W/64), H); block 256 = 64 pixels x 4 channel groups of 16.
struct TvConst {
  float k1, k3;        // gradient factors 4/(3 n1), 4/(12 n3) times tv_weight
  float l1, l3;        // loss factors 2/(3 n1), 2/(12 n3)
};

// gradient of the (unweighted) TV sum w.r.t. the replicate-padded grid position (a,b) of channel plane `x`
// (padded coordinates: pixel (y,x) sits at (y+1,x+1)); general (slow) path used for border folds only.
__device__ float tv_gpad_slow(const float* __restrict__ x, int H, int W, int a, int b, float k1, float k3) {
  auto P = [&](int i, int j) { return __ldg(x + (size_t)clampi(i - 1, 0, H - 1) * W + clampi(j - 1, 0, W - 1)); };
  float g = 0.f;
  const float c = P(a, b);
  // e3[i][j] = P[i+1][j+1]-P[i][j], i in [0,H], j in [0,W]
  if (a >= 1 && b >= 1) g += k3 * (c - P(a - 1, b - 1));
  if (a <= H && b <= W) g -= k3 * (P(a + 1, b + 1) - c);
  // e4[i][j] = P[i+1][j]-P[i][j+1]
  if (a >= 1 && b <= W) g += k3 * (c - P(a - 1, b + 1));
  if (a <= H && b >= 1) g -= k3 * (P(a + 1, b - 1) - c);
  // e1[y][x] = P[y+1][x+2]-P[y+1][x+1], rows a in [1,H]
  if (a >= 1 && a <= H) {
    if (b >= 2) g += k1 * (c - P(a, b - 1));
    if (b >= 1 && b <= W) g -= k1 * (P(a, b + 1) - c);
  }
  // e2[y][x] = P[y+2][x+1]-P[y+1][x+1], cols b in [1,W]
  if (b >= 1 && b <= W) {
    if (a >= 2) g += k1 * (c - P(a - 1, b));
    if (a >= 1 && a <= H) g -= k1 * (P(a + 1, b) - c);
  }
  return g;
}

// Nine-point L2 TV loss (ST:184-195) and its gradient (times tv_weight) on the raw image.  One thread per pixel,
// all three channels; block partials of the loss are summed in fixed order by finalize_loss.
__global__ void __launch_bounds__(256)
tv_kernel(const float* __restrict__ img, int H, int W, int row0, TvConst tc, float* __restrict__ gtv,
          float* __restrict__ tv_partials) {
  __shared__ float s_red[8];
  const int y = row0 + blockIdx.y;
  const int x = blockIdx.x * 256 + threadIdx.x;
  float tv_local = 0.f;
  if (x < W) {
    // in-plane offsets once (32-bit), plane base per channel: the 27 loads were 2/3 address arithmetic before
    const int ro[3] = {clampi(y - 1, 0, H - 1) * W, y * W, clampi(y + 1, 0, H - 1) * W};
    const int xs[3] = {clampi(x - 1, 0, W - 1), x, clampi(x + 1, 0, W - 1)};
    const bool hasL = x > 0, hasR = x < W - 1, hasU = y > 0, hasD = y < H - 1;
    const size_t plane_sz = (size_t)H * W;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float* __restrict__ pl = img + c * plane_sz;
      float n[3][3];
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) n[i][j] = __ldg(pl + ro[i] + xs[j]);
      const float ctr = n[1][1];
      // owned loss entries e1[y][x], e2[y][x], e3[y][x], e4[y][x] (+ extra row i=H / col j=W at the far borders)
      const float e1 = n[1][2] - ctr, e2 = n[2][1] - ctr, e3 = ctr - n[0][0], e4 = n[1][0] - n[0][1];
      float l = tc.l1 * (e1 * e1 + e2 * e2) + tc.l3 * (e3 * e3 + e4 * e4);
      if (!hasD) { const float d = ctr - n[1][0]; l += tc.l3 * (d * d + d * d); }
      if (!hasR) { const float d = ctr - n[0][1]; l += tc.l3 * (d * d + d * d); }
      tv_local += l;
      float g;
      if (hasL && hasR && hasU && hasD) {
        g = tc.k1 * (4.f * ctr - n[1][0] - n[1][2] - n[0][1] - n[2][1]) +
            tc.k3 * (4.f * ctr - n[0][0] - n[2][2] - n[0][2] - n[2][0]);
      } else {
        const float* plane = img + (size_t)c * H * W;
        g = 0.f;
        for (int a = (hasU ? y + 1 : 0); a <= (hasD ? y + 1 : H + 1); ++a)
          for (int b = (hasL ? x + 1 : 0); b <= (hasR ? x + 1 : W + 1); ++b)
            g += tv_gpad_slow(plane, H, W, a, b, tc.k1, tc.k3);
      }
      gtv[c * plane_sz + ro[1] + x] = g;
    }
  }
  float sum = warp_sum(tv_local);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += s_red[i];
    tv_partials[blockIdx.y * gridDim.x + blockIdx.x] = t;
  }
}

// conv0 forward weights in the split K layout of conv0_tc.cu: k < 27 the tap (c*3+ky)*3+kx (multiplies the bf16 "hi"
// part of the pixel), 27 <= k < 54 the same tap again (multiplies the residual), rest zero.
__global__ void pack_w0_fwd_kernel(const float* __restrict__ w0, bf16* __restrict__ out) {
  // out[n][k]: k < 27 -> w0[n][k]; 27 <= k < 54 -> w0[n][k-27]; else 0
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 64 * 64) {
    const int n = i >> 6, k = i & 63;
    out[i] = __float2bfloat16(k < 27 ? w0[n * 27 + k] : (k < 54 ? w0[n * 27 + k - 27] : 0.f));
  }
}

// ------------------------------------------------------------------------------------------------ conv0 bwd + Adam
// Persistent warps; one work item = a strip of 32 consecutive pixels of one row.  Lanes are CHANNELS (lane l owns g0
// channels 2l, 2l+1 and keeps their 2 x 27 weights in registers for the whole kernel); the strip is walked pixel by
// pixel with a sliding 3x3 window of coalesced 128-byte loads (the next column is prefetched before the current
// pixel's math), the three image-channel sums are butterfly-reduced and parked on lane p; afterwards lane p applies
// Normalize-backward + TV gradient + Adam + clamp + EMA to pixel p (coalesced).
struct F2 { float x, y; };

__global__ void __launch_bounds__(256)
conv0_bwd_adam_kernel(const bf16* __restrict__ g0, const bool interior_done, const float* __restrict__ w0,
                      const float* __restrict__ gtv, float* __restrict__ img, float* __restrict__ exp_avg,
                      float* __restrict__ exp_avg_sq, float* __restrict__ ema, float* __restrict__ grad_out, int H,
                      int W, const AdamScalars* __restrict__ acp, int apply_update) {
  __shared__ float s_w[64 * 27];
  AdamScalars ac{};
  if (apply_update) ac = *acp;
  for (int i = threadIdx.x; i < 64 * 27; i += 256) s_w[i] = w0[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int strips = (W + 31) >> 5;
  const long total = (long)H * strips;
  const long nwarps = (long)gridDim.x * 8;
  const uint32_t* __restrict__ g32 = reinterpret_cast<const uint32_t*>(g0);

  // wr[tap][c]: weights of this lane's two channels; tap = ky*3+kx
  F2 wr[9][3];
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      wr[t][c].x = s_w[((2 * lane) * 3 + c) * 9 + t];
      wr[t][c].y = s_w[((2 * lane + 1) * 3 + c) * 9 + t];
    }

  // interior_done: the interior pixels were updated by the tensor-core dgrad's epilogue (pixel GEMM mode 3); only
  // strips that contain border pixels are
  // enumerated here: rows 0 and H-1 completely, first and last strip of every other row
  const int side = strips >= 2 ? 2 : 1;
  const long total_items = interior_done ? ((long)2 * strips + (long)(H > 2 ? H - 2 : 0) * side) : total;
  for (long wg = (long)blockIdx.x * 8 + (threadIdx.x >> 5); wg < total_items; wg += nwarps) {
    int y, xs;
    if (!interior_done) {
      y = (int)(wg / strips);
      xs = (int)(wg % strips) * 32;
    } else if (wg < strips) {
      y = 0; xs = (int)wg * 32;
    } else if (wg < 2l * strips) {
      y = H - 1; xs = (int)(wg - strips) * 32;
      if (H == 1) continue;
    } else {
      const long r = wg - 2l * strips;
      y = 1 + (int)(r / side);
      xs = (r % side == 0) ? 0 : (strips - 1) * 32;
    }
    auto ld = [&](int yo, int xo) -> F2 {
      F2 r{0.f, 0.f};
      if (yo >= 0 && yo < H && xo >= 0 && xo < W) {
        const uint32_t u = __ldg(g32 + ((size_t)yo * W + xo) * 32 + lane);
        r.x = bf16lo(u);
        r.y = bf16hi(u);
      }
      return r;
    };
    float keep[3] = {0.f, 0.f, 0.f};
    F2 win[3][3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int cidx = 0; cidx < 3; ++cidx)
        win[r][cidx] = (!interior_done) ? ld(y - 1 + r, xs - 1 + cidx) : F2{0.f, 0.f};
    const bool row_interior = (y > 0) && (y < H - 1);
    const int xe = min(xs + 32, W);
    // interior_done: the zero-pad dgrad of the interior pixels was already computed on the tensor cores
    // (pixel_gemm with conv0's weights zero-padded to 64 output channels); only border pixels (where replicate
    // padding folds extra taps onto the pixel) are evaluated here.
    const bool strip_has_border = !row_interior || xs == 0 || xe == W;
    if (!interior_done || strip_has_border)
    for (int x = xs; x < xe; ++x) {
      if (interior_done && row_interior && x > 0 && x < W - 1) continue;
      F2 nxt[3];
#pragma unroll
      for (int r = 0; r < 3; ++r) nxt[r] = ld(y - 1 + r, x + 2);  // prefetch the next window column
      float acc[3] = {0.f, 0.f, 0.f};
      if (row_interior && x > 0 && x < W - 1) {
        // padded position (y+1, x+1): g0[y+1-ky][x+1-kx] <-> win[2-ky][2-kx]
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
          for (int cidx = 0; cidx < 3; ++cidx) {
            const int t = (2 - r) * 3 + (2 - cidx);
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              acc[c] = fmaf(win[r][cidx].x, wr[t][c].x, acc[c]);
              acc[c] = fmaf(win[r][cidx].y, wr[t][c].y, acc[c]);
            }
          }
      } else {
        // border pixel: sum over the padded positions that replicate-padding folds onto it (warp-uniform branch)
        const int a0 = (y == 0) ? 0 : y + 1, a1 = (y == H - 1) ? H + 1 : y + 1;
        const int b0 = (x == 0) ? 0 : x + 1, b1 = (x == W - 1) ? W + 1 : x + 1;
        for (int a = a0; a <= a1; ++a)
          for (int b = b0; b <= b1; ++b)
#pragma unroll
            for (int ky = 0; ky < 3; ++ky)
#pragma unroll
              for (int kx = 0; kx < 3; ++kx) {
                const F2 v = ld(a - ky, b - kx);
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                  acc[c] = fmaf(v.x, wr[ky * 3 + kx][c].x, acc[c]);
                  acc[c] = fmaf(v.y, wr[ky * 3 + kx][c].y, acc[c]);
                }
              }
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], o);
      }
      if (lane == x - xs) { keep[0] = acc[0]; keep[1] = acc[1]; keep[2] = acc[2]; }
#pragma unroll
      for (int r = 0; r < 3; ++r) { win[r][0] = win[r][1]; win[r][1] = win[r][2]; win[r][2] = nxt[r]; }
    }

    const int x = xs + lane;
    if (x < W) {
      const bool from_tc = interior_done && row_interior && x > 0 && x < W - 1;  // done by the pixel GEMM's mode-3 epilogue
      for (int c = 0; c < 3 && !from_tc; ++c) {
        const size_t idx = ((size_t)c * H + y) * W + x;
        const float g = keep[c] / c_std[c] + (gtv ? gtv[idx] : 0.f);
        if (grad_out) grad_out[idx] = g;
        if (apply_update) {
          float m = exp_avg[idx], v = exp_avg_sq[idx], p = img[idx], e = ema[idx];
          m = m + (g - m) * ac.one_minus_b1;
          v = v * ac.b2 + ac.one_minus_b2 * g * g;
          const float denom = sqrtf(v) * ac.inv_sqrt_bc2 + ac.eps;
          p = p - ac.step_size * (m / denom);
          p = fminf(fmaxf(p, 0.f), 1.f);
          e = e * ac.ema_decay + ac.one_minus_decay * p;
          exp_avg[idx] = m; exp_avg_sq[idx] = v; img[idx] = p; ema[idx] = e;
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ pooling
// (pool forward lives in the epilogue of the conv that feeds it: conv_tc.cu)
// backward through pool + the ReLU that produced the pool input y:  gin = pool_bwd(gout; y) * (y > 0).
// One thread = one 2x2 input window x 8 channels; windows beyond the floor-mode extent write zeros.
template <int POOL>
__global__ void __launch_bounds__(256)
pool_bwd_kernel(const bf16* __restrict__ gout, const bf16* __restrict__ y, bf16* __restrict__ gin, int H, int W,
                int C) {
  const int Ho = H >> 1, Wo = W >> 1, C8 = C >> 3;
  const int Hc = (H + 1) >> 1, Wc = (W + 1) >> 1;  // windows incl. the ragged last row / column
  const long total = (long)Hc * Wc * C8;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c8 = i % C8;
    const long p = i / C8;
    const int xo = p % Wc, yo = p / Wc;
    const bool full = (yo < Ho) && (xo < Wo);
    if (!full) {
      for (int dy = 0; dy < 2; ++dy)
        for (int dx = 0; dx < 2; ++dx) {
          const int yy = 2 * yo + dy, xx = 2 * xo + dx;
          if (yy < H && xx < W && !(yy < 2 * Ho && xx < 2 * Wo))
            *reinterpret_cast<uint4*>(gin + ((size_t)yy * W + xx) * C + c8 * 8) = make_uint4(0, 0, 0, 0);
        }
      // (positions of a ragged window that still belong to a full window do not exist: windows are disjoint)
      continue;
    }
    const size_t ibase = ((size_t)(2 * yo) * W + 2 * xo) * C + c8 * 8;
    const size_t offs[4] = {0, (size_t)C, (size_t)W * C, (size_t)W * C + C};
    uint4 v[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) v[q] = __ldg(reinterpret_cast<const uint4*>(y + ibase + offs[q]));
    const uint4 gv = __ldg(reinterpret_cast<const uint4*>(gout + ((size_t)yo * Wo + xo) * C + c8 * 8));
    uint32_t r[4][4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t gu = reinterpret_cast<const uint32_t*>(&gv)[k];
      float gq[2] = {bf16lo(gu), bf16hi(gu)};
      float xin[2][4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const uint32_t u = reinterpret_cast<const uint32_t*>(&v[q])[k];
        xin[0][q] = bf16lo(u);
        xin[1][q] = bf16hi(u);
      }
      float o[2][4];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (POOL == STB_POOL_MAX) {
          const float m = fmaxf(fmaxf(xin[h][0], xin[h][1]), fmaxf(xin[h][2], xin[h][3]));
          bool taken = false;
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const bool sel = (xin[h][q] == m) && !taken;  // first maximum in scan order wins (ATen)
            taken = taken || sel;
            o[h][q] = (sel && xin[h][q] > 0.f) ? gq[h] : 0.f;
          }
        } else if (POOL == STB_POOL_AVERAGE) {
#pragma unroll
          for (int q = 0; q < 4; ++q) o[h][q] = xin[h][q] > 0.f ? gq[h] * 0.5f : 0.f;
        } else {
          const float s = sqrtf(xin[h][0] * xin[h][0] + xin[h][1] * xin[h][1] + xin[h][2] * xin[h][2] +
                                xin[h][3] * xin[h][3]);
          const float inv = s > 0.f ? 0.78f / s : 0.f;
#pragma unroll
          for (int q = 0; q < 4; ++q) o[h][q] = xin[h][q] > 0.f ? gq[h] * xin[h][q] * inv : 0.f;
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) r[q][k] = pack_bf16x2(o[0][q], o[1][q]);
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)
      *reinterpret_cast<uint4*>(gin + ibase + offs[q]) = make_uint4(r[q][0], r[q][1], r[q][2], r[q][3]);
  }
}

// ------------------------------------------------------------------------------------------------ content SSE
__global__ void __launch_bounds__(256)
sse_kernel(const bf16* __restrict__ a, const bf16* __restrict__ b, long n8, float* __restrict__ partials) {
  __shared__ float s_red[8];
  float s = 0.f;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long)gridDim.x * blockDim.x) {
    const uint4 av = __ldg(reinterpret_cast<const uint4*>(a) + i);
    const uint4 bv = __ldg(reinterpret_cast<const uint4*>(b) + i);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t au = reinterpret_cast<const uint32_t*>(&av)[k], bu = reinterpret_cast<const uint32_t*>(&bv)[k];
      const float d0 = bf16lo(au) - bf16lo(bu), d1 = bf16hi(au) - bf16hi(bu);
      s = fmaf(d0, d0, s);
      s = fmaf(d1, d1, s);
    }
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += s_red[i];
    partials[blockIdx.x] = t;
  }
}

}  // namespace

// ================================================================================================ launchers
int launch_tv(const float* img, int H, int W, int row0, int rows, int H_norm, float tv_weight, float* gtv,
              float* tv_partials, int* n_partials, cudaStream_t s) {
  // rows [row0, row0+rows) of the local H x W image are processed; H_norm is the height the loss means are taken over
  // (the global image height when this image is a band of a taller one)
  TvConst tc{};
  const double n1 = 3.0 * H_norm * W, n3 = 3.0 * (H_norm + 1.0) * (W + 1.0);
  tc.k1 = (float)(tv_weight * 4.0 / (3.0 * n1));
  tc.k3 = (float)(tv_weight * 4.0 / (12.0 * n3));
  tc.l1 = (float)(2.0 / (3.0 * n1));
  tc.l3 = (float)(2.0 / (12.0 * n3));
  dim3 tgrid((W + 255) / 256, rows);
  if (n_partials) *n_partials = tgrid.x * tgrid.y;
  tv_kernel<<<tgrid, 256, 0, s>>>(img, H, W, row0, tc, gtv, tv_partials);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

int pack_weights_conv0_fwd(const float* w0, bf16* out, cudaStream_t s) {
  pack_w0_fwd_kernel<<<16, 256, 0, s>>>(w0, out);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

int launch_conv0_bwd_adam(const bf16* g0, bool interior_done, const float* w0, const float* gtv, float* img,
                          float* exp_avg, float* exp_avg_sq, float* ema, float* grad_out, int H, int W,
                          const AdamScalars* a, int apply_update, cudaStream_t s) {
  const int strips = (W + 31) / 32;
  const long warps = interior_done ? (2l * strips + (long)(H > 2 ? H - 2 : 0) * (strips >= 2 ? 2 : 1)) : (long)H * strips;
  long want = (warps + 7) / 8;
  const long cap = (long)num_sms() * 2 * 4;  // persistent: a few waves of 8-warp CTAs
  const int blocks = (int)(want < cap ? want : cap);
  conv0_bwd_adam_kernel<<<blocks, 256, 0, s>>>(g0, interior_done, w0, gtv, img, exp_avg, exp_avg_sq, ema, grad_out, H, W,
                                               a, apply_update);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

static int grid_for(long work_items, int block) {
  long b = (work_items + block - 1) / block;
  const long cap = (long)num_sms() * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

int launch_pool_bwd(int pooling, const bf16* gout, const bf16* y, bf16* gin, int H, int W, int C, cudaStream_t s) {
  const long total = (long)((H + 1) / 2) * ((W + 1) / 2) * (C / 8);
  const int g = grid_for(total, 256);
  if (pooling == STB_POOL_MAX) pool_bwd_kernel<STB_POOL_MAX><<<g, 256, 0, s>>>(gout, y, gin, H, W, C);
  else if (pooling == STB_POOL_AVERAGE) pool_bwd_kernel<STB_POOL_AVERAGE><<<g, 256, 0, s>>>(gout, y, gin, H, W, C);
  else pool_bwd_kernel<STB_POOL_L2><<<g, 256, 0, s>>>(gout, y, gin, H, W, C);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

// ------------------------------------------------------------------------------------------------ per-scale resize
// F.interpolate(x, (Ho, Wo), mode='bicubic' | 'bilinear') with align_corners=False, antialias=False, as the reference
// uses it for the warm start of a scale: image bicubic + clamp (ST:420), Adam exp_avg bicubic, exp_avg_sq bilinear +
// relu (ST:285-295).  Restates ATen's upsample_bicubic2d / upsample_bilinear2d (UpSample.h: cubic convolution with
// A = -0.75, source index scale * (dst + 0.5) - 0.5, bounded reads; bilinear clamps the source index at 0).
__device__ __forceinline__ void cubic_coeffs(float t, float (&w)[4]) {
  const float A = -0.75f;
  const float x0 = t + 1.f, x1 = t, x2 = 1.f - t, x3 = 2.f - t;
  w[0] = ((A * x0 - 5.f * A) * x0 + 8.f * A) * x0 - 4.f * A;
  w[1] = ((A + 2.f) * x1 - (A + 3.f)) * x1 * x1 + 1.f;
  w[2] = ((A + 2.f) * x2 - (A + 3.f)) * x2 * x2 + 1.f;
  w[3] = ((A * x3 - 5.f * A) * x3 + 8.f * A) * x3 - 4.f * A;
}

// mode: 0 bilinear, 1 bicubic; post: 0 none, 1 relu, 2 clamp to [0, 1]
__global__ void __launch_bounds__(256)
resize_kernel(const float* __restrict__ in, int C, int H, int W, float* __restrict__ out, int Ho, int Wo, float sh,
              float sw, int mode, int post) {
  const long total = (long)C * Ho * Wo;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int xo = (int)(i % Wo);
    const long t2 = i / Wo;
    const int yo = (int)(t2 % Ho), c = (int)(t2 / Ho);
    const float* __restrict__ pl = in + (size_t)c * H * W;
    float v;
    if (mode == 1) {
      const float ry = sh * (yo + 0.5f) - 0.5f, rx = sw * (xo + 0.5f) - 0.5f;
      const float fy = floorf(ry), fx = floorf(rx);
      const int iy = (int)fy, ix = (int)fx;
      float wy[4], wx[4];
      cubic_coeffs(ry - fy, wy);
      cubic_coeffs(rx - fx, wx);
      v = 0.f;
      float rows[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        const float* __restrict__ row = pl + (size_t)clampi(iy - 1 + a, 0, H - 1) * W;
        // ATen: cubic_interp1d(x0, x1, x2, x3, t) = x0*c0 + x1*c1 + x2*c2 + x3*c3, rows first, then columns
        rows[a] = __ldg(row + clampi(ix - 1, 0, W - 1)) * wx[0] + __ldg(row + clampi(ix, 0, W - 1)) * wx[1] +
                  __ldg(row + clampi(ix + 1, 0, W - 1)) * wx[2] + __ldg(row + clampi(ix + 2, 0, W - 1)) * wx[3];
      }
      v = rows[0] * wy[0] + rows[1] * wy[1] + rows[2] * wy[2] + rows[3] * wy[3];
    } else {
      const float ry = fmaxf(sh * (yo + 0.5f) - 0.5f, 0.f), rx = fmaxf(sw * (xo + 0.5f) - 0.5f, 0.f);
      const int y0 = (int)ry, x0 = (int)rx;
      const int y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
      const float ly = ry - y0, lx = rx - x0, hy = 1.f - ly, hx = 1.f - lx;
      v = hy * (hx * __ldg(pl + (size_t)y0 * W + x0) + lx * __ldg(pl + (size_t)y0 * W + x1)) +
          ly * (hx * __ldg(pl + (size_t)y1 * W + x0) + lx * __ldg(pl + (size_t)y1 * W + x1));
    }
    if (post == 1) v = fmaxf(v, 0.f);
    else if (post == 2) v = fminf(fmaxf(v, 0.f), 1.f);
    out[i] = v;
  }
}

int launch_resize(const float* in, int C, int H, int W, float* out, int Ho, int Wo, int mode, int post, cudaStream_t s) {
  STB_CHECK(in && out && C > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0, STB_ERR_INVALID, "resize: bad shape");
  STB_CHECK((mode == 0 || mode == 1) && post >= 0 && post <= 2, STB_ERR_INVALID, "resize: mode=%d post=%d", mode, post);
  // ATen area_pixel_compute_scale with align_corners=False and no explicit scale_factor: input / output, in float
  const float sh = (float)H / (float)Ho, sw = (float)W / (float)Wo;
  resize_kernel<<<grid_for((long)C * Ho * Wo, 256), 256, 0, s>>>(in, C, H, W, out, Ho, Wo, sh, sw, mode, post);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

int preload_image_kernels() {
  cudaFuncAttributes fa;
#define STB_PRELOAD(k) STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(k)))
  STB_PRELOAD(tv_kernel); STB_PRELOAD(pack_w0_fwd_kernel); STB_PRELOAD(conv0_bwd_adam_kernel);
  STB_PRELOAD(pool_bwd_kernel<STB_POOL_MAX>); STB_PRELOAD(pool_bwd_kernel<STB_POOL_AVERAGE>);
  STB_PRELOAD(pool_bwd_kernel<STB_POOL_L2>); STB_PRELOAD(sse_kernel); STB_PRELOAD(resize_kernel);
#undef STB_PRELOAD
  return STB_OK;
}

int launch_sse(const bf16* a, const bf16* b, long n, float* partials, int* n_partials, cudaStream_t s) {
  // the kernel reads 8 elements per 16-byte load: a remainder would be silently left out of the sum
  STB_CHECK(n >= 0 && n % 8 == 0, STB_ERR_INVALID, "sse: n = %ld is not a multiple of 8", n);
  const long n8 = n / 8;
  int g = grid_for(n8, 256);
  if (g > 1024) g = 1024;
  if (n_partials) *n_partials = g;
  sse_kernel<<<g, 256, 0, s>>>(a, b, n8, partials);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

}  // namespace stb
