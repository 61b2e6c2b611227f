// Source images on the device: Pillow's `Image.resize((Wo, Ho), Image.BICUBIC)` of an 8-bit RGB image, bit for bit, fused
// with TF.to_tensor (ST:417, 437 resize the content and style images on the CPU once per scale).
//
// Pillow resamples 8-bit images in fixed point, one axis at a time: an output sample is
//   clip8((2^21 + sum_j source[first + j] * k[j]) >> 22)      (int32, arithmetic shift, clamp to 0..255)
// over the `count` taps of its window, k the bicubic weights with 22 fractional bits.  The horizontal pass runs first and
// its result is stored as uint8 before the vertical pass reads it; a pass whose axis keeps its size is skipped.  The
// tables (k, first, count) are built by the caller in double, as Pillow builds them (style_transfer.resample_coeffs):
// the kernels below are integer arithmetic only, so they reproduce Pillow exactly whatever the order of the taps.
//   resample_h_kernel : uint8 [Hs][Ws][3] -> uint8 [n_rows][Wo][3], only the source rows the requested output rows need
//   resample_v_kernel : that (or the source itself, when the width is kept) -> fp32 planar [3][rows][Wo], value u8 / 255
#include "kernels.h"

namespace stb {

namespace {

constexpr int RS_TX = 64, RS_TY = 4;      // CTA tile: 64 output columns x 4 rows (256 threads), both kernels
constexpr int RS_SMEM_MAX = 96 * 1024;    // staged source segments of the horizontal pass; two CTAs per SM

__device__ __forceinline__ int clip8(int acc) { return min(max((acc + (1 << 21)) >> 22, 0), 255); }

// One CTA = RS_TX neighbouring outputs of RS_TY source rows.  The windows of neighbouring outputs overlap by all but
// in / out samples, so the CTA first copies the source span of its outputs, [lo, hi) of each of its rows, into shared
// memory with aligned 32-bit loads, and the taps read it from there.  A span that does not fit (a reduction by more than
// ~120 : 1) is read from global memory directly by the same loop.  Bounds from the table are clamped to the source row:
// a table that does not belong to these sizes gives wrong pixels, never a read outside the image.
__global__ void __launch_bounds__(RS_TX * RS_TY)
resample_h_kernel(const uint8_t* __restrict__ src, long src_bytes, int Ws, int Wo, int src_row0, int n_rows,
                  const int32_t* __restrict__ kx, const int32_t* __restrict__ bx, int ksize, int seg_cap,
                  uint8_t* __restrict__ tmp) {
  extern __shared__ __align__(16) uint8_t s_seg[];
  __shared__ int s_lo, s_hi;
  const int tiles_x = (Wo + RS_TX - 1) / RS_TX;
  const int tx = threadIdx.x % RS_TX, ty = threadIdx.x / RS_TX;
  const int x = (int)(blockIdx.x % tiles_x) * RS_TX + tx;
  const int r0 = (int)(blockIdx.x / tiles_x) * RS_TY;   // first row of this CTA in tmp; source row src_row0 + r0

  int first = 0, count = 0;
  if (x < Wo) {
    first = min(max(bx[2 * x], 0), Ws);
    count = min(max(bx[2 * x + 1], 0), min(ksize, Ws - first));
  }
  if (threadIdx.x == 0) { s_lo = Ws; s_hi = 0; }
  __syncthreads();
  if (ty == 0 && count > 0) { atomicMin(&s_lo, first); atomicMax(&s_hi, first + count); }
  __syncthreads();
  const int lo = s_lo, span_bytes = max(s_hi - lo, 0) * 3;
  const bool staged = span_bytes + 8 <= seg_cap;   // 3 bytes of misalignment in front, the last word rounded up
  const uintptr_t src_begin = reinterpret_cast<uintptr_t>(src), src_end = src_begin + src_bytes;

  if (staged) {
    for (int rr = 0; rr < RS_TY && r0 + rr < n_rows; ++rr) {
      const uintptr_t g0 = src_begin + ((size_t)(src_row0 + r0 + rr) * Ws + lo) * 3;
      const uintptr_t base = g0 & ~(uintptr_t)3;
      const int words = (int)(g0 - base + span_bytes + 3) >> 2;
      uint32_t* __restrict__ dst = reinterpret_cast<uint32_t*>(s_seg + (size_t)rr * seg_cap);
      for (int w = threadIdx.x; w < words; w += RS_TX * RS_TY) {
        const uintptr_t a = base + 4 * (uintptr_t)w;
        uint32_t v = 0;
        if (a >= src_begin && a + 4 <= src_end) {
          v = __ldg(reinterpret_cast<const uint32_t*>(a));
        } else {   // the first or last word of the image: only the bytes inside it
          for (int b = 0; b < 4; ++b)
            if (a + b >= src_begin && a + b < src_end) v |= (uint32_t)__ldg(reinterpret_cast<const uint8_t*>(a + b)) << (8 * b);
        }
        dst[w] = v;
      }
    }
    __syncthreads();
  }

  const int r = r0 + ty;
  if (x >= Wo || r >= n_rows) return;
  const size_t g_row = (size_t)(src_row0 + r) * Ws * 3;
  const uint8_t* p = src + g_row + (size_t)first * 3;
  if (staged && count > 0)   // the staged copy of this row starts at the 32-bit word that holds sample `lo`
    p = s_seg + (size_t)ty * seg_cap + ((src_begin + g_row + (size_t)lo * 3) & 3) + (size_t)(first - lo) * 3;
  const int32_t* __restrict__ k = kx + (size_t)x * ksize;
  int a0 = 0, a1 = 0, a2 = 0;
  for (int j = 0; j < count; ++j) {
    const int kj = __ldg(k + j);
    a0 += (int)p[3 * j] * kj;
    a1 += (int)p[3 * j + 1] * kj;
    a2 += (int)p[3 * j + 2] * kj;
  }
  uint8_t* __restrict__ o = tmp + ((size_t)r * Wo + x) * 3;
  o[0] = (uint8_t)clip8(a0);
  o[1] = (uint8_t)clip8(a1);
  o[2] = (uint8_t)clip8(a2);
}

// One thread = one output pixel, three channels; a warp reads 96 consecutive bytes of an input row per tap (the weight is
// the same for the whole warp) and writes 128 consecutive bytes per plane.  `in` is [in_rows][Wo][3] and holds rows
// in_row0 .. in_row0 + in_rows of the horizontally resampled image; ky == nullptr: the height is kept, row y is copied.
// inv255: 1.0f / 255.0f, the factor torch multiplies by for `uint8_tensor.to(float32).div_(255)` on the device.
__global__ void __launch_bounds__(RS_TX * RS_TY)
resample_v_kernel(const uint8_t* __restrict__ in, int in_row0, int in_rows, int Wo, int row0, int rows,
                  const int32_t* __restrict__ ky, const int32_t* __restrict__ by, int ksize, float inv255,
                  float* __restrict__ out) {
  const int tiles_x = (Wo + RS_TX - 1) / RS_TX;
  const int x = (int)(blockIdx.x % tiles_x) * RS_TX + threadIdx.x % RS_TX;
  const int yl = (int)(blockIdx.x / tiles_x) * RS_TY + threadIdx.x / RS_TX;   // row of the output window
  if (x >= Wo || yl >= rows) return;
  const int y = row0 + yl;
  int v0, v1, v2;
  if (ky != nullptr) {
    const int first = min(max(__ldg(by + 2 * y), in_row0), in_row0 + in_rows);
    const int count = min(max(__ldg(by + 2 * y + 1), 0), min(ksize, in_row0 + in_rows - first));
    const uint8_t* __restrict__ p = in + ((size_t)(first - in_row0) * Wo + x) * 3;
    const int32_t* __restrict__ k = ky + (size_t)y * ksize;
    const size_t stride = (size_t)Wo * 3;
    int a0 = 0, a1 = 0, a2 = 0;
    for (int j = 0; j < count; ++j, p += stride) {
      const int kj = __ldg(k + j);
      a0 += (int)__ldg(p) * kj;
      a1 += (int)__ldg(p + 1) * kj;
      a2 += (int)__ldg(p + 2) * kj;
    }
    v0 = clip8(a0); v1 = clip8(a1); v2 = clip8(a2);
  } else {
    const uint8_t* __restrict__ p = in + ((size_t)(y - in_row0) * Wo + x) * 3;
    v0 = __ldg(p); v1 = __ldg(p + 1); v2 = __ldg(p + 2);
  }
  const size_t plane = (size_t)rows * Wo, i = (size_t)yl * Wo + x;
  out[i] = __fmul_rn((float)v0, inv255);
  out[plane + i] = __fmul_rn((float)v1, inv255);
  out[2 * plane + i] = __fmul_rn((float)v2, inv255);
}

// Input samples [lo, hi) that output samples o0 .. o1 of an axis read: Pillow's window bounds (the same expressions as
// resample_coeffs, whose tables the kernels are given), or the samples themselves on an axis that keeps its size.
void axis_window(int n_in, int n_out, int o0, int o1, int* lo, int* hi) {
  if (n_in == n_out) { *lo = o0; *hi = o1 + 1; return; }
  const double scale = (double)n_in / n_out, support = 2.0 * (scale > 1.0 ? scale : 1.0);
  const int a = (int)((o0 + 0.5) * scale - support + 0.5), b = (int)((o1 + 0.5) * scale + support + 0.5);
  *lo = a < 0 ? 0 : a;
  *hi = b > n_in ? n_in : b;
}

int check_window(int Hs, int Ws, int Ho, int Wo, int row0, int rows) {
  STB_CHECK(Hs >= 1 && Ws >= 1 && Ho >= 1 && Wo >= 1, STB_ERR_INVALID, "resample: bad size %d x %d -> %d x %d", Ws, Hs,
            Wo, Ho);
  STB_CHECK(row0 >= 0 && rows >= 1 && rows <= Ho - row0, STB_ERR_INVALID,
            "resample: rows [%d, %d + %d) are not inside the %d output rows", row0, row0, rows, Ho);
  return STB_OK;
}

}  // namespace

int resample_tmp_bytes(int Hs, int Ws, int Ho, int Wo, int row0, int rows, size_t* bytes) {
  STB_CHECK(bytes != nullptr, STB_ERR_INVALID, "resample: null argument");
  STB_TRY(check_window(Hs, Ws, Ho, Wo, row0, rows));
  int lo, hi;
  axis_window(Hs, Ho, row0, row0 + rows - 1, &lo, &hi);
  *bytes = Ws == Wo ? 0 : (size_t)(hi - lo) * Wo * 3;   // a kept width needs no horizontal pass
  return STB_OK;
}

int launch_resample_rgb8(const uint8_t* src, int Hs, int Ws, int Ho, int Wo, int row0, int rows, const int32_t* kx,
                         const int32_t* bx, int ksize_x, const int32_t* ky, const int32_t* by, int ksize_y, void* tmp,
                         size_t tmp_bytes, float* out, cudaStream_t s) {
  STB_CHECK(src && out, STB_ERR_INVALID, "resample: null image pointer");
  size_t need = 0;
  STB_TRY(resample_tmp_bytes(Hs, Ws, Ho, Wo, row0, rows, &need));
  const bool horiz = Ws != Wo, vert = Hs != Ho;
  STB_CHECK(!horiz || (kx && bx && ksize_x >= 1), STB_ERR_INVALID, "resample: no tables for the horizontal pass");
  STB_CHECK(!vert || (ky && by && ksize_y >= 1), STB_ERR_INVALID, "resample: no tables for the vertical pass");
  STB_CHECK(need == 0 || (tmp && tmp_bytes >= need), STB_ERR_INVALID, "resample: scratch of %zu bytes, %zu needed",
            tmp ? tmp_bytes : (size_t)0, need);
  int lo, hi;
  axis_window(Hs, Ho, row0, row0 + rows - 1, &lo, &hi);
  const long tiles_x = (Wo + RS_TX - 1) / RS_TX;
  STB_CHECK(tiles_x * ((Hs + RS_TY - 1) / RS_TY) < (1l << 31) && tiles_x * ((rows + RS_TY - 1) / RS_TY) < (1l << 31),
            STB_ERR_INVALID, "resample: %d x %d -> %d x %d is too large", Ws, Hs, Wo, Ho);
  const uint8_t* in = src;
  int in_row0 = 0, in_rows = Hs;
  if (horiz) {
    // source span of RS_TX neighbouring outputs: their centres are (RS_TX - 1) * scale apart, a window reaches `support`
    // to either side, and each end moves by less than one sample when it is truncated
    const double scale = (double)Ws / Wo, support = 2.0 * (scale > 1.0 ? scale : 1.0);
    double span = (RS_TX - 1) * scale + 2.0 * support + 2.0;
    if (span > Ws) span = Ws;
    long cap = ((long)span * 3 + 8 + 3) & ~3l;
    if (cap * RS_TY > RS_SMEM_MAX) cap = 0;   // read the taps from global memory
    const int seg_cap = (int)cap;
    STB_TRY(ensure_dynamic_smem(reinterpret_cast<const void*>(resample_h_kernel), RS_SMEM_MAX));
    const unsigned blocks = (unsigned)(tiles_x * ((hi - lo + RS_TY - 1) / RS_TY));
    resample_h_kernel<<<blocks, RS_TX * RS_TY, (size_t)seg_cap * RS_TY, s>>>(
        src, (long)Hs * Ws * 3, Ws, Wo, lo, hi - lo, kx, bx, ksize_x, seg_cap, static_cast<uint8_t*>(tmp));
    STB_CUDA_CHECK(cudaGetLastError());
    in = static_cast<const uint8_t*>(tmp);
    in_row0 = lo;
    in_rows = hi - lo;
  }
  const unsigned blocks = (unsigned)(tiles_x * ((rows + RS_TY - 1) / RS_TY));
  resample_v_kernel<<<blocks, RS_TX * RS_TY, 0, s>>>(in, in_row0, in_rows, Wo, row0, rows, vert ? ky : nullptr, by,
                                                    ksize_y, 1.0f / 255.0f, out);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

int preload_resample_kernels() {
  cudaFuncAttributes fa;
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(resample_h_kernel)));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(resample_v_kernel)));
  return STB_OK;
}

}  // namespace stb
