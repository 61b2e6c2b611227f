// wgmma / TMA implicit-GEMM for the VGG-19 3x3 convolutions (forward and dgrad) and the per-tap feature-gradient
// GEMM, on NHWC bf16 activations with fp32 accumulation in registers.
//
// Replaces, on the reference's hot path (ST = style_transfer/style_transfer.py of the reference):
//   * ST:86-89  `self.model[i](input)` for the twelve 3x3/zero-pad convs + ReLU(inplace)  (torchvision vgg.py:73-87)
//   * ST:475    `loss.backward()` through those convs (cuDNN/oneDNN backward-data; weights frozen at ST:49, so no
//               wgrad), the ReLU `threshold_backward`, and the Gram/mean backward `dL/dF = F(G+G^T)/N + 1 gmu^T/N`
//               of ST:163-168 which is folded in as extra K-blocks accumulating into the same accumulators.
//
// Tiling: one CTA tile = MT horizontally adjacent sub-tiles of 16x8 output pixels (M = 128 each) x BN output channels
// (BN in {64,128,256}; MT = 2 for BN <= 128 so that every weight stage feeds two sub-tiles), K = 9 taps x Cin.
// Persistent CTAs (one per SM) walk tiles; roles:
//   warp 8      TMA producer (the only active warp of warpgroup 2, which gives its registers to the consumers):
//               per 64-channel chunk it loads three "dx buffers" (18 rows x 8 px x 64 ch, SW128,
//               zero-filled out of bounds = the conv's zero padding); the three dy taps are 1 KiB-aligned row
//               shifts inside a dx buffer, so each activation byte is fetched 3.4x instead of 9x from L2.
//               Weights stream tap by tap through a second ring.  In dgrad (MODE 1) the epilogue operands, the
//               ReLU mask and the content target, follow a tile's K stages through the A ring, one box per
//               64-channel output chunk (or the staged tap operand A2 is kept as the mask when it is the mask).
//   warps 0-7   two consumer warpgroups: warpgroup g owns pixel rows 8g .. 8g+7 of every sub-tile (M = 64), issues
//               its wgmma (bf16 x bf16 -> fp32 registers, one MMA group in flight while the next is issued), then
//               runs the epilogue: bias/ReLU or mask/content -> bf16 -> swizzled smem -> TMA store (+ fused pool).
#include <cstdlib>

#include "kernels.h"
#include "ptx.cuh"

namespace stb {

namespace {

constexpr int TILE_H = 16, TILE_W = 8;           // output pixels per sub-tile = 128 = two wgmma M blocks
constexpr int A_ROWS = TILE_H + 2;               // dx buffer rows (halo above/below)
constexpr int HALF_H = TILE_H / 2;               // pixel rows of one consumer warpgroup
constexpr int STG_BYTES = HALF_H * 1024;         // 64 pixels x 64 ch bf16 staging for the TMA store
constexpr int PSTG_BYTES = (HALF_H / 2) * (TILE_W / 2) * 128;
constexpr int NUM_CONSUMERS = 256;               // two warpgroups
constexpr int NUM_THREADS = NUM_CONSUMERS + 128; // + the producer warpgroup

// MT = horizontally adjacent 16x8 sub-tiles per CTA tile that share every weight stage (halves the L2->smem
// weight traffic per MMA for the narrow-N layers).
template <int BN>
struct Cfg {
  static constexpr int MT = BN == 256 ? 1 : 2;
  static constexpr int NA = 3;
  static constexpr int NB = 4;
  static constexpr int A_PITCH = MT * 1024;                 // bytes per row of 8*MT pixels
  static constexpr int A_STAGE_BYTES = A_ROWS * A_PITCH;    // dx buffer: 18 rows x 8*MT px x 64 ch
  static constexpr int A2_BYTES = TILE_H * A_PITCH;         // centre box for the 1x1 source
  static constexpr int B_STAGE_BYTES = BN * 128;
  static constexpr int OFF_A = 0;
  static constexpr int OFF_B = OFF_A + NA * A_STAGE_BYTES;
  static constexpr int OFF_STG = OFF_B + NB * B_STAGE_BYTES;   // 2 warpgroups x 2 store staging buffers
  static constexpr int OFF_PSTG = OFF_STG + 4 * STG_BYTES;     // 2 x 2 x 2 KiB: pooled 4x4-pixel tile of the fused pool
  static constexpr int OFF_BIAS = OFF_PSTG + 4 * PSTG_BYTES;
  static constexpr int OFF_BAR = OFF_BIAS + 512 * 4;
  static constexpr int NUM_BARS = 2 * NA + 2 * NB;
  static constexpr int SMEM_BYTES = OFF_BAR + NUM_BARS * 8 + 1024;  // + slack for manual 1 KiB alignment
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory per block");
};

struct KParams {
  int H, W, Cin, Cout, C2;
  int tiles_x, tiles_y, n_tiles_n, total_tiles;
  int a2_row0;
  const float* bias;
  const bf16* mask_src;
  const bf16* ctarget;
  float cscale;
  int row_lo, row_hi;
  int pooling;  // MODE 0: -1 = none, else STB_POOL_*: also emit the 2x2-pooled output (tmPool)
  int y_origin; // first output row of the tile grid (row window of a band that computes its own rows only)
  int mask_reuse; // MODE 1: the A2 chunks of a tile are its mask chunks; keep them in the ring for the epilogue
};

template <int BN, int MODE>
__global__ void __launch_bounds__(NUM_THREADS, 1)
pixel_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
                  const __grid_constant__ CUtensorMap tmOut, const __grid_constant__ CUtensorMap tmPool,
                  const __grid_constant__ CUtensorMap tmMask, const __grid_constant__ CUtensorMap tmCt,
                  const KParams p) {
  using C = Cfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::OFF_BAR);
  uint64_t* a_full = bars;
  uint64_t* a_empty = a_full + C::NA;
  uint64_t* b_full = a_empty + C::NA;
  uint64_t* b_empty = b_full + C::NB;
  float* s_bias = reinterpret_cast<float*>(smem + C::OFF_BIAS);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int n_chunks = p.Cin >> 6;
  const int n_chunks2 = p.C2 >> 6;

  // ---- one-time setup
  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmA2);
    tma_prefetch_desc(&tmB2);
    tma_prefetch_desc(&tmOut);
    tma_prefetch_desc(&tmPool);
    tma_prefetch_desc(&tmMask);
    tma_prefetch_desc(&tmCt);
    // empty barriers: one arrival per consumer warp once its wgmma reads of the stage are complete
    for (int i = 0; i < C::NA; ++i) { mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], 8); }
    for (int i = 0; i < C::NB; ++i) { mbar_init(&b_full[i], 1); mbar_init(&b_empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  // Programmatic dependent launch (see launch_cfg): everything above touched no global data and may have run while
  // the previous kernel of the iteration was still draining; its outputs (activations, and in MODE 1 the bias = gmu
  // produced by the W2 chain) are read only from here on.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  for (int i = threadIdx.x; i < p.Cout && i < 512; i += NUM_THREADS) s_bias[i] = p.bias ? p.bias[i] : 0.f;
  __syncthreads();

  if (warp >= 8) {
    // =============================================================== TMA producer
    setmaxnreg_dec<40>();
    if (warp == 8 && lane == 0) {
      int sa = 0, sb = 0;
      uint32_t pa = 0, pb = 0;  // ring phases
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const int tn = tile % p.n_tiles_n;
        const int t2 = tile / p.n_tiles_n;
        const int tx = t2 % p.tiles_x, ty = t2 / p.tiles_x;
        const int y0 = p.y_origin + ty * TILE_H, x0 = tx * TILE_W * C::MT, n0 = tn * BN;
        for (int c = 0; c < n_chunks; ++c) {
          for (int dx = 0; dx < 3; ++dx) {
            mbar_wait(&a_empty[sa], pa ^ 1);
            mbar_expect_tx(&a_full[sa], C::A_STAGE_BYTES);
            tma_load_3d(smem + C::OFF_A + sa * C::A_STAGE_BYTES, &tmA, &a_full[sa], c * 64, x0 + dx - 1, y0 - 1);
            if (++sa == C::NA) { sa = 0; pa ^= 1; }
            for (int dy = 0; dy < 3; ++dy) {
              mbar_wait(&b_empty[sb], pb ^ 1);
              mbar_expect_tx(&b_full[sb], C::B_STAGE_BYTES);
              tma_load_3d(smem + C::OFF_B + sb * C::B_STAGE_BYTES, &tmB, &b_full[sb], c * 64, n0, dy * 3 + dx);
              if (++sb == C::NB) { sb = 0; pb ^= 1; }
            }
          }
        }
        for (int c = 0; c < n_chunks2; ++c) {
          mbar_wait(&a_empty[sa], pa ^ 1);
          mbar_expect_tx(&a_full[sa], C::A2_BYTES);
          tma_load_3d(smem + C::OFF_A + sa * C::A_STAGE_BYTES, &tmA2, &a_full[sa], c * 64, x0, y0 - p.a2_row0);
          if (++sa == C::NA) { sa = 0; pa ^= 1; }
          mbar_wait(&b_empty[sb], pb ^ 1);
          mbar_expect_tx(&b_full[sb], C::B_STAGE_BYTES);
          tma_load_3d(smem + C::OFF_B + sb * C::B_STAGE_BYTES, &tmB2, &b_full[sb], c * 64, n0, 0);
          if (++sb == C::NB) { sb = 0; pb ^= 1; }
        }
        // MODE 1 epilogue operands: per 64-channel output chunk j, the mask box (unless the A2 chunks just loaded
        // are the mask) and on the content layer the content-target box, both at the output tile's coordinates and
        // zero-filled outside the image.  The consumers walk the same sequence: K stages, C2 stages, then these.
        // No deadlock: the slot a chunk needs last held either a K / C2 stage, which the consumers release at the
        // latest with the final MMA wait before the epilogue, or an earlier epilogue chunk, which they release once
        // that chunk is stored; neither release waits on a load issued after it.  Held A2 chunks (mask_reuse) are
        // at most NA - 1 with a content target, so a target chunk always finds a slot that frees.
        if (MODE == 1) {
          for (int j = 0; j < BN / 64; ++j) {
            for (int t = p.mask_reuse ? 1 : 0; t < (p.ctarget != nullptr ? 2 : 1); ++t) {
              mbar_wait(&a_empty[sa], pa ^ 1);
              mbar_expect_tx(&a_full[sa], C::A2_BYTES);
              tma_load_3d(smem + C::OFF_A + sa * C::A_STAGE_BYTES, t ? &tmCt : &tmMask, &a_full[sa], n0 + j * 64, x0,
                          y0);
              if (++sa == C::NA) { sa = 0; pa ^= 1; }
            }
          }
        }
      }
    }
    __syncwarp();
  } else {
    // =============================================================== consumers: MMA + epilogue
    setmaxnreg_inc<232>();
    const int wg = warp >> 2;                      // pixel rows 8 wg .. 8 wg + 7 of every sub-tile
    const int wq = warp & 3;
    const int et = threadIdx.x & 127;              // thread inside the warpgroup
    const uint32_t bar0 = 1 + 3 * wg;              // named barriers of this warpgroup
    const uint32_t a_base0 = smem_u32(smem + C::OFF_A) + wg * HALF_H * C::A_PITCH;
    const uint32_t b_base0 = smem_u32(smem + C::OFF_B);
    const uint32_t a_ring = smem_u32(smem + C::OFF_A);  // MODE 1 epilogue operands are read from here
    int sa = 0, sb = 0;
    uint32_t pa = 0, pb = 0;
    int stg = 0;
    float acc[C::MT][BN / 2];
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const int tn = tile % p.n_tiles_n;
      const int t2 = tile / p.n_tiles_n;
      const int tx = t2 % p.tiles_x, ty = t2 / p.tiles_x;
      const int y0 = p.y_origin + ty * TILE_H + wg * HALF_H, n0 = tn * BN;
      // Stages are released one MMA group late: after issuing group g, wait until only g is in flight, then hand
      // the stages of group g-1 back to the producer.
      int rel_b = -1, rel_a = -1;
      uint32_t accum = 0;  // 0 only for the first weight stage of the tile
      auto release = [&](int keep) {
        if (keep) wgmma_wait<1>(); else wgmma_wait<0>();
        if (lane == 0) {
          if (rel_b >= 0) mbar_arrive(&b_empty[rel_b]);
          if (rel_a >= 0) mbar_arrive(&a_empty[rel_a]);
        }
      };
      auto mma_stage = [&](uint32_t a_stage, int b_slot, int a_release) {
        const uint64_t bd = gmma_desc_k(b_base0 + b_slot * C::B_STAGE_BYTES);
        wgmma_fence();
#pragma unroll
        for (int m = 0; m < C::MT; ++m) {
          const uint64_t ad = gmma_desc_k(a_stage + m * 1024, C::A_PITCH);
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_bf16<0, 0>(acc[m], ad + 2 * k, bd + 2 * k, accum | (k > 0));
        }
        wgmma_commit();
        release(1);
        rel_b = b_slot;
        rel_a = a_release;
        accum = 1;
      };
      for (int c = 0; c < n_chunks; ++c) {
        for (int dx = 0; dx < 3; ++dx) {
          mbar_wait(&a_full[sa], pa);
          const uint32_t a_stage = a_base0 + sa * C::A_STAGE_BYTES;
          for (int dy = 0; dy < 3; ++dy) {
            mbar_wait(&b_full[sb], pb);
            mma_stage(a_stage + dy * C::A_PITCH, sb, dy == 2 ? sa : -1);
            if (++sb == C::NB) { sb = 0; pb ^= 1; }
          }
          if (++sa == C::NA) { sa = 0; pa ^= 1; }
        }
      }
      const bool reuse = MODE == 1 && p.mask_reuse;
      const int sa2 = sa;  // ring slot of A2 chunk 0; with mask_reuse, A2 chunk j stays there as mask chunk j
      for (int c = 0; c < n_chunks2; ++c) {
        mbar_wait(&a_full[sa], pa);
        mbar_wait(&b_full[sb], pb);
        mma_stage(a_base0 + sa * C::A_STAGE_BYTES, sb, reuse ? -1 : sa);
        if (++sb == C::NB) { sb = 0; pb ^= 1; }
        if (++sa == C::NA) { sa = 0; pa ^= 1; }
      }
      release(0);
#pragma unroll
      for (int m = 0; m < C::MT; ++m) wgmma_fence_acc(acc[m]);

      // ---- epilogue: this warpgroup's 8 x 8 pixels of sub-tile m, 64 channels (j) at a time.  MODE 1 walks the
      // chunks j outermost, so that each mask / content-target chunk in the A ring is read by every sub-tile and
      // then released; the other modes walk the sub-tiles outermost.
      const int rr = wq * 16 + (lane >> 2);        // pixel (row) of the first accumulator row held by this thread
      const int cq = 2 * (lane & 3);               // first of the two columns held per 8-column group
      constexpr int NJ = BN / 64;
      int mslot = 0, tslot = 0;                    // MODE 1: A ring slots of chunk j's mask and content target
#pragma unroll
      for (int e = 0; e < C::MT * NJ; ++e) {
        const int m = MODE == 1 ? e % C::MT : e / NJ;
        const int j = MODE == 1 ? e / C::MT : e % NJ;
        const int x0 = (tx * C::MT + m) * TILE_W;
        if (MODE == 1 && m == 0) {
          if (reuse) {
            mslot = (sa2 + j) % C::NA;
          } else {
            mslot = sa;
            mbar_wait(&a_full[sa], pa);
            if (++sa == C::NA) { sa = 0; pa ^= 1; }
          }
          if (p.ctarget != nullptr) {
            tslot = sa;
            mbar_wait(&a_full[sa], pa);
            if (++sa == C::NA) { sa = 0; pa ^= 1; }
          }
        }
        {
          uint8_t* stage = smem + C::OFF_STG + (2 * wg + stg) * STG_BYTES;
          // make sure the TMA store that last read this staging buffer is done, then let everyone write
          if (et == 0) tma_store_wait_read<1>();
          named_bar_sync(bar0, 128);
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const int r = rr + 8 * half;
            const int py = y0 + (r >> 3), px = x0 + (r & 7);
            const bool inb = (py < p.H) && (px < p.W);
            const bool in_rows = (py >= p.row_lo) && (py < p.row_hi);
            const bool has_c = (p.ctarget != nullptr) && in_rows && inb;
            // pixel r of sub-tile m in a [TILE_H][8 MT][64 ch] SW128 box of the A ring (MODE 1 operands)
            const int box_off = ((wg * HALF_H + (r >> 3)) * TILE_W * C::MT + m * TILE_W + (r & 7)) * 128 + cq * 2;
            const uint32_t mrow = a_ring + mslot * C::A_STAGE_BYTES + box_off;
            const uint32_t trow = a_ring + tslot * C::A_STAGE_BYTES + box_off;
#pragma unroll
            for (int q = 0; q < 8; ++q) {
              const int cb = j * 64 + q * 8 + cq;    // column inside the N tile
              float a = acc[m][(j * 8 + q) * 4 + 2 * half], b = acc[m][(j * 8 + q) * 4 + 2 * half + 1];
              uint32_t packed;
              if (MODE == 0) {
                packed = pack_bf16x2(fmaxf(a + s_bias[n0 + cb], 0.f), fmaxf(b + s_bias[n0 + cb + 1], 0.f));
              } else if (MODE == 2) {
                packed = pack_bf16x2(a, b);
              } else {
                const uint32_t yw = lds_u32(mrow + ((q ^ (r & 7)) << 4));
                const float ya = bf16lo(yw), yb = bf16hi(yw);
                if (in_rows) {
                  a += s_bias[n0 + cb];
                  b += s_bias[n0 + cb + 1];
                }
                if (has_c) {
                  const uint32_t tw = lds_u32(trow + ((q ^ (r & 7)) << 4));
                  a += p.cscale * (ya - bf16lo(tw));
                  b += p.cscale * (yb - bf16hi(tw));
                }
                packed = pack_bf16x2(ya > 0.f ? a : 0.f, yb > 0.f ? b : 0.f);
              }
              // swizzled (SW128) staging write: 16-byte chunk q of pixel r lives at chunk (q ^ (r & 7))
              *reinterpret_cast<uint32_t*>(stage + r * 128 + ((q ^ (r & 7)) << 4) + cq * 2) = packed;
            }
          }
          fence_proxy_async_smem();
          named_bar_sync(bar0 + 1, 128);
          if (MODE == 1 && m == C::MT - 1 && lane == 0) {
            // the warp's reads of chunk j's operands are done (they fed the staging writes): hand the slots back
            mbar_arrive(&a_empty[mslot]);
            if (p.ctarget != nullptr) mbar_arrive(&a_empty[tslot]);
          }
          const bool pooled = (MODE == 0) && p.pooling >= 0;
          if (et == 0) {
            tma_store_3d(&tmOut, stage, n0 + j * 64, x0, y0);
            if (!pooled) tma_store_commit();
          }
          if (MODE == 0 && pooled) {
            // fused 2x2 / stride-2 pool (ST:21-22, 41-46) of the 8x8 pixels just staged: 4 x 4 pooled pixels x 8
            // chunks of 8 channels = 128 tasks; windows never straddle tiles (origin and size are even)
            uint8_t* pst = smem + C::OFF_PSTG + (2 * wg + stg) * PSTG_BYTES;
            const int pp = et >> 3, c16 = et & 7;
            const int r0 = ((pp >> 2) * 2) * TILE_W + (pp & 3) * 2;  // top-left source pixel
            uint4 v[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const int rs = r0 + (q >> 1) * TILE_W + (q & 1);
              v[q] = *reinterpret_cast<const uint4*>(stage + rs * 128 + ((c16 ^ (rs & 7)) << 4));
            }
            uint32_t o[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              float lo[4], hi[4];
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                const uint32_t u = reinterpret_cast<const uint32_t*>(&v[q])[k];
                lo[q] = bf16lo(u);
                hi[q] = bf16hi(u);
              }
              float a, b;
              if (p.pooling == STB_POOL_MAX) {
                a = fmaxf(fmaxf(lo[0], lo[1]), fmaxf(lo[2], lo[3]));
                b = fmaxf(fmaxf(hi[0], hi[1]), fmaxf(hi[2], hi[3]));
              } else if (p.pooling == STB_POOL_AVERAGE) {
                a = (lo[0] + lo[1] + lo[2] + lo[3]) * 0.25f * 2.0f;
                b = (hi[0] + hi[1] + hi[2] + hi[3]) * 0.25f * 2.0f;
              } else {
                a = sqrtf(lo[0] * lo[0] + lo[1] * lo[1] + lo[2] * lo[2] + lo[3] * lo[3]) * 0.78f;
                b = sqrtf(hi[0] * hi[0] + hi[1] * hi[1] + hi[2] * hi[2] + hi[3] * hi[3]) * 0.78f;
              }
              o[k] = pack_bf16x2(a, b);
            }
            *reinterpret_cast<uint4*>(pst + pp * 128 + ((c16 ^ (pp & 7)) << 4)) = make_uint4(o[0], o[1], o[2], o[3]);
            fence_proxy_async_smem();
            named_bar_sync(bar0 + 2, 128);
            if (et == 0) {
              tma_store_3d(&tmPool, pst, n0 + j * 64, x0 >> 1, y0 >> 1);
              tma_store_commit();
            }
          }
          stg ^= 1;
        }
      }
    }
    if (et == 0) tma_store_wait_all0();
  }
}

template <int BN, int MODE>
int launch_cfg(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmA2, const CUtensorMap& tmB2,
               const CUtensorMap& tmOut, const CUtensorMap& tmPool, const CUtensorMap& tmMask, const CUtensorMap& tmCt,
               const KParams& kp, cudaStream_t stream) {
  using C = Cfg<BN>;
  auto kern = pixel_gemm_kernel<BN, MODE>;
  STB_TRY(ensure_dynamic_smem(reinterpret_cast<const void*>(kern), C::SMEM_BYTES));
  int grid = kp.total_tiles < num_sms() ? kp.total_tiles : num_sms();
  // launched with programmatic stream serialization: the CTAs may become resident (and run their prologue) as soon
  // as the previous kernel's CTAs retire; griddepcontrol.wait in the kernel orders the data accesses
  static const bool pdl = [] { const char* e = getenv("STB_PDL"); return !(e && e[0] == '0'); }();
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(NUM_THREADS);
  cfg.dynamicSmemBytes = C::SMEM_BYTES;
  cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  STB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, tmA, tmB, tmA2, tmB2, tmOut, tmPool, tmMask, tmCt, kp));
  return STB_OK;
}

}  // namespace

int launch_pixel_gemm(const PixelGemmArgs& a, cudaStream_t stream) {
  STB_CHECK(a.H > 0 && a.W > 0, STB_ERR_INVALID, "pixel_gemm: bad spatial size %dx%d", a.H, a.W);
  STB_CHECK(a.Cout % 64 == 0 && a.Cout <= 512, STB_ERR_INVALID, "pixel_gemm: Cout=%d", a.Cout);
  STB_CHECK(a.Cin % 64 == 0 && a.C2 % 64 == 0 && (a.Cin + a.C2) > 0, STB_ERR_INVALID, "pixel_gemm: Cin=%d C2=%d",
            a.Cin, a.C2);
  const int BN = a.Cout >= 256 ? 256 : a.Cout;
  KParams kp;
  kp.H = a.H; kp.W = a.W; kp.Cin = a.Cin; kp.Cout = a.Cout; kp.C2 = a.C2;
  const int MT = BN == 256 ? 1 : 2;  // must match Cfg<BN>::MT
  const int tile_w = TILE_W * MT;
  kp.tiles_x = (a.W + tile_w - 1) / tile_w;
  // row window [y_origin, y_origin + y_rows): a band in per-layer-halo mode computes its own rows only
  const int y_rows = a.y_rows > 0 ? a.y_rows : a.H - a.y_origin;
  STB_CHECK(a.y_origin >= 0 && y_rows > 0 && a.y_origin + y_rows <= a.H, STB_ERR_INVALID,
            "pixel_gemm: row window %d+%d of %d", a.y_origin, y_rows, a.H);
  STB_CHECK(a.pool_out == nullptr || a.y_origin % 2 == 0, STB_ERR_INVALID, "pixel_gemm: fused pool needs an even row origin");
  kp.y_origin = a.y_origin;
  kp.tiles_y = (y_rows + TILE_H - 1) / TILE_H;
  kp.n_tiles_n = a.Cout / BN;
  kp.total_tiles = kp.tiles_x * kp.tiles_y * kp.n_tiles_n;
  kp.a2_row0 = a.a2_row0;
  kp.bias = a.bias; kp.mask_src = a.mask_src; kp.ctarget = a.ctarget; kp.cscale = a.cscale;
  kp.row_lo = a.row_lo; kp.row_hi = a.row_hi;
  STB_CHECK(a.mode >= 0 && a.mode <= 2, STB_ERR_INVALID, "pixel_gemm: mode=%d", a.mode);
  if (a.mode == 1) STB_CHECK(a.mask_src != nullptr, STB_ERR_INVALID, "pixel_gemm: bwd needs mask_src");

  // The tap operand is the mask itself on the 64- and 128-channel style taps (A2 = the tap's activation, which the
  // dgrad masks): its chunks, staged in the A ring for the C2 GEMM, then serve as the mask chunks.  Only where A2
  // holds the mask at every row the tiles store: a band computing its aprons (y_origin below the A2 window) sees A2
  // zero-filled there, so it streams the mask; and the held chunks must leave a ring slot for the content target.
  const int a2_rows = a.a2_rows > 0 ? a.a2_rows : a.H;
  const int y_end = a.y_origin + kp.tiles_y * TILE_H < a.H ? a.y_origin + kp.tiles_y * TILE_H : a.H;
  kp.mask_reuse = a.mode == 1 && a.C2 == a.Cout && BN == a.Cout && a.A2 != nullptr &&
                  a.A2 == a.mask_src + static_cast<size_t>(a.a2_row0) * a.W * a.C2 &&
                  a.C2 / 64 + (a.ctarget != nullptr) <= Cfg<64>::NA && a.a2_row0 <= a.y_origin &&
                  a.a2_row0 + a2_rows >= y_end;
  static_assert(Cfg<64>::NA == Cfg<128>::NA, "one A ring depth for the reusable widths");

  CUtensorMap tmA, tmB, tmA2, tmB2, tmOut, tmPool, tmMask, tmCt;
  const uint64_t W = a.W, H = a.H;
  // output first; unused maps alias it so that every descriptor handed to the kernel is valid
  STB_TRY(make_tmap_bf16_3d(&tmOut, a.out, a.Cout, W, H, a.Cout * 2ull, W * a.Cout * 2ull, 64, TILE_W, HALF_H));
  tmA = tmB = tmA2 = tmB2 = tmPool = tmMask = tmCt = tmOut;
  if (a.mode == 1) {
    // epilogue operands, [H][W][Cout], loaded per output tile and 64-channel chunk in the A2 box geometry
    STB_TRY(make_tmap_bf16_3d(&tmMask, a.mask_src, a.Cout, W, H, a.Cout * 2ull, W * a.Cout * 2ull, 64, tile_w, TILE_H));
    if (a.ctarget != nullptr)
      STB_TRY(make_tmap_bf16_3d(&tmCt, a.ctarget, a.Cout, W, H, a.Cout * 2ull, W * a.Cout * 2ull, 64, tile_w, TILE_H));
  }
  kp.pooling = -1;
  if (a.pool_out != nullptr) {
    STB_CHECK(a.mode == 0 && a.pooling >= 0 && a.pooling <= 2 && H >= 2 && W >= 2, STB_ERR_INVALID,
              "pixel_gemm: fused pool needs mode 0 and a valid pooling");
    kp.pooling = a.pooling;
    STB_TRY(make_tmap_bf16_3d(&tmPool, a.pool_out, a.Cout, W / 2, H / 2, a.Cout * 2ull, (W / 2) * a.Cout * 2ull, 64,
                              TILE_W / 2, HALF_H / 2));
  }
  if (a.Cin > 0) {
    STB_TRY(make_tmap_bf16_3d(&tmA, a.A, a.Cin, W, H, a.Cin * 2ull, W * a.Cin * 2ull, 64, tile_w, A_ROWS));
    STB_TRY(make_tmap_bf16_3d(&tmB, a.Bw, a.Cin, a.Cout, 9, a.Cin * 2ull, (uint64_t)a.Cout * a.Cin * 2ull, 64, BN, 1));
  }
  if (a.C2 > 0) {
    const int rows = a.a2_rows > 0 ? a.a2_rows : a.H;
    STB_TRY(make_tmap_bf16_3d(&tmA2, a.A2, a.C2, W, rows, a.C2 * 2ull, W * a.C2 * 2ull, 64, tile_w, TILE_H));
    STB_TRY(make_tmap_bf16_3d(&tmB2, a.B2, a.C2, a.Cout, 1, a.C2 * 2ull, (uint64_t)a.Cout * a.C2 * 2ull, 64, BN, 1));
  }
  if (a.mode == 0) {
    if (BN == 256) return launch_cfg<256, 0>(tmA, tmB, tmA2, tmB2, tmOut, tmPool, tmMask, tmCt, kp, stream);
    if (BN == 128) return launch_cfg<128, 0>(tmA, tmB, tmA2, tmB2, tmOut, tmPool, tmMask, tmCt, kp, stream);
    return launch_cfg<64, 0>(tmA, tmB, tmA2, tmB2, tmOut, tmPool, tmMask, tmCt, kp, stream);
  } else if (a.mode == 1) {
    if (BN == 256) return launch_cfg<256, 1>(tmA, tmB, tmA2, tmB2, tmOut, tmPool, tmMask, tmCt, kp, stream);
    if (BN == 128) return launch_cfg<128, 1>(tmA, tmB, tmA2, tmB2, tmOut, tmPool, tmMask, tmCt, kp, stream);
    return launch_cfg<64, 1>(tmA, tmB, tmA2, tmB2, tmOut, tmPool, tmMask, tmCt, kp, stream);
  } else {
    if (BN == 256) return launch_cfg<256, 2>(tmA, tmB, tmA2, tmB2, tmOut, tmPool, tmMask, tmCt, kp, stream);
    if (BN == 128) return launch_cfg<128, 2>(tmA, tmB, tmA2, tmB2, tmOut, tmPool, tmMask, tmCt, kp, stream);
    return launch_cfg<64, 2>(tmA, tmB, tmA2, tmB2, tmOut, tmPool, tmMask, tmCt, kp, stream);
  }
}

// ---------------------------------------------------------------- weight packing
namespace {
__global__ void pack_w_kernel(const float* __restrict__ w, bf16* __restrict__ out, int Cout, int Cin, int bwd) {
  // fwd: out[tap][co][ci] = w[co][ci][tap];  bwd: out[tap][ci][co] = w[co][ci][8 - tap]
  const long total = 9l * Cout * Cin;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int k = i % (bwd ? Cout : Cin);
    const long t = i / (bwd ? Cout : Cin);
    const int n = t % (bwd ? Cin : Cout);
    const int tap = t / (bwd ? Cin : Cout);
    const int co = bwd ? k : n, ci = bwd ? n : k;
    const int src_tap = bwd ? 8 - tap : tap;
    out[i] = __float2bfloat16(w[((long)co * Cin + ci) * 9 + src_tap]);
  }
}
}  // namespace


// Force the (lazily loaded) kernels of this file into the context: a first launch may need a context-wide
// synchronisation, which must not happen while a peer-wait kernel of the tiled path is resident (comm.cu).
int preload_conv_kernels() {
  cudaFuncAttributes fa;
#define STB_PRELOAD(k) STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(k)))
  STB_PRELOAD((pixel_gemm_kernel<64, 0>)); STB_PRELOAD((pixel_gemm_kernel<64, 1>)); STB_PRELOAD((pixel_gemm_kernel<64, 2>));
  STB_PRELOAD((pixel_gemm_kernel<128, 0>)); STB_PRELOAD((pixel_gemm_kernel<128, 1>)); STB_PRELOAD((pixel_gemm_kernel<128, 2>));
  STB_PRELOAD((pixel_gemm_kernel<256, 0>)); STB_PRELOAD((pixel_gemm_kernel<256, 1>)); STB_PRELOAD((pixel_gemm_kernel<256, 2>));
  STB_PRELOAD(pack_w_kernel);
#undef STB_PRELOAD
  return STB_OK;
}

int pack_weights_fwd(const float* w, bf16* out, int Cout, int Cin, cudaStream_t s) {
  pack_w_kernel<<<256, 256, 0, s>>>(w, out, Cout, Cin, 0);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}
int pack_weights_bwd(const float* w, bf16* out, int Cout, int Cin, cudaStream_t s) {
  pack_w_kernel<<<256, 256, 0, s>>>(w, out, Cout, Cin, 1);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

}  // namespace stb
