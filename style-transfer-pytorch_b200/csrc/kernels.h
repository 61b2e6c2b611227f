// Internal launcher prototypes (all stream-ordered, no host sync).  Layout conventions:
//   activations / feature gradients : NHWC bf16, i.e. [H][W][C] with C contiguous ("pixel-major")
//   image, Adam moments, EMA        : the reference's own NCHW fp32 [1,3,H,W] torch tensors
//   conv weights                    : packed bf16 [tap][N][K] (K contiguous), see pack_weights_*
#pragma once
#include <vector>

#include "host_util.h"

namespace stb {

typedef __nv_bfloat16 bf16;

// ---------------------------------------------------------------- wgmma implicit-GEMM "pixel GEMM"
// out[p][n] = epilogue( sum_{tap,k} A[p + off(tap)][k] * B[tap][n][k]  +  sum_k A2[p][k] * B2[n][k] )
//   fwd  (mode 0): + bias[n], ReLU                       (VGG conv 3x3 + bias + ReLU; ST:86-89 -> torchvision vgg.py)
//   bwd  (mode 1): + bias[n] (rows in [row_lo,row_hi)), + cscale*(y - ctarget), * (y > 0)
//                                                         (conv dgrad + tap-gradient GEMM + ReLU mask; autograd of ST:475)
//   lin  (mode 2): none (dgrad whose consumer is the pool backward)
struct PixelGemmArgs {
  int H = 0, W = 0;
  int Cin = 0;    // main 3x3 source channels (multiple of 64) or 0
  int Cout = 0;   // output channels (multiple of 64)
  int C2 = 0;     // second (1x1) source channels (multiple of 64) or 0
  int mode = 0;
  const bf16* A = nullptr;        // [H][W][Cin]
  const bf16* Bw = nullptr;       // [9][Cout][Cin]
  const bf16* A2 = nullptr;       // [H2][W][C2]  (rows a2_row0 .. a2_row0+H2 of the output grid)
  int a2_row0 = 0, a2_rows = 0;   // row window in which the second source contributes (multi-GPU own rows)
  const bf16* B2 = nullptr;       // [Cout][C2]
  bf16* out = nullptr;            // [H][W][Cout]
  const float* bias = nullptr;    // [Cout] or null
  const bf16* mask_src = nullptr; // bwd: [H][W][Cout]
  const bf16* ctarget = nullptr;  // bwd, optional: [H][W][Cout]
  float cscale = 0.f;
  int row_lo = 0, row_hi = 1 << 30;  // rows where bias (bwd) / content term apply
  int y_origin = 0, y_rows = 0;   // output row window (0 rows = all): tiles start at y_origin, inputs outside are halo rows
  bf16* pool_out = nullptr;       // fwd, optional: [H/2][W/2][Cout], the 2x2/stride-2 pool of `out` (floor mode)
  int pooling = -1;               // STB_POOL_* of pool_out
};
int launch_pixel_gemm(const PixelGemmArgs& a, cudaStream_t stream);

// fp32 OIHW [Cout][Cin][3][3] -> bf16 [9][Cout][Cin] (fwd) / [9][Cin][Cout] with 180-degree rotated taps (dgrad)
int pack_weights_fwd(const float* w, bf16* out, int Cout, int Cin, cudaStream_t s);
int pack_weights_bwd(const float* w, bf16* out, int Cout, int Cin, cudaStream_t s);

// ---------------------------------------------------------------- image-space / pooling kernels (image_ops.cu)
struct AdamScalars {  // torch/optim/adam.py:413-546 scalars, evaluated on the host in double like torch does
  float one_minus_b1, b2, one_minus_b2, step_size, inv_sqrt_bc2, eps, ema_decay, one_minus_decay;
};
// the scalars of Adam step `step` (1-based): on the device by adam_scalars_kernel, on the host by the test library's
// stb_test_conv0_bwd_adam (each side with its own pow / sqrt)
__host__ __device__ inline AdamScalars make_adam_scalars(int64_t step, float lr, float beta1, float beta2,
                                                         float adam_eps, float ema_decay) {
  AdamScalars as{};
  const double bc1 = 1.0 - pow((double)beta1, (double)step);
  const double bc2 = 1.0 - pow((double)beta2, (double)step);
  as.one_minus_b1 = 1.f - beta1; as.b2 = beta2; as.one_minus_b2 = 1.f - beta2;
  as.step_size = (float)((double)lr / bc1);
  as.inv_sqrt_bc2 = (float)(1.0 / sqrt(bc2));
  as.eps = adam_eps; as.ema_decay = ema_decay; as.one_minus_decay = 1.f - ema_decay;
  return as;
}
// Adam + clamp to [0, 1] + EMA of one element: moments m, v, image p, EMA e; g is the gradient.  Every Adam update
// (conv0's fused epilogues, the band seam) runs this one copy, so they all round alike.
__device__ __forceinline__ void adam_element(const AdamScalars& ac, float g, float& m, float& v, float& p, float& e) {
  m = m + (g - m) * ac.one_minus_b1;
  v = v * ac.b2 + ac.one_minus_b2 * g * g;
  const float denom = sqrtf(v) * ac.inv_sqrt_bc2 + ac.eps;
  p = p - ac.step_size * (m / denom);
  p = fminf(fmaxf(p, 0.f), 1.f);
  e = e * ac.ema_decay + ac.one_minus_decay * p;
}
// TV loss partials + gradient (times tv_weight) on the raw image; weights of the tensor-core conv0 in its split
// K layout (27 hi taps, 27 lo residuals, 10 zeros).
int launch_tv(const float* img, int H, int W, int row0, int rows, int H_norm, float tv_weight, float* gtv,
              float* tv_partials, int* n_partials, cudaStream_t s);
int pack_weights_conv0_fwd(const float* w0, bf16* out, cudaStream_t s);
// conv0 forward on wgmma with the im2col rows built in shared memory (conv0_tc.cu); out: bf16 NHWC [H][W][64]
int launch_conv0_fwd(const float* img, const bf16* w0_packed, const float* bias, bf16* out, int H, int W,
                     cudaStream_t s);
// g0: masked gradient w.r.t. conv0's pre-activation, bf16 NHWC [H][W][64].  interior_done: the interior pixels were
// already updated by the tensor-core dgrad (pixel GEMM mode 3); only the border pixels, where the adjoint of the
// replicate pad folds extra taps onto the pixel, are evaluated here.  grad_out (optional) receives d loss/d image.
int launch_conv0_bwd_adam(const bf16* g0, bool interior_done, const float* w0, const float* gtv, float* img,
                          float* exp_avg, float* exp_avg_sq, float* ema, float* grad_out, int H, int W,
                          const AdamScalars* d_adam, int apply_update, cudaStream_t s);  // d_adam: DEVICE pointer
// conv0 backward on wgmma (conv0_tc.cu): weights fp32 OIHW [64][3][3][3] -> bf16 [32 (ky,kx,c; 27 used)][64 co];
// the kernel updates the interior pixels (1x1 GEMM + col2im in smem + Normalize bwd + TV grad + Adam + clamp + EMA)
int pack_weights_conv0_bwd(const float* w0, bf16* out, cudaStream_t s);
int launch_conv0_bwd_interior(const bf16* g0, const bf16* w0q, const float* gtv, float* img, float* exp_avg,
                              float* exp_avg_sq, float* ema, float* grad_out, int H, int W, const AdamScalars* d_adam,
                              int apply_update, cudaStream_t s);
int launch_pool_bwd(int pooling, const bf16* gout, const bf16* y, bf16* gin, int H, int W, int C, cudaStream_t s);
int launch_sse(const bf16* a, const bf16* b, long n, float* partials, int* n_partials, cudaStream_t s);
// F.interpolate(align_corners=False) on fp32 [C][H][W] planes: mode 0 bilinear / 1 bicubic; post 0 none / 1 relu /
// 2 clamp to [0,1]  (warm start of a scale, ST:285-295, 420)
int launch_resize(const float* in, int C, int H, int W, float* out, int Ho, int Wo, int mode, int post, cudaStream_t s);
// fp32 [3][H][W] / denom, clamped to [0,1], quantised to interleaved [H][W][3]: kind 0 uint8, 1 uint16 (stb_snapshot)
int launch_snapshot(const float* value, int H, int W, double denom, int kind, void* out, cudaStream_t s);

// ---------------------------------------------------------------- source images (resample.cu)
// out fp32 planar [3][rows][Wo] = rows [row0, row0 + rows) of to_tensor(Image.resize((Wo, Ho), BICUBIC)) of the uint8 RGB
// image src[Hs][Ws][3] (stb_resample_rgb8); tmp: resample_tmp_bytes(...) bytes for the horizontal pass's result
int resample_tmp_bytes(int Hs, int Ws, int Ho, int Wo, int row0, int rows, size_t* bytes);
int launch_resample_rgb8(const uint8_t* src, int Hs, int Ws, int Ho, int Wo, int row0, int rows, const int32_t* kx,
                         const int32_t* bx, int ksize_x, const int32_t* ky, const int32_t* by, int ksize_y, void* tmp,
                         size_t tmp_bytes, float* out, cudaStream_t s);
int preload_resample_kernels();

// ---------------------------------------------------------------- L-BFGS step on the device (lbfgs.cu)
// torch.optim.LBFGS.step (lr 1, max_iter 1, history STB_LBFGS_HISTORY, no line search) + EMA on n-float vectors; the
// state is one caller-owned block of lbfgs_state_bytes(n) bytes (256-byte aligned), reset by launch_lbfgs_reset.
size_t lbfgs_state_bytes(long n);
float* lbfgs_grad_buffer(void* state, long n);  // where the gradient of the step must be written
int launch_lbfgs_reset(void* state, cudaStream_t s);
// fixed launch sequence (capturable): the step on x, then ema = ema * decay + (1 - decay) * x
int launch_lbfgs_step(void* state, long n, float* x, float* ema, float ema_decay, cudaStream_t s);
// synchronous read of the pair count and the step length t of the current direction (test hook)
int lbfgs_read_info(const void* state, int* pairs, float* t, cudaStream_t s);
struct CommDev;
// Banded step of a tiled iteration (a rank's own rows only; the state holds n = 3 * own_rows * W floats).  Runs after
// comm phase 2, with this rank's local gradient [3][h_local][W] in its mailbox: seam gather into the compact g, then the
// launch sequence of launch_lbfgs_step with a one-block cross-rank reduction (lbfgs_xreduce_kernel) after pass 0 and
// after every round, so that every rank holds the same global scalars; the final pass updates the own rows of the local
// image x / ema [3][h_local][W] and fills the outboxes.
constexpr int LBFGS_XREDUCES = 2 * STB_LBFGS_HISTORY + 2;   // pass 0 + 21 rounds
int launch_lbfgs_step_banded(void* state, const CommDev& c, float* x, float* ema, float ema_decay, int add_seams,
                             cudaStream_t s);
int preload_lbfgs_kernels();

// ---------------------------------------------------------------- Gram / channel sums on wgmma (gram_tc.cu)
int gram_num_splits(long P, int C);
size_t gram_partials_floats(long P, int C);
size_t gram_max_partials_floats(int C);  // bound of gram_partials_floats over every P (what the workspace reserves)
// F: [P][C] bf16 pixel-major.  S_raw [C][C] and sums [C] receive the un-normalised sums over the P pixels.
int launch_gram(const bf16* F, long P, int C, float* partials_ws, size_t partials_capacity_floats, float* S_raw,
                float* sums, cudaStream_t stream);

// ---------------------------------------------------------------- W2 style loss engine (w2_tc.cu)
// Every matrix of the chain is 4 fp32 planes of n*n floats: hi, lo (3xTF32 split) and the same for its transpose.
struct TcProb {  // D = alpha * A * B + gamma * I, all n x n row-major; a matrix = planes hi, lo, hi^T, lo^T
  const CUtensorMap* amap;  // [hi, lo] tensor maps of A with 128-row boxes (device memory)
  const CUtensorMap* bmap;  // [hi, lo] tensor maps of B^T with 64-row boxes
  const CUtensorMap* dmap;  // [hi, lo] tensor maps of D for the TMA stores (128-row boxes)
  float* D;
  float* red_out;  // optional: per-tile {sum of squares, trace} of D
  int n;
  float alpha, gamma;
  int write_t;  // also write the planes of D^T (D is later used as a right factor)
  int in_half;  // operands are fp16 plane pairs (hi, lo * 2^11) instead of TF32 pairs: kind::f16 MMAs, half the bytes
  int out_half; // D is written as an fp16 plane pair
};
// a round holds up to two problems per layer; six layers of 64, 128, 256, 512, 512, 512 channels give 214 tiles
constexpr int W2_MAX_LAYERS = 6, W2_MAX_PROBS = 2 * W2_MAX_LAYERS, W2_MAX_TILES = 216, W2_TRACE_WORDS = 8 * 128;
struct W2Round {  // one grouped GEMM step of all layers; lives in device memory, walked by w2_chain_kernel
  int n_tiles, n_probs;
  TcProb probs[W2_MAX_PROBS];
  uint32_t tiles[W2_MAX_TILES];  // prob << 16 | tile row << 8 | tile col
};
enum { W2S_NORM_A = 0, W2S_TR_COV = 1, W2S_TR_COV_T = 2, W2S_MEAN_DIFF = 3, W2S_LOSS = 4, W2S_QSCALE = 5 };
struct W2Layer {
  int n;            // channels
  float eps;        // 1e-4 (ST:152)
  float weight;     // style layer weight (ST:320-322)
  float npix;       // number of pixels the raw sums were taken over (global count under multi-GPU)
  float *S_raw, *sums;                 // inputs: reduced raw second moment [n][n] and channel sums [n]
  float *mu, *cov;                     // current mean / covariance (cov: plane pair)
  float *mean_t, *srm_t, *cov_t, *P;   // target: mean, second raw moment, covariance (pair), sqrtm(cov_t) (pair)
  float *M, *X, *Y[2], *Z[2], *T;      // forward chain (plane pairs)
  float *A[2], *Q[2], *E, *X1, *X23, *U, *Gc, *Gs;  // backward chain (pairs; Gs, X1 single planes)
  float* Qf;        // the final q of the Lyapunov iteration as a TF32 plane pair (U = P^T q runs on the TF32 path)
  float* gc_alpha;  // device address of the alpha of this layer's Gc GEMM (w2_fwd_finish patches it: 0.5 / q scale)
  float* gmu_bias;  // out: (d loss / d mean) / npix              -> per-channel bias of the tap-gradient GEMM
  bf16* gs_bf16;    // out: (G + G^T) / npix as bf16 [n][n]       -> B operand of the tap-gradient GEMM
  float* scal;      // W2S_* scalars
  float* red;       // reduction partials {sum of squares, trace} x 128
};
struct W2Engine {
  int n_layers = 0;
  W2Layer host_layers[W2_MAX_LAYERS];
  W2Layer* d_layers = nullptr;
  CUtensorMap* d_maps = nullptr;
  W2Round* d_rounds = nullptr;        // device copy of `rounds` (the chain kernel walks it)
  unsigned* d_grid_counter = nullptr; // grid barrier of the chain kernel (zeroed before every launch)
  unsigned long long* d_trace = nullptr;  // STB_W2_TRACE=1: 8 %globaltimer stamps per round written by CTA 0
  std::vector<W2Round> rounds;
  int r_target_begin = 0, r_target_end = 0, r_fwd_begin = 0, r_fwd_ns_begin = 0, r_fwd_end = 0, r_bwd_begin = 0,
      r_bwd_end = 0, gc_round = 0;
  static size_t layer_floats(int n);
  static size_t workspace_bytes();
  // n_layers (0..W2_MAX_LAYERS) problems of n_per_layer[l] channels each, in {64, 128, 256, 512}
  int init(void* ws, size_t bytes, int n_layers, const int* n_per_layer);
  int upload_layers(cudaStream_t s);           // after editing host_layers (weights, npix, S_raw/sums pointers)
  int run_rounds(int r0, int r1, cudaStream_t s);
  int build_targets(cudaStream_t s);            // mean_t/srm_t -> cov_t, P = sqrtm_ns(cov_t)   (ST:152-160)
  int forward_backward(float* loss_terms, cudaStream_t s);  // S_raw/sums -> loss_terms[n_layers], gs_bf16, gmu_bias
  static int read_matrix(float* dst, const float* pair, int n, cudaStream_t s);  // dst = hi + lo (test hook)
};

// ---------------------------------------------------------------- multi-GPU peer-memory exchange (comm.cu)
constexpr int COMM_APRON = 80;       // halo rows on each interior side of a band (receptive-field radius of relu5_1)
constexpr int COMM_MAX_RANKS = 8;
// u64 slots at the head of a mailbox (one 128-byte line each; the head is 4096 bytes, zeroed by stb_comm_reset).
// COMM_XVAL: the banded L-BFGS step's cross-rank reductions, [2 (iteration parity)][LBFGS_XREDUCES][4] doubles.
enum { COMM_ITER = 0, COMM_FLAG_STATS = 16, COMM_FLAG_GRAD = 32, COMM_FLAG_HALO = 48, COMM_ERR = 64, COMM_PROG = 80,
       COMM_FLAG_XRED = 96, COMM_XVAL = 112 };
struct CommDev {  // passed by value to the exchange kernels
  int rank, world;
  uint8_t* mbox[COMM_MAX_RANKS];   // mailbox of every rank as mapped into THIS process (own one included)
  size_t off_stats[2], off_grad, off_outbox[2];
  int W, h_local, own0, own_rows;           // this band: local image height, first own row, number of own rows
  int up_h_local, up_apron_row0, dn_h_local;  // neighbours' local heights; first bottom-apron row of the upper band
  uint8_t* ws[COMM_MAX_RANKS];                // per-layer-halo mode: every rank's WORKSPACE as mapped here (else null)
  unsigned long long timeout_ns;              // a peer wait longer than this traps instead of hanging
  int pdl;  // 1: exchange kernels may launch their successor early (programmatic dependent launch).  Only when every
            // rank has its own GPU: with several ranks on ONE device (test emulation) an early-resident conv grid that
            // waits for an exchange kernel, which waits for another rank, would starve that rank of SMs.
};
size_t comm_mailbox_bytes(size_t stats_floats, int max_h_local, int max_W, size_t off[5]);
int launch_comm_phase(const CommDev& c, int phase, cudaStream_t s);   // 0 begin, 1 stats, 2 grad, 3 end
int launch_halo_pull(const CommDev& c, float* img, cudaStream_t s);
int launch_stats_allreduce(const CommDev& c, float* stats, size_t n_floats, cudaStream_t s);
int launch_adam_seam(const CommDev& c, float* img, float* exp_avg, float* exp_avg_sq, float* ema,
                     const AdamScalars* d_adam, int add_seams, cudaStream_t s);
// g[3][own_rows][W] = own rows of the mailbox gradient (+ the neighbours' apron rows when add_seams)
int launch_lbfgs_seam_gather(const CommDev& c, float* g, int add_seams, cudaStream_t s);
// per-layer halo exchange: publish progress stamp `seq` of this iteration, wait for the neighbours' same stamp, then copy
// one boundary row (row_bytes) from each neighbour's buffer into this rank's halo rows.  Pointers are absolute (peer
// workspaces are mapped); a null source / destination skips that side.
struct HaloRowArgs {
  const uint8_t* src_up;   // upper neighbour's LAST own row of the tensor
  uint8_t* dst_up;         // my row just above my first own row
  const uint8_t* src_dn;   // lower neighbour's FIRST own row
  uint8_t* dst_dn;         // my row just below my last own row
  size_t row_bytes;
  int seq;
};
int launch_halo_rows(const CommDev& c, const HaloRowArgs& a, cudaStream_t s);

// the comm connection of a context when it is connected and has a geometry, else null (test hooks)
const CommDev* ctx_comm(const stb_ctx* ctx);

// force every kernel of the library into the context (lazy module loading may otherwise synchronise the context at
// a first launch, which deadlocks against a resident peer-wait kernel)
int comm_preload();
int preload_conv_kernels();
int preload_gram_kernels();
int preload_w2_kernels();
int preload_conv0_kernels();
int preload_image_kernels();

}  // namespace stb
