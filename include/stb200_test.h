/* libstb200_test -- kernel-level test hooks (NOT part of the product library).
 *
 * libstb200_test.so is built from the same translation units as libstb200.so plus csrc/api_test.cu; each hook wraps
 * exactly one internal launcher so that tests/test_gpu_kernels.py can check every kernel against the oracle in
 * isolation.  The product library (include/stb200.h) exports none of these.
 */
#ifndef STB200_TEST_H_
#define STB200_TEST_H_

#include "stb200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* message of the last failing hook on this thread (the test library keeps its own buffer) */
STB_API const char* stb_test_last_error(void);
STB_API int stb_pack_weights(const float* w_oihw, void* out_bf16, int Cout, int Cin, int bwd, void* stream);
STB_API int stb_test_pixel_gemm(int H, int W, int Cin, int Cout, int C2, int mode, const void* A, const void* Bw,
                                const void* A2, int a2_row0, int a2_rows, const void* B2, void* out,
                                const float* bias, const void* mask_src, const void* ctarget, float cscale,
                                int row_lo, int row_hi, void* stream);
/* TV loss partials and gradient (times tv_weight) on rows [row0, row0+rows) of the fp32 [3][H][W] image, with the loss
 * means taken over H_norm rows (a band's global height): gtv [3][H][W] (own rows written), tv_partials
 * ceil(W/256) * rows floats, one per (row, 256-column block), their count in *n_partials. */
STB_API int stb_test_tv(const float* img, int H, int W, int row0, int rows, int H_norm, float tv_weight, float* gtv,
                        float* tv_partials, int* n_partials, void* stream);
/* conv0 forward, out bf16 [H][W][64]; when gtv is not NULL, first stb_test_tv on the whole image */
STB_API int stb_test_conv0_fwd(const float* img, const float* w0, const float* b0, void* out_bf16, int H, int W,
                               float tv_weight, float* gtv, float* tv_partials, int* n_partials, void* stream);
/* conv0 backward as the end of the product's backward pass runs it: the wgmma interior kernel, then the SIMT border
 * kernel.  g0 bf16 [H][W][64], gtv (optional) and grad_out (optional) fp32 [3][H][W].  apply_update: both kernels also
 * take the Adam + clamp + EMA step of Adam step `step` on img / exp_avg / exp_avg_sq / ema (fp32 [3][H][W]). */
STB_API int stb_test_conv0_bwd_adam(const void* g0_bf16, const float* w0, const float* gtv, float* grad_out, int H,
                                    int W, float* img, float* exp_avg, float* exp_avg_sq, float* ema, int64_t step,
                                    float lr, float beta1, float beta2, float eps, float ema_decay, int apply_update,
                                    void* stream);
/* stb_test_conv0_bwd_adam without the update */
STB_API int stb_test_conv0_bwd(const void* g0_bf16, const float* w0, const float* gtv, float* grad_out, int H, int W,
                               void* stream);
/* content SSE partials: sum((a - b)^2) over n bf16 elements (n a multiple of 8, else STB_ERR_INVALID), at most 1024
 * partials, their count in *n_partials. */
STB_API int stb_test_sse(const void* a_bf16, const void* b_bf16, long n, float* partials, int* n_partials,
                         void* stream);
/* conv 3x3 + bias + ReLU with the 2x2 pool fused into its epilogue (the product's only pool-forward path):
 * out [H][W][Cout] and pool_out [H/2][W/2][Cout], both bf16 NHWC. */
STB_API int stb_test_conv_pool(int H, int W, int Cin, int Cout, const void* A, const void* Bw, const float* bias,
                               void* out, void* pool_out, int pooling, void* stream);
/* pool backward (+ ReLU mask of the pool input y): gin [H][W][C] from gout [H/2][W/2][C]. */
STB_API int stb_test_pool_bwd(int pooling, const void* gout, const void* y, void* gin, int H, int W, int C,
                              void* stream);
STB_API int stb_test_gram(const void* F_bf16, long P, int C, float* partials_ws, size_t partials_floats,
                          float* S_raw, float* sums, void* stream);
STB_API size_t stb_test_gram_partials_floats(long P, int C);
STB_API int stb_test_w2(const float* mean_t, const float* srm_t, const float* S_raw, const float* sums, int C,
                        float npix, float weight, void* ws, size_t ws_bytes, float* loss_out, float* gs_out,
                        float* gmu_out, float* csqrt_out, void* stream);
STB_API size_t stb_test_w2_workspace_bytes(void);
/* the five-layer W2 engine as the iteration drives it, one engine kept per workspace: layer l in slot l (C = 64, 128,
 * 256, 512, 512), all five problems through the same grouped rounds.  Arrays of five device pointers per layer: target
 * moments mean_t [C] and srm_t [C][C], statistics S_raw [C][C] and sums [C] (un-normalised sums over npix[l] pixels);
 * npix and weight are five host floats.  build_targets = 0 reuses the targets of the previous call on the same workspace
 * (mean_t and srm_t are then not read).  forward_backward runs n_calls >= 1 times; the outputs (device) are those of the
 * last call: loss_out [5] loss terms, per layer Gs [C][C] fp32 (G + G^T, not divided by npix), gs_bf16 [C][C] (bf16
 * Gs / npix, what the tap-gradient GEMM reads), gmu [C] (divided by npix), mu [C] and csqrt [C][C] = sqrtm(cov_t). */
STB_API int stb_test_w2_layers(const float* const* mean_t, const float* const* srm_t, const float* const* S_raw,
                               const float* const* sums, const float* npix, const float* weight, int build_targets,
                               int n_calls, void* ws, size_t ws_bytes, float* loss_out, float* const* gs_out,
                               void* const* gs_bf16_out, float* const* gmu_out, float* const* mu_out,
                               float* const* csqrt_out, void* stream);
/* the L-BFGS step of stb_iterate_lbfgs alone (closure replaced by a given gradient, grad NULL: the gradient already held
 * by the state): state of stb_lbfgs_state_bytes(H, W) bytes, x / ema fp32 [3*H*W].  pairs_out / t_out (optional; the
 * call then synchronises the stream): history pairs held and step length of the current direction. */
STB_API int stb_test_lbfgs_step(void* state, size_t bytes, int H, int W, float* x, const float* grad, float* ema,
                                float ema_decay, int* pairs_out, float* t_out, void* stream);
/* load every kernel of the test library now (lazy module loading would otherwise synchronise the context at a first
 * launch, which deadlocks against a peer's resident wait kernel): call once before ranks step concurrently */
STB_API int stb_test_preload(void);
/* the banded L-BFGS step of stb_iterate_lbfgs_banded alone, on a context whose comm connection and geometry are set
 * (stb_comm_connect_*, stb_comm_set_geometry): comm phase 0, halo pull into x, grad (this rank's local gradient,
 * [3][h_local][W]) into the mailbox, phase 2, the banded step (seam gather with the neighbours' apron rows when
 * add_seams, cross-rank reductions, own-row update of x / ema [3][h_local][W], outbox fill) and phase 3.  The state
 * has stb_lbfgs_state_bytes(own_rows, W) bytes.  pairs_out / t_out as for stb_test_lbfgs_step. */
STB_API int stb_test_lbfgs_step_banded(stb_ctx* ctx, void* state, size_t bytes, float* x, const float* grad,
                                       float* ema, float ema_decay, int add_seams, int* pairs_out, float* t_out,
                                       void* stream);
/* copy the 3*H*W floats of the gradient the last L-BFGS step consumed out of a state of stb_lbfgs_state_bytes(H, W)
 * bytes (stream-ordered): after stb_iterate_lbfgs the whole-image closure gradient; after stb_iterate_lbfgs_banded
 * (H = own rows) the band's own-row gradient after the seam reduce. */
STB_API int stb_test_lbfgs_gradient(const void* state, size_t bytes, int H, int W, float* out, void* stream);
/* on a context with comm connection and geometry set: *pdl_out = 1 when its exchange kernels launch their successors
 * early (one process per GPU, stb_comm_connect_ipc, or in-process ranks on pairwise distinct devices); the devices of
 * its own mailbox and of its own peer-mapped workspace (-1 when it has none: apron mode) */
STB_API int stb_test_comm_info(stb_ctx* ctx, int* pdl_out, int* mailbox_device_out, int* workspace_device_out);

#ifdef __cplusplus
}
#endif
#endif /* STB200_TEST_H_ */
