/* libstb200 -- C ABI of the H100-native stylize() hot path.
 *
 * The reference (crowsonkb/style-transfer-pytorch) has no FFI layer: its hot path is the Python loop body of
 * StyleTransfer.stylize() (style_transfer/style_transfer.py:472-486, "ST" below).  This header is the seam a
 * maintainer binds directly beneath that class (see INTEGRATION.md for the ctypes stub).  Every entry point is
 * stream-ordered, borrows caller-owned device pointers (torch tensors) for the duration of the call, never throws,
 * never exits; it returns 0 on success or a negative STB_ERR_* code, with stb_last_error() giving the message.
 *
 * Data layouts
 *   image / exp_avg / exp_avg_sq / ema : fp32 NCHW [1,3,H,W]   (exactly the reference's tensors, ST:420-421, 457-463)
 *   activations inside the workspace   : bf16 NHWC
 *   style statistics                   : fp32, mean [C], second raw moment [C,C] row-major (ST:163-168)
 */
#ifndef STB200_H_
#define STB200_H_

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define STB_API __attribute__((visibility("default")))
#else
#define STB_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define STB_OK 0
#define STB_ERR_INVALID (-1)   /* bad argument              -> ValueError   (ST:83, ST:331, ST:373, ST:405, ST:467) */
#define STB_ERR_CUDA (-2)      /* CUDA runtime/driver error -> RuntimeError                                          */
#define STB_ERR_WORKSPACE (-3) /* workspace unbound / small -> RuntimeError                                          */
#define STB_ERR_STATE (-4)     /* call-order violation      -> RuntimeError                                          */

#define STB_POOL_MAX 0     /* nn.MaxPool2d(2)                 ST:21 */
#define STB_POOL_AVERAGE 1 /* Scale(nn.AvgPool2d(2), 2.0)     ST:21-22, 41-46 */
#define STB_POOL_L2 2      /* Scale(nn.LPPool2d(2, 2), 0.78)  ST:21-22, 41-46 */

#define STB_NUM_CONVS 13      /* VGG-19 features[:30]: convs at 0,2,5,7,10,12,14,16,19,21,23,25,28 */
#define STB_NUM_STYLE_TAPS 5  /* ReLU outputs 1,6,11,20,29 (ST:317): the default style layers */
#define STB_NUM_TAPS 6        /* ReLU outputs 1,6,11,20,22,29: the taps of the reference model (ST:324) */
#define STB_MAX_LOSS_TERMS 14 /* total + 6 content + 6 style + TV */

typedef struct stb_ctx stb_ctx;

/* Thread-local message for the last failing call on this thread. */
STB_API const char* stb_last_error(void);

/* ------------------------------------------------------------------ context (replaces ST:324-333)
 * conv_w[i] / conv_b[i]: DEVICE fp32 pointers to the 13 conv weights (OIHW) and biases of vgg19().features[:30] in
 * layer order.  The context packs them once into its own bf16 tensor-core layouts (the only memory it owns). */
STB_API int stb_ctx_create(int device, int pooling, const float* const* conv_w, const float* const* conv_b,
                           void* stream, stb_ctx** out);
STB_API void stb_ctx_destroy(stb_ctx* ctx);

/* ------------------------------------------------------------------ workspace (caller/torch owns all memory;
 * mirrors the reference's per-scale allocations, ST:413-414, 469-470).  Bytes needed to run any entry point on
 * an H x W image; bind a 1 KiB-aligned device block of at least the maximum over the sizes that will be used.
 * Rebinding invalidates the targets. */
STB_API int stb_workspace_bytes(stb_ctx* ctx, int H, int W, size_t* bytes);
STB_API int stb_bind_workspace(stb_ctx* ctx, void* ptr, size_t bytes, void* stream);

/* ------------------------------------------------------------------ layer table (StyleTransfer.content_layers,
 * style_layers; ST:316-317, 365-455).  content_layers: 1 to 6 taps, style_layers: 0 to 6 taps, each from the six
 * ReLU taps {1, 6, 11, 20, 22, 29} of the reference model, no tap twice in one list (a tap may be in both lists).
 * The order of each list is the order of the per-layer arrays of the calls below and of the loss terms.
 * STB_ERR_INVALID for anything else, before any state changes.  The call resets the graphs, invalidates the targets
 * and re-lays the W2 engine out over the style taps; stb_workspace_bytes then reflects the table (activations are
 * kept through the deepest configured conv only; a content target at tap 1 is H x W x 64 bf16, 537 MB at 2048^2).
 * An iteration runs the forward through the conv of the deepest configured tap and starts the backward there.
 * A context that never calls it has the default table: content [22], style [1, 6, 11, 20, 29]. */
STB_API int stb_set_layers(stb_ctx* ctx, int n_content, const int* content_layers, int n_style, const int* style_layers);

/* ------------------------------------------------------------------ target extraction (no-grad VGG forward)
 * stb_style_stats      = self.model(style, layers=style_layers) + StyleLossW2.get_target   (ST:440-443, 163-168)
 *                        mean_out[l]: [C_l] fp32, srm_out[l]: [C_l,C_l] fp32, l over taps 1,6,11,20,29
 * stb_content_features = self.model(content, layers=[22])[22]                               (ST:425)
 *                        target_out: bf16 NHWC [H/8][W/8][512]
 * `img` is a device fp32 NCHW [1,3,H,W] tensor with values in [0,1]; H,W >= 16 (ST:61-69, 82-83). */
STB_API int stb_style_stats(stb_ctx* ctx, const float* img, int H, int W, float* const* mean_out,
                            float* const* srm_out, void* stream);
STB_API int stb_content_features(stb_ctx* ctx, const float* img, int H, int W, void* target_out_bf16, void* stream);
/* Under the context's layer table: stb_style_stats fills one (mean, srm) pair per style tap, in table order (nothing
 * without style taps); stb_content_features_ex one bf16 NHWC target [h_l][w_l][C_l] per content tap.
 * stb_content_features / stb_set_targets are the default table's calls (STB_ERR_STATE under any other table). */
STB_API int stb_content_features_ex(stb_ctx* ctx, const float* img, int H, int W, void* const* targets_out,
                                    void* stream);

/* ------------------------------------------------------------------ per-scale loss state (ST:426-455)
 * mean_t/srm_t: the style-weight-blended target moments (ST:443-450); the library forms cov = srm - mean mean^T
 * + eps I and cov_sqrt = sqrtm_ns(cov, 12) (ST:152-160).  style_w: the five layer weights (ST:320-322). */
STB_API int stb_set_targets(stb_ctx* ctx, int H, int W, const void* content_target_bf16, float content_weight,
                            const float* const* mean_t, const float* const* srm_t, const float* style_w,
                            float tv_weight, float eps, void* stream);
/* Per-layer arrays in table order: content_targets / content_w (content_weight / len(content_layers), ST:366) per
 * content tap; mean_t / srm_t / style_w per style tap. */
STB_API int stb_set_targets_ex(stb_ctx* ctx, int H, int W, const void* const* content_targets, const float* content_w,
                               const float* const* mean_t, const float* const* srm_t, const float* style_w,
                               float tv_weight, float eps, void* stream);
/* The loss-term vector of the last iteration, [total, content terms..., style terms..., tv] in table order: 2 +
 * n_content + n_style <= STB_MAX_LOSS_TERMS floats ({loss, content, style1..5, tv} for the default table).
 * *n_terms receives the count; min(count, capacity) floats are copied, stream-ordered, into host memory `out`.
 * loss_out_host8 of the iteration calls receives the first eight words of this vector. */
STB_API int stb_loss_terms(stb_ctx* ctx, float* out, int capacity, int* n_terms, void* stream);

/* ------------------------------------------------------------------ THE HOT PATH: one iteration of ST:480-486
 * forward + losses + backward + Adam(lr, betas, eps; bias correction with `step` = 1-based count carried across
 * scales, ST:287-295/461-462) + clamp_(0,1) + EMA value update, all stream-ordered with no host sync.
 * loss_out_host8 (pinned host, optional) receives asynchronously {loss, content, style1..5, tv} of the
 * PRE-update image (what `opt.step(closure)` returns, ST:481). */
STB_API int stb_iterate(stb_ctx* ctx, float* img, float* exp_avg, float* exp_avg_sq, float* ema, int64_t step,
                        float lr, float beta1, float beta2, float adam_eps, float ema_decay, float* loss_out_host8,
                        void* stream);
/* closure-only variant (apply_update = 0): loss and d loss/d image (grad_out fp32 NCHW), e.g. for a host optimizer. */
STB_API int stb_iterate_ex(stb_ctx* ctx, float* img, float* exp_avg, float* exp_avg_sq, float* ema, int64_t step,
                           float lr, float beta1, float beta2, float adam_eps, float ema_decay, int apply_update,
                           float* grad_out, float* loss_out_host8, void* stream);

/* ------------------------------------------------------------------ optimizer='lbfgs' (ST:464-465) on the device
 * One iteration = closure (forward, losses, backward) + torch.optim.LBFGS.step with lr = 1, max_iter = 1,
 * history_size = STB_LBFGS_HISTORY, tolerance_grad = 1e-7, tolerance_change = 1e-9 and no line search, followed by
 * ema = ema * decay + (1 - decay) * img.  There is no clamp on this path (ST:482-485), as in the reference.
 * The optimizer state (history ring, g, g_prev, d, scalars) is ONE caller-owned device block of
 * stb_lbfgs_state_bytes(H, W) bytes, 256-byte aligned (~25 x 3HW floats: ~1.26 GB at 2048^2).  The reference builds
 * a fresh optim.LBFGS per scale: call stb_lbfgs_reset once per scale, before its first iteration.
 * stb_iterate_lbfgs runs on the targets' H x W (stb_set_targets) and needs a context without a band (stb_iterate_lbfgs_banded runs a band).  It is one
 * stream-ordered sequence, replayed as a CUDA graph, with no host sync; the loss of the PRE-step image goes to the loss
 * ring (stb_set_loss_ring) under the stamp `step`, the running iteration count of the whole stylize() call, and
 * optionally to loss_out_host8. */
#define STB_LBFGS_HISTORY 10
STB_API int stb_lbfgs_state_bytes(int H, int W, size_t* bytes);
STB_API int stb_lbfgs_reset(void* state, int H, int W, void* stream);
STB_API int stb_iterate_lbfgs(stb_ctx* ctx, float* img, float* ema, void* state, size_t state_bytes, int64_t step,
                              float ema_decay, float* loss_out_host8, void* stream);

/* ------------------------------------------------------------------ spatial tiling across GPUs (SURVEY.md 8e)
 * A context may work on a horizontal band (plus halo aprons) of a taller image: H passed to the other calls is the
 * LOCAL height, rows [own_row0, own_row0+own_rows) (multiples of 16) are the band's own rows, H_global the full
 * height.  Only own rows enter the statistics, losses and tap gradients.  An iteration of a band is one call of
 * stb_iterate_banded (or stb_iterate_lbfgs_banded), with the exchanges between the ranks inside it (below).  Where the
 * ranks cannot map each other's memory, the host drives the same iteration in phases instead:
 *   stb_iterate_fwd  -> all-reduce(sum) of the stats block over the ranks (one NCCL call, ~2.4 MB)
 *   stb_iterate_bwd  -> grad_out = d loss / d (local image) incl. contributions to the halo rows
 *   [exchange + add the halo rows of grad_out with the neighbouring bands]
 *   stb_adam_update  on the own rows, then refresh the halo rows of the image from the neighbours.
 * With a band set, stb_style_stats returns RAW sums over the own rows (all-reduce, then divide by the global count). */
STB_API int stb_set_band(stb_ctx* ctx, int enabled, int H_global, int own_row0, int own_rows);
STB_API int stb_stats_block(stb_ctx* ctx, int H, int W, float** dev_ptr, size_t* n_floats);
STB_API int stb_iterate_fwd(stb_ctx* ctx, const float* img, void* stream);
STB_API int stb_iterate_bwd(stb_ctx* ctx, float* img, float* grad_out, float* loss_out_host8, void* stream);
STB_API int stb_adam_update(float* img, const float* grad, float* exp_avg, float* exp_avg_sq, float* ema, int H, int W,
                            int row0, int rows, int64_t step, float lr, float beta1, float beta2, float adam_eps,
                            float ema_decay, void* stream);

/* ------------------------------------------------------------------ sync-free loss read-back (ST:487-493)
 * host_ring: PINNED host memory, slots x 16 floats (NULL switches it off).  Each updating iteration stores its loss-term
 * vector (stb_loss_terms) into slot (step % slots), term k at word k for k < 8 and at word k + 1 above, and then the
 * step as the slot's int32 stamp (word 8), from the loss kernel itself,
 * BEFORE the backward pass starts: the host polls the stamp -- the per-iteration callback needs no stream sync and
 * overlaps the rest of the iteration. */
STB_API int stb_set_loss_ring(stb_ctx* ctx, float* host_ring, int slots);

/* ------------------------------------------------------------------ per-scale warm start (ST:285-295, 420)
 * out[1,C,Ho,Wo] = F.interpolate(in[1,C,H,W], (Ho,Wo), mode, align_corners=False) on the device, fp32.
 * mode: 0 bilinear, 1 bicubic (A = -0.75).  post: 0 none, 1 relu (exp_avg_sq, ST:293), 2 clamp to [0,1] (image). */
STB_API int stb_resize(const float* in, int C, int H, int W, float* out, int Ho, int Wo, int mode, int post,
                       void* stream);

/* ------------------------------------------------------------------ source images (ST:417, 437)
 * out[1,3,rows,Wo] fp32 planar = rows [row0, row0 + rows) of TF.to_tensor(Image.resize((Wo, Ho), Image.BICUBIC)) of the
 * 8-bit RGB image src[Hs][Ws][3] (device, interleaved), bit for bit: Pillow's two fixed-point passes (horizontal first,
 * its result stored as uint8; a pass whose axis keeps its size is skipped) and value = u8 * (1.0f / 255.0f), which is
 * what torch computes for `.to(float32).div_(255)` on the device.  A row window costs the source rows it needs only.
 *   kx / ky : device int32 [Wo][ksize_x] / [Ho][ksize_y], the weights of every output sample with 22 fractional bits
 *   bx / by : device int32 [Wo][2] / [Ho][2], (first input sample, number of taps) of every output sample
 *             an output sample is clip8((2^21 + sum_j in[first + j] * k[j]) >> 22); the tables are Pillow's, built by
 *             the caller in double (style_transfer.resample_coeffs); those of an axis that keeps its size are ignored
 *   tmp     : caller-owned scratch of stb_resample_tmp_bytes(...) bytes (0 when Ws == Wo: may be NULL then)
 * The bounds are clamped to the image, so tables of other sizes give wrong pixels but no access outside src / tmp.
 * STB_ERR_INVALID, with nothing launched, for a null src / out / needed table, a size < 1, a window that is empty or
 * not inside [0, Ho), or a scratch that is missing or too small. */
STB_API int stb_resample_tmp_bytes(int Hs, int Ws, int Ho, int Wo, int row0, int rows, size_t* bytes);
STB_API int stb_resample_rgb8(const uint8_t* src, int Hs, int Ws, int Ho, int Wo, int row0, int rows,
                              const int32_t* kx, const int32_t* bx, int ksize_x, const int32_t* ky, const int32_t* by,
                              int ksize_y, void* tmp, size_t tmp_bytes, float* out, void* stream);

/* ------------------------------------------------------------------ image snapshot (get_image, periodic saves)
 * value: planar fp32 [3][H][W] (the EMA's storage); out: interleaved [H][W][3], written in one pass on `stream`.
 *   kind 0: uint8  = trunc(clamp(value / denom, 0, 1) * 255)       (to_pil_image: mul(255).byte())
 *   kind 1: uint16 = round_half_even(clamp(value / denom, 0, 1) * 65535)   (np.uint16(np.round(x * 65535)))
 * The division is a multiply by 1 / denom, computed in double and rounded to float, as torch computes
 * `tensor / python_float` on CUDA, so the result is bit-identical to those expressions on EMA.get().  denom = 1 - accum, or 1 for an image that is already
 * bias-corrected.  STB_ERR_INVALID for null pointers, H or W < 1, or a kind other than 0 and 1. */
STB_API int stb_snapshot(const float* value, int H, int W, double denom, int kind, void* out, void* stream);

/* ------------------------------------------------------------------ tiled iteration, exchanges inside the library
 * (csrc/comm.cu).  Each rank owns a MAILBOX (iteration stamps, its statistics block, its image gradient, its first /
 * last 80 updated rows) that the peers map with CUDA IPC and read over NVLink; stb_iterate_banded is then the whole
 * iteration of a band -- halo pull, forward, all-reduce of the statistics, backward, seam reduce of the gradient fused
 * with Adam + clamp + EMA -- as ONE stream-ordered sequence (one CUDA graph), with no host call between its phases.
 *   stb_comm_create        allocate the own mailbox for bands up to max_h_local x max_W (same numbers on every rank);
 *                          ipc_handle_out64: 64-byte cudaIpcMemHandle_t to ship to the peers; mailbox_out: the pointer
 *   stb_comm_connect_ipc   handles: world x 64 bytes in rank order (one process per GPU)
 *   stb_comm_connect_local mailboxes[world]: device pointers of contexts living in THIS process (tests / emulation)
 *   stb_comm_set_geometry  per scale: local height, first own row, own rows of this band; the neighbours' local
 *                          heights and the first bottom-apron row of the upper one (all in their local coordinates)
 *   stb_comm_reset         zero the iteration stamps; the host barriers over all ranks before AND after
 * A peer that does not show up within 30 s makes the waiting kernel trap (CUDA error), it never hangs. */
STB_API int stb_comm_create(stb_ctx* ctx, int rank, int world, int max_h_local, int max_W, void* ipc_handle_out64,
                            void** mailbox_out);
STB_API int stb_comm_connect_ipc(stb_ctx* ctx, const void* handles);
STB_API int stb_comm_connect_local(stb_ctx* ctx, void* const* mailboxes);
STB_API int stb_comm_disconnect(stb_ctx* ctx);  /* unmap the peers' mailboxes (host barrier, then re-create) */
/* per-layer-halo mode (default of tiled runs): the band computes only its own rows of every layer and pulls the one row
 * above / below them from the neighbours' workspaces, which therefore are cudaMalloc blocks of the library mapped by
 * the neighbours (CUDA IPC).  stb_comm_alloc_workspace allocates, zeroes and binds (as stb_bind_workspace does) and
 * returns the 64-byte IPC handle / the pointer; stb_comm_connect_ws_* takes every rank's handle (world x 64 bytes) or
 * pointer in rank order; stb_comm_set_geometry(..., halo_rows = 1) then selects that mode for a scale (0: the band
 * recomputes 80-row aprons instead, no per-layer exchange -- cheaper when the layers are small, see DESIGN.md section 6);
 * stb_comm_release_workspace(unmap_only = 1) unmaps the neighbours, (0) also frees the own block (host barrier in
 * between). */
STB_API int stb_comm_alloc_workspace(stb_ctx* ctx, size_t bytes, void* ipc_handle_out64, void** ptr_out, void* stream);
STB_API int stb_comm_connect_ws_ipc(stb_ctx* ctx, const void* handles);
STB_API int stb_comm_connect_ws_local(stb_ctx* ctx, void* const* pointers);
STB_API int stb_comm_release_workspace(stb_ctx* ctx, int unmap_only);
STB_API int stb_comm_set_geometry(stb_ctx* ctx, int W, int h_local, int own0, int own_rows, int up_h_local,
                                  int up_apron_row0, int dn_h_local, int halo_rows);
STB_API int stb_comm_reset(stb_ctx* ctx, void* stream);
STB_API int stb_iterate_banded(stb_ctx* ctx, float* img, float* exp_avg, float* exp_avg_sq, float* ema, int64_t step,
                               float lr, float beta1, float beta2, float adam_eps, float ema_decay,
                               float* loss_out_host8, void* stream);
/* optimizer='lbfgs' on a band: the iteration of stb_iterate_banded up to the seam, then the L-BFGS step of
 * stb_iterate_lbfgs on this band's own rows.  The state holds the own rows only: stb_lbfgs_state_bytes(own_rows, W)
 * bytes, reset once per scale with stb_lbfgs_reset.  Every dot product of the step is summed over the ranks inside the
 * graph (a one-block kernel per reduction, ranks combined in rank order), so every rank holds bit-identical scalars
 * and takes the same branches.  img / ema: the local [1,3,h_local,W] band; only the own rows are updated, the halo rows
 * are refreshed from the neighbours.  STB_ERR_STATE without a band, a comm connection and geometry, or when the
 * geometry does not match the band; STB_ERR_INVALID for a state that is too small or misaligned. */
STB_API int stb_iterate_lbfgs_banded(stb_ctx* ctx, float* img, float* ema, void* state, size_t state_bytes,
                                     int64_t step, float ema_decay, float* loss_out_host8, void* stream);
/* 1: iterations replay as CUDA graphs, 2: enabled but nothing captured yet, 0: eager launches (note_out says why). */
STB_API int stb_graph_status(stb_ctx* ctx, char* note_out, size_t note_bytes);
/* Kernel launches issued through graph replays so far, counted from the captured graphs: number of replays, kernels
 * they launched (the L-BFGS entry points' replays included), and the kernel nodes of the graphs of
 * {stb_iterate, stb_iterate_fwd, stb_iterate_bwd, stb_iterate_banded}; the L-BFGS graphs have no entry there. */
STB_API int stb_launch_count(stb_ctx* ctx, int64_t* graph_replays, int64_t* kernels_replayed, int* kernels_per_graph4);

/* ------------------------------------------------------------------ measurement (bench.py roofline leg)
 * CUDA-event timing per kernel class on the launching stream; classes in order: conv0_fwd_tv, conv_fwd, pool_fwd,
 * gram, sse, w2, conv_bwd, pool_bwd, conv0_bwd_adam, finalize (STB_PROF_CLASSES entries). */
#define STB_PROF_CLASSES 10
STB_API int stb_profile_enable(stb_ctx* ctx, int enable);
STB_API int stb_profile_read(stb_ctx* ctx, float* ms_out, int* count_out, int n_classes);

/* ------------------------------------------------------------------ diagnostics
 * stb_debug_w2_trace (with STB_W2_TRACE=1 in the environment): per-round %globaltimer stamps of CTA 0 of the W2 chain
 * kernel, 8 words per round for up to 128 rounds (tools/w2_trace.py prints the timeline). */
STB_API int stb_debug_w2_trace(stb_ctx* ctx, unsigned long long* host_out, size_t words, int* rounds_out);
/*
 * Copy of an internal activation (post-ReLU output of conv `conv_index`, bf16 NHWC) of the last forward. */
STB_API int stb_debug_activation(stb_ctx* ctx, int H, int W, int conv_index, void* out_bf16, size_t out_bytes,
                                 void* stream);

#ifdef __cplusplus
}
#endif
#endif /* STB200_H_ */
