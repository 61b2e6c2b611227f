// Kernel-level C-ABI entry points used by tests/ (each wraps exactly one launcher so that the parity tests can
// check every kernel against the oracle in isolation).  Declared in include/stb200_test.h; linked ONLY into
// libstb200_test.so -- the product library libstb200.so does not contain this file.
#include "kernels.h"
#include "stb200_test.h"

using namespace stb;

extern "C" {

const char* stb_test_last_error(void) { return last_error_string().c_str(); }

int stb_pack_weights(const float* w_oihw, void* out_bf16, int Cout, int Cin, int bwd, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  return bwd ? pack_weights_bwd(w_oihw, static_cast<bf16*>(out_bf16), Cout, Cin, s)
             : pack_weights_fwd(w_oihw, static_cast<bf16*>(out_bf16), Cout, Cin, s);
}

int stb_test_pixel_gemm(int H, int W, int Cin, int Cout, int C2, int mode, const void* A, const void* Bw,
                        const void* A2, int a2_row0, int a2_rows, const void* B2, void* out, const float* bias,
                        const void* mask_src, const void* ctarget, float cscale, int row_lo, int row_hi,
                        void* stream) {
  PixelGemmArgs a;
  a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout; a.C2 = C2; a.mode = mode;
  a.A = static_cast<const bf16*>(A);
  a.Bw = static_cast<const bf16*>(Bw);
  a.A2 = static_cast<const bf16*>(A2);
  a.a2_row0 = a2_row0; a.a2_rows = a2_rows;
  a.B2 = static_cast<const bf16*>(B2);
  a.out = static_cast<bf16*>(out);
  a.bias = bias;
  a.mask_src = static_cast<const bf16*>(mask_src);
  a.ctarget = static_cast<const bf16*>(ctarget);
  a.cscale = cscale;
  a.row_lo = row_lo; a.row_hi = row_hi;
  return launch_pixel_gemm(a, static_cast<cudaStream_t>(stream));
}

}  // extern "C"

extern "C" {

int stb_test_tv(const float* img, int H, int W, int row0, int rows, int H_norm, float tv_weight, float* gtv,
                float* tv_partials, int* n_partials, void* stream) {
  STB_CHECK(img && gtv && tv_partials && H > 0 && W > 0 && H_norm > 0, STB_ERR_INVALID, "bad argument");
  STB_CHECK(row0 >= 0 && rows > 0 && row0 + rows <= H, STB_ERR_INVALID, "row window [%d, %d) outside 0..%d", row0,
            row0 + rows, H);
  return launch_tv(img, H, W, row0, rows, H_norm, tv_weight, gtv, tv_partials, n_partials,
                   static_cast<cudaStream_t>(stream));
}

int stb_test_conv0_fwd(const float* img, const float* w0, const float* b0, void* out_bf16, int H, int W,
                       float tv_weight, float* gtv, float* tv_partials, int* n_partials, void* stream) {
  // product path of conv0: TV on the whole image (when gtv is given) and the fused im2col + wgmma GEMM + bias + ReLU
  // kernel
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (gtv != nullptr) STB_TRY(stb_test_tv(img, H, W, 0, H, H, tv_weight, gtv, tv_partials, n_partials, stream));
  bf16* wp = nullptr;
  STB_CUDA_CHECK(cudaMalloc(&wp, 64 * 64 * 2));
  int rc = pack_weights_conv0_fwd(w0, wp, s);
  if (rc == 0) rc = launch_conv0_fwd(img, wp, b0, static_cast<bf16*>(out_bf16), H, W, s);
  cudaStreamSynchronize(s);
  cudaFree(wp);
  return rc;
}

int stb_test_conv0_bwd_adam(const void* g0_bf16, const float* w0, const float* gtv, float* grad_out, int H, int W,
                            float* img, float* exp_avg, float* exp_avg_sq, float* ema, int64_t step, float lr,
                            float beta1, float beta2, float eps, float ema_decay, int apply_update, void* stream) {
  // the tail of the product's backward pass: interior via the wgmma 1x1 GEMM + col2im kernel with the image-space
  // epilogue, then the border ring in SIMT, each with the fused Adam + clamp + EMA step when apply_update
  STB_CHECK(!apply_update || (img && exp_avg && exp_avg_sq && ema && step >= 1), STB_ERR_INVALID,
            "apply_update needs img, exp_avg, exp_avg_sq, ema and step >= 1");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  bf16* wp = nullptr;
  AdamScalars* d_adam = nullptr;
  STB_CUDA_CHECK(cudaMalloc(&wp, 32 * 64 * 2));
  int rc = STB_OK;
  if (apply_update) {
    const AdamScalars as = make_adam_scalars(step, lr, beta1, beta2, eps, ema_decay);
    if (cudaMalloc(&d_adam, sizeof(AdamScalars)) != cudaSuccess ||
        cudaMemcpyAsync(d_adam, &as, sizeof(AdamScalars), cudaMemcpyHostToDevice, s) != cudaSuccess)
      rc = set_error(STB_ERR_CUDA, "conv0 bwd: Adam scalars to the device");
  }
  if (rc == 0) rc = pack_weights_conv0_bwd(w0, wp, s);
  if (rc == 0)
    rc = launch_conv0_bwd_interior(static_cast<const bf16*>(g0_bf16), wp, gtv, img, exp_avg, exp_avg_sq, ema,
                                   grad_out, H, W, d_adam, apply_update, s);
  if (rc == 0)
    rc = launch_conv0_bwd_adam(static_cast<const bf16*>(g0_bf16), true, w0, gtv, img, exp_avg, exp_avg_sq, ema,
                               grad_out, H, W, d_adam, apply_update, s);
  cudaStreamSynchronize(s);
  cudaFree(wp);
  if (d_adam) cudaFree(d_adam);
  return rc;
}

int stb_test_conv0_bwd(const void* g0_bf16, const float* w0, const float* gtv, float* grad_out, int H, int W,
                       void* stream) {
  return stb_test_conv0_bwd_adam(g0_bf16, w0, gtv, grad_out, H, W, nullptr, nullptr, nullptr, nullptr, 0, 0.f, 0.f,
                                 0.f, 0.f, 0.f, 0, stream);
}

int stb_test_sse(const void* a_bf16, const void* b_bf16, long n, float* partials, int* n_partials, void* stream) {
  return launch_sse(static_cast<const bf16*>(a_bf16), static_cast<const bf16*>(b_bf16), n, partials, n_partials,
                    static_cast<cudaStream_t>(stream));
}

int stb_test_conv_pool(int H, int W, int Cin, int Cout, const void* A, const void* Bw, const float* bias, void* out,
                       void* pool_out, int pooling, void* stream) {
  PixelGemmArgs a;
  a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout; a.mode = 0;
  a.A = static_cast<const bf16*>(A);
  a.Bw = static_cast<const bf16*>(Bw);
  a.out = static_cast<bf16*>(out);
  a.bias = bias;
  a.pool_out = static_cast<bf16*>(pool_out);
  a.pooling = pooling;
  return launch_pixel_gemm(a, static_cast<cudaStream_t>(stream));
}

int stb_test_pool_bwd(int pooling, const void* gout, const void* y, void* gin, int H, int W, int C, void* stream) {
  return launch_pool_bwd(pooling, static_cast<const bf16*>(gout), static_cast<const bf16*>(y), static_cast<bf16*>(gin),
                         H, W, C, static_cast<cudaStream_t>(stream));
}

size_t stb_test_gram_partials_floats(long P, int C) { return gram_partials_floats(P, C); }

int stb_test_gram(const void* F_bf16, long P, int C, float* partials_ws, size_t partials_floats, float* S_raw,
                  float* sums, void* stream) {
  STB_CHECK(partials_floats >= gram_partials_floats(P, C), STB_ERR_WORKSPACE, "gram partials workspace too small");
  return launch_gram(static_cast<const bf16*>(F_bf16), P, C, partials_ws, partials_floats, S_raw, sums,
                     static_cast<cudaStream_t>(stream));
}

// The launch sequence of the L-BFGS step of stb_iterate_lbfgs on a scripted gradient (NULL: the gradient already in
// the state, e.g. to time the step alone).  pairs_out / t_out (optional, synchronous): history pairs and step length.
int stb_test_lbfgs_step(void* state, size_t bytes, int H, int W, float* x, const float* grad, float* ema,
                        float ema_decay, int* pairs_out, float* t_out, void* stream) {
  STB_CHECK(state && x && ema && H > 0 && W > 0, STB_ERR_INVALID, "bad argument");
  STB_CHECK((reinterpret_cast<uintptr_t>(state) & 255) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 &&
                (reinterpret_cast<uintptr_t>(ema) & 15) == 0,
            STB_ERR_INVALID, "state must be 256-byte aligned, x and ema 16-byte aligned");
  const long n = 3l * H * W;
  STB_CHECK(bytes >= lbfgs_state_bytes(n), STB_ERR_INVALID, "L-BFGS state too small");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (grad)
    STB_CUDA_CHECK(cudaMemcpyAsync(lbfgs_grad_buffer(state, n), grad, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
  STB_TRY(launch_lbfgs_step(state, n, x, ema, ema_decay, s));
  if (pairs_out || t_out) STB_TRY(lbfgs_read_info(state, pairs_out, t_out, s));
  return STB_OK;
}

// The gradient the last L-BFGS step consumed: after stb_iterate_lbfgs the whole-image closure gradient, after
// stb_iterate_lbfgs_banded (H = own rows) the band's own-row gradient after the seam reduce.
int stb_test_lbfgs_gradient(const void* state, size_t bytes, int H, int W, float* out, void* stream) {
  STB_CHECK(state && out && H > 0 && W > 0, STB_ERR_INVALID, "bad argument");
  STB_CHECK((reinterpret_cast<uintptr_t>(state) & 255) == 0, STB_ERR_INVALID, "state must be 256-byte aligned");
  const long n = 3l * H * W;
  STB_CHECK(bytes >= lbfgs_state_bytes(n), STB_ERR_INVALID, "L-BFGS state too small");
  STB_CUDA_CHECK(cudaMemcpyAsync(out, lbfgs_grad_buffer(const_cast<void*>(state), n), n * sizeof(float),
                                 cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)));
  return STB_OK;
}

// Loads every kernel of THIS library (it holds its own copies of the product kernels).  A banded test step must not be
// the first launch of a kernel: a lazy module load synchronises the context, which deadlocks against a peer's resident
// wait kernel (see comm_preload).
int stb_test_preload(void) {
  STB_TRY(comm_preload()); STB_TRY(preload_conv_kernels()); STB_TRY(preload_gram_kernels());
  STB_TRY(preload_w2_kernels()); STB_TRY(preload_conv0_kernels()); STB_TRY(preload_image_kernels());
  return STB_OK;
}

// The banded step of stb_iterate_lbfgs_banded on a scripted gradient, on a context with a comm connection and geometry:
// comm phase 0, halo pull, grad [3][h_local][W] into the mailbox, phase 2, the banded step, phase 3.
int stb_test_lbfgs_step_banded(stb_ctx* ctx, void* state, size_t bytes, float* x, const float* grad, float* ema,
                               float ema_decay, int add_seams, int* pairs_out, float* t_out, void* stream) {
  STB_CHECK(ctx && state && x && grad && ema, STB_ERR_INVALID, "null argument");
  const CommDev* c = ctx_comm(ctx);
  STB_CHECK(c != nullptr, STB_ERR_STATE, "stb_comm_connect_* + stb_comm_set_geometry first");
  STB_CHECK((reinterpret_cast<uintptr_t>(state) & 255) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 &&
                (reinterpret_cast<uintptr_t>(ema) & 15) == 0,
            STB_ERR_INVALID, "state must be 256-byte aligned, x and ema 16-byte aligned");
  STB_CHECK(bytes >= lbfgs_state_bytes(3l * c->own_rows * c->W), STB_ERR_INVALID, "L-BFGS state too small");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  STB_TRY(launch_comm_phase(*c, 0, s));
  STB_TRY(launch_halo_pull(*c, x, s));
  STB_CUDA_CHECK(cudaMemcpyAsync(c->mbox[c->rank] + c->off_grad, grad, 3ul * c->h_local * c->W * sizeof(float),
                                 cudaMemcpyDeviceToDevice, s));
  STB_TRY(launch_comm_phase(*c, 2, s));
  STB_TRY(launch_lbfgs_step_banded(state, *c, x, ema, ema_decay, add_seams, s));
  STB_TRY(launch_comm_phase(*c, 3, s));
  if (pairs_out || t_out) STB_TRY(lbfgs_read_info(state, pairs_out, t_out, s));
  return STB_OK;
}

// whether the exchange kernels of a connected context release their dependents early (CommDev::pdl), and the devices
// that hold its own mailbox and its own peer-mapped workspace (-1: none)
int stb_test_comm_info(stb_ctx* ctx, int* pdl_out, int* mailbox_device_out, int* workspace_device_out) {
  STB_CHECK(ctx && pdl_out && mailbox_device_out && workspace_device_out, STB_ERR_INVALID, "null argument");
  const CommDev* c = ctx_comm(ctx);
  STB_CHECK(c != nullptr, STB_ERR_STATE, "stb_comm_connect_* + stb_comm_set_geometry first");
  *pdl_out = c->pdl;
  const void* own[2] = {c->mbox[c->rank], c->ws[c->rank]};
  int* out[2] = {mailbox_device_out, workspace_device_out};
  for (int i = 0; i < 2; ++i) {
    *out[i] = -1;
    if (own[i] == nullptr) continue;
    cudaPointerAttributes pa;
    STB_CUDA_CHECK(cudaPointerGetAttributes(&pa, own[i]));
    *out[i] = pa.device;
  }
  return STB_OK;
}

size_t stb_test_w2_workspace_bytes(void) { return W2Engine::workspace_bytes(); }

// Runs the W2 engine with the given problem placed in the slot of matching size (other slots get a benign
// identity problem).  Outputs: weighted loss, Gs = G + G^T (fp32, NOT divided by npix), gmu (not divided),
// and the target's sqrtm(cov_t).
int stb_test_w2(const float* mean_t, const float* srm_t, const float* S_raw, const float* sums, int C, float npix,
                float weight, void* ws, size_t ws_bytes, float* loss_out, float* gs_out, float* gmu_out,
                float* csqrt_out, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  static W2Engine eng;  // test-only
  const int ns[5] = {64, 128, 256, 512, 512};
  STB_TRY(eng.init(ws, ws_bytes, 5, ns));
  int slot = -1;
  for (int l = 0; l < 5; ++l)
    if (ns[l] == C) { slot = l; break; }
  STB_CHECK(slot >= 0, STB_ERR_INVALID, "C must be one of 64,128,256,512");
  // benign content for the other slots: srm = I, mean = 0, S_raw = I, sums = 0, npix = 1
  for (int l = 0; l < 5; ++l) {
    W2Layer& L = eng.host_layers[l];
    const int n = L.n;
    std::vector<float> eye((size_t)n * n, 0.f), zero(n, 0.f);
    for (int i = 0; i < n; ++i) eye[(size_t)i * n + i] = 1.f;
    L.weight = 1.f; L.npix = 1.f;
    L.S_raw = L.X1;   // scratch matrices that the forward does not touch before reading S_raw
    L.sums = L.gmu_bias;
    STB_CUDA_CHECK(cudaMemcpyAsync(L.srm_t, eye.data(), eye.size() * 4, cudaMemcpyHostToDevice, s));
    STB_CUDA_CHECK(cudaMemcpyAsync(L.S_raw, eye.data(), eye.size() * 4, cudaMemcpyHostToDevice, s));
    STB_CUDA_CHECK(cudaMemcpyAsync(L.mean_t, zero.data(), n * 4, cudaMemcpyHostToDevice, s));
    STB_CUDA_CHECK(cudaMemcpyAsync(L.sums, zero.data(), n * 4, cudaMemcpyHostToDevice, s));
    STB_CUDA_CHECK(cudaStreamSynchronize(s));
  }
  W2Layer& T = eng.host_layers[slot];
  T.weight = weight; T.npix = npix;
  STB_CUDA_CHECK(cudaMemcpyAsync(T.srm_t, srm_t, (size_t)C * C * 4, cudaMemcpyDeviceToDevice, s));
  STB_CUDA_CHECK(cudaMemcpyAsync(T.mean_t, mean_t, (size_t)C * 4, cudaMemcpyDeviceToDevice, s));
  STB_CUDA_CHECK(cudaMemcpyAsync(T.S_raw, S_raw, (size_t)C * C * 4, cudaMemcpyDeviceToDevice, s));
  STB_CUDA_CHECK(cudaMemcpyAsync(T.sums, sums, (size_t)C * 4, cudaMemcpyDeviceToDevice, s));
  STB_TRY(eng.upload_layers(s));
  STB_TRY(eng.build_targets(s));
  STB_TRY(eng.forward_backward(T.scal + 32, s));
  STB_CUDA_CHECK(cudaMemcpyAsync(loss_out, T.scal + W2S_LOSS, 4, cudaMemcpyDeviceToDevice, s));
  STB_CUDA_CHECK(cudaMemcpyAsync(gs_out, T.Gs, (size_t)C * C * 4, cudaMemcpyDeviceToDevice, s));
  STB_TRY(W2Engine::read_matrix(csqrt_out, T.P, C, s));
  // gmu_bias holds gmu / npix
  STB_CUDA_CHECK(cudaMemcpyAsync(gmu_out, T.gmu_bias, (size_t)C * 4, cudaMemcpyDeviceToDevice, s));
  return STB_OK;
}

// The engine as stb_set_targets / the iteration drive it: five problems in their own slots, S_raw / sums bound in place
// (as the statistics block is), targets built once and forward_backward run n_calls times on one engine, so that the
// ping-pong iterates, the scalars and the device-patched Gc alpha carry over from call to call.
int stb_test_w2_layers(const float* const* mean_t, const float* const* srm_t, const float* const* S_raw,
                       const float* const* sums, const float* npix, const float* weight, int build_targets,
                       int n_calls, void* ws, size_t ws_bytes, float* loss_out, float* const* gs_out,
                       void* const* gs_bf16_out, float* const* gmu_out, float* const* mu_out, float* const* csqrt_out,
                       void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  static W2Engine eng;  // test-only
  static void* bound = nullptr;
  const int ns[5] = {64, 128, 256, 512, 512};
  STB_CHECK(S_raw && sums && npix && weight && ws && loss_out && gs_out && gs_bf16_out && gmu_out && mu_out &&
                csqrt_out && n_calls >= 1,
            STB_ERR_INVALID, "bad argument");
  STB_CHECK(build_targets || ws == bound, STB_ERR_STATE, "build_targets = 0 needs the workspace of the previous call");
  if (ws != bound) {
    STB_TRY(eng.init(ws, ws_bytes, 5, ns));
    bound = ws;
  }
  for (int l = 0; l < 5; ++l) {
    W2Layer& L = eng.host_layers[l];
    const size_t nn = (size_t)L.n * L.n;
    L.weight = weight[l]; L.npix = npix[l];
    L.S_raw = const_cast<float*>(S_raw[l]);
    L.sums = const_cast<float*>(sums[l]);
    if (build_targets) {
      STB_CHECK(mean_t && srm_t && mean_t[l] && srm_t[l], STB_ERR_INVALID, "build_targets needs mean_t and srm_t");
      STB_CUDA_CHECK(cudaMemcpyAsync(L.mean_t, mean_t[l], L.n * 4, cudaMemcpyDeviceToDevice, s));
      STB_CUDA_CHECK(cudaMemcpyAsync(L.srm_t, srm_t[l], nn * 4, cudaMemcpyDeviceToDevice, s));
    }
  }
  STB_TRY(eng.upload_layers(s));
  if (build_targets) STB_TRY(eng.build_targets(s));
  for (int c = 0; c < n_calls; ++c) STB_TRY(eng.forward_backward(loss_out, s));
  for (int l = 0; l < 5; ++l) {
    const W2Layer& L = eng.host_layers[l];
    const size_t nn = (size_t)L.n * L.n;
    STB_CUDA_CHECK(cudaMemcpyAsync(gs_out[l], L.Gs, nn * 4, cudaMemcpyDeviceToDevice, s));
    STB_CUDA_CHECK(cudaMemcpyAsync(gs_bf16_out[l], L.gs_bf16, nn * 2, cudaMemcpyDeviceToDevice, s));
    STB_CUDA_CHECK(cudaMemcpyAsync(gmu_out[l], L.gmu_bias, L.n * 4, cudaMemcpyDeviceToDevice, s));
    STB_CUDA_CHECK(cudaMemcpyAsync(mu_out[l], L.mu, L.n * 4, cudaMemcpyDeviceToDevice, s));
    STB_TRY(W2Engine::read_matrix(csqrt_out[l], L.P, L.n, s));
  }
  return STB_OK;
}

}  // extern "C"
