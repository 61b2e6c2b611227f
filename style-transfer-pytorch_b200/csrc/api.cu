// C-ABI of the H100-native stylize() hot path (see include/stb200.h).  The context owns an explicit, static
// forward/backward schedule for torchvision vgg19().features[:30] -- no autograd on the path:
//   forward   ST:78-90     conv0 (+TV) -> 12 x wgmma conv/bias/ReLU, 4 pools, taps 1,6,11,20,22,29
//   losses    ST:119-126, 149-181, 184-195, 198-234  content MSE, 5 x W2 style (Gram on wgmma, sqrtm in fp32), TV
//   backward  ST:475       tap-gradient GEMMs folded into the dgrad chain, pool backward, conv0 dgrad
//   update    ST:481-486   Adam + clamp + EMA fused into the last kernel
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <string>

#include "kernels.h"
#include "ptx.cuh"

using namespace stb;

namespace {

constexpr int NCONV = STB_NUM_CONVS;
const int kCin[NCONV] = {3, 64, 64, 128, 128, 256, 256, 256, 256, 512, 512, 512, 512};
const int kCout[NCONV] = {64, 64, 128, 128, 256, 256, 256, 256, 512, 512, 512, 512, 512};
const bool kPoolAfter[NCONV] = {false, true, false, true, false, false, false, true, false, false, false, true, false};
// The six ReLU taps of the reference model, VGGFeatures(style_layers + content_layers) with the default lists (ST:324),
// and the convs whose ReLU output they are.  A layer table selects content and style taps among them.
constexpr int kNumTaps = STB_NUM_TAPS;
const int kTapLayer[kNumTaps] = {1, 6, 11, 20, 22, 29};
const int kTapConv[kNumTaps] = {0, 2, 4, 8, 9, 12};
constexpr int kStatsTailMax = 8;    // the stats tail of the largest table: six content SSEs + TV, padded to 4 floats
constexpr int kSsePartials = 1024;  // launch_sse writes at most this many partials

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// content and style taps in the caller's list order (stb_set_layers); the default is the reference's (ST:316-317)
struct LayerTable {
  int n_content = 1, content_conv[kNumTaps] = {9};
  int n_style = 5, style_conv[kNumTaps] = {0, 2, 4, 8, 12};
  int style_c(int l) const;
  int last_conv() const {   // the deepest conv any loss term reads: the forward stops there, the backward starts there
    int last = 0;
    for (int k = 0; k < n_content; ++k) last = std::max(last, content_conv[k]);
    for (int l = 0; l < n_style; ++l) last = std::max(last, style_conv[l]);
    return last;
  }
  int last_style_conv() const {
    int last = 0;
    for (int l = 0; l < n_style; ++l) last = std::max(last, style_conv[l]);
    return last;
  }
  int last_content_conv() const {
    int last = 0;
    for (int k = 0; k < n_content; ++k) last = std::max(last, content_conv[k]);
    return last;
  }
  int style_at(int conv) const {   // style index of the tap at `conv`, or -1
    for (int l = 0; l < n_style; ++l) if (style_conv[l] == conv) return l;
    return -1;
  }
  int content_at(int conv) const {
    for (int k = 0; k < n_content; ++k) if (content_conv[k] == conv) return k;
    return -1;
  }
  bool is_default() const {
    const LayerTable d;
    return n_content == d.n_content && n_style == d.n_style &&
           std::memcmp(content_conv, d.content_conv, sizeof(int) * n_content) == 0 &&
           std::memcmp(style_conv, d.style_conv, sizeof(int) * n_style) == 0;
  }
  // {content SSE per content tap, TV sum} ride at the tail of the stats block, padded to four floats
  size_t stats_tail() const { return align_up((size_t)n_content + 1, 4); }
};

int LayerTable::style_c(int l) const { return kCout[style_conv[l]]; }

// the stats block of the largest configuration (all six taps in both roles): the size of a mailbox's stats slots
size_t stats_floats_max() {
  size_t sf = kStatsTailMax;
  for (int t = 0; t < kNumTaps; ++t) sf += (size_t)kCout[kTapConv[t]] * kCout[kTapConv[t]] + kCout[kTapConv[t]];
  return sf;
}

struct Plan {
  int H = 0, W = 0;
  int h[NCONV], w[NCONV];      // spatial size of conv i's input == output
  size_t act_off[NCONV];       // post-ReLU output of conv i (bf16 NHWC)
  size_t pool_off[4];          // pooled copies
  size_t g_off[2];             // gradient ping-pong
  size_t gtv_off, tvp_off, ssep_off, gramp_off, stats_off, loss_off;
  size_t ctarget_off[kNumTaps];        // content target of each content tap (bf16 NHWC)
  size_t stats_layer_off[kNumTaps];    // in floats, inside the stats block: S_raw then sums per style tap
  size_t stats_scalars = 0, stats_floats = 0, gramp_floats = 0;
  size_t total = 0;
  int n_tv_partials = 0, n_sse_partials = 0;
};

}  // namespace

// Optional per-kernel-class timing with CUDA events on the launching stream (bench.py's roofline leg).
enum ProfClass { PC_CONV0_FWD = 0, PC_CONV_FWD, PC_POOL_FWD, PC_GRAM, PC_SSE, PC_W2, PC_CONV_BWD, PC_POOL_BWD,
                 PC_CONV0_BWD_ADAM, PC_FINALIZE, PC_COUNT };
struct Prof {
  bool on = false;
  std::vector<cudaEvent_t> pool;
  struct Span { int cls; int e0, e1; };
  std::vector<Span> spans;
  int used = 0;
  int get_event() {
    if (used == (int)pool.size()) {
      cudaEvent_t e;
      cudaEventCreate(&e);
      pool.push_back(e);
    }
    return used++;
  }
  void begin(int cls, cudaStream_t s) {
    if (!on) return;
    Span sp{cls, get_event(), -1};
    cudaEventRecord(pool[sp.e0], s);
    spans.push_back(sp);
  }
  void end(cudaStream_t s) {
    if (!on) return;
    spans.back().e1 = get_event();
    cudaEventRecord(pool[spans.back().e1], s);
  }
};

// one captured graph per iteration entry point; stb_launch_count reports the first four
enum GraphSlotId { GS_ITERATE = 0, GS_ITERATE_FWD, GS_ITERATE_BWD, GS_ITERATE_BANDED, GS_ITERATE_LBFGS,
                   GS_ITERATE_LBFGS_BANDED, GS_COUNT };

struct stb_ctx {
  Prof prof;
  int device = 0;
  int pooling = STB_POOL_MAX;
  float* w0 = nullptr;  // conv0 fp32 OIHW (borrowed copy)
  float* bias[NCONV] = {};
  bf16* wf[NCONV] = {};  // packed forward weights  [9][Cout][Cin]
  bf16* wb[NCONV] = {};  // packed dgrad weights    [9][Cin][Cout]
  void* owned = nullptr; // one cudaMalloc block holding all of the above
  uint8_t* ws = nullptr;
  size_t ws_bytes = 0;
  size_t w2_bytes = 0;
  W2Engine w2;
  bool w2_ready = false;
  // per-scale loss state
  bool targets_set = false;
  int tH = 0, tW = 0;
  LayerTable layers;
  float content_w[kNumTaps] = {}, tv_weight = 0.f;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  // spatial tiling (multi-GPU): this context works on a horizontal band of a taller image.  The local image is the
  // band plus halo aprons; only the "own" rows contribute to the statistics / losses / tap gradients.
  int n_tv_partials = 0;
  // device-resident optimiser scalars (so that an iteration is a fixed launch sequence -> CUDA graph)
  AdamScalars* d_adam = nullptr;
  long long* d_step = nullptr;
  long long dev_step_mirror = -1;  // host's view of *d_step
  // CUDA graph of one fused iteration, keyed by everything baked into the launches (null / 0: not an argument of the
  // entry point)
  struct GraphKey {
    int H, W; const void *ws, *img, *exp_avg, *exp_avg_sq, *ema, *grad_out, *state, *loss;
    float lr, b1, b2, eps, decay;
    bool operator==(const GraphKey& o) const { return std::memcmp(this, &o, sizeof(GraphKey)) == 0; }
  };
  struct GraphSlot {
    GraphKey key{};
    int hits = 0;
    int kernel_nodes = 0;   // kernel launches one replay stands for (counted from the captured graph)
    cudaGraphExec_t exec = nullptr;
    void reset() {
      if (exec) cudaGraphExecDestroy(exec);
      exec = nullptr; key = GraphKey{}; hits = 0; kernel_nodes = 0;
    }
  };
  GraphSlot gslot[GS_COUNT];
  void reset_graphs() { for (auto& g : gslot) g.reset(); }
  bool graphs_enabled = true;
  std::string graph_note;  // why graph replay was switched off for this context (stb_graph_status)
  long long graph_replays = 0, kernels_replayed = 0;   // stb_launch_count
  // sync-free loss read-back (stb_set_loss_ring): pinned host ring written by the finalize kernel itself
  float* ring_dev = nullptr;   // device alias of the pinned host ring
  int ring_slots = 0;
  bool band_on = false;
  int band_H_global = 0, band_own0 = 0, band_own_rows = 0;
  // peer-memory exchange of the tiled iteration (comm.cu)
  CommDev comm{};
  bool comm_ready = false, comm_geometry = false, comm_ipc = false;
  void* comm_mailbox = nullptr;       // own cudaMalloc block
  size_t comm_bytes = 0;
  int comm_max_h = 0, comm_max_w = 0;
  // per-layer-halo mode: the workspace itself is a cudaMalloc block of the library, mapped by the neighbours (they pull
  // single boundary rows of the activation / gradient tensors out of it)
  void* shared_ws = nullptr;
  size_t shared_ws_bytes = 0;
  bool shared_ws_ipc = false, halo_mode = false;
  int halo_seq = 0;                   // exchange counter inside the iteration being recorded
};

// every ctx entry point runs on the context's device, whatever the caller's current device is
#define STB_ENTER(ctx)                                                       \
  do {                                                                       \
    STB_CHECK((ctx) != nullptr, STB_ERR_INVALID, "null ctx");                \
    STB_CUDA_CHECK(cudaSetDevice((ctx)->device));                            \
  } while (0)

namespace {

// workspace layout for an H x W image under the context's layer table: activations up to its deepest conv only
void make_plan(const stb_ctx* ctx, int H, int W, Plan* pl) {
  const LayerTable& lt = ctx->layers;
  const int last = lt.last_conv();
  pl->H = H; pl->W = W;
  int h = H, w = W;
  size_t off = align_up(ctx->w2_bytes, 1024);
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 1024); return o; };
  int np = 0;
  size_t gmax = 0;
  for (int i = 0; i < NCONV; ++i) {
    pl->h[i] = h; pl->w[i] = w;
    pl->act_off[i] = i <= last ? take((size_t)h * w * kCout[i] * 2) : 0;
    if (i <= last) gmax = std::max(gmax, (size_t)h * w * kCout[i] * 2);
    if (kPoolAfter[i]) {
      h /= 2; w /= 2;
      pl->pool_off[np++] = i < last ? take((size_t)std::max(h, 1) * std::max(w, 1) * kCout[i] * 2) : 0;
    }
  }
  pl->g_off[0] = take(gmax);
  pl->g_off[1] = take(gmax);
  pl->gtv_off = take((size_t)3 * H * W * 4);
  pl->n_tv_partials = ((W + 255) / 256) * H;
  pl->tvp_off = take((size_t)pl->n_tv_partials * 4);
  pl->ssep_off = take((size_t)kSsePartials * lt.n_content * 4);   // the SSE partials of content tap k at k * 1024
  // split-K partials of the Gram kernels: the bound over every pixel count, because a banded context launches them
  // on its own rows only and the split count is not monotonic in the pixel count (~40 MB)
  size_t gp = 0;
  for (int l = 0; l < lt.n_style; ++l) gp = std::max(gp, gram_max_partials_floats(lt.style_c(l)));
  pl->gramp_floats = gp;
  pl->gramp_off = take(gp * 4);
  size_t sf = 0;
  for (int l = 0; l < lt.n_style; ++l) {
    const int C = lt.style_c(l);
    pl->stats_layer_off[l] = sf;
    sf += (size_t)C * C + C;
  }
  pl->stats_scalars = sf;  // {content SSE per content tap, TV sum} ride at the tail: one all-reduce covers everything
  sf += lt.stats_tail();
  pl->stats_floats = sf;
  pl->stats_off = take(sf * 4);
  pl->loss_off = take(64 * 4);
  for (int k = 0; k < lt.n_content; ++k) {
    const int ci = lt.content_conv[k];
    pl->ctarget_off[k] = take((size_t)pl->h[ci] * pl->w[ci] * kCout[ci] * 2);
  }
  pl->total = off;
}

int check_size(int H, int W, int last_conv) {
  int min_size = 1;
  for (int i = 0; i < last_conv; ++i)
    if (kPoolAfter[i]) min_size *= 2;
  STB_CHECK(H >= min_size && W >= min_size && H > 0 && W > 0, STB_ERR_INVALID,
            "Input is %dx%d but must be at least %dx%d", H, W, min_size, min_size);  // ST:82-83
  return STB_OK;
}

int ensure_ws(const stb_ctx* ctx, const Plan& pl) {
  STB_CHECK(ctx->ws != nullptr, STB_ERR_WORKSPACE, "no workspace bound (call stb_bind_workspace)");
  STB_CHECK(pl.total <= ctx->ws_bytes, STB_ERR_WORKSPACE, "workspace too small for %dx%d: need %zu bytes, have %zu",
            pl.H, pl.W, pl.total, ctx->ws_bytes);
  return STB_OK;
}

template <typename T>
T* at(const stb_ctx* ctx, size_t off) { return reinterpret_cast<T*>(ctx->ws + off); }

// pyramid level of conv i's grid: the number of pools before it
int level_of(int conv) {
  int level = 0;
  for (int i = 0; i < conv; ++i)
    if (kPoolAfter[i]) ++level;
  return level;
}

struct BandRows { int own0, rows, h_global; };
// own rows of conv i's output grid and the global height at its level
BandRows band_rows(const stb_ctx* ctx, const Plan& pl, int conv) {
  BandRows b;
  if (!ctx->band_on) { b.own0 = 0; b.rows = pl.h[conv]; b.h_global = pl.h[conv]; return b; }
  const int level = level_of(conv);
  const bool is_bottom = ctx->band_own0 + ctx->band_own_rows >= pl.H;
  b.own0 = ctx->band_own0 >> level;
  b.rows = is_bottom ? pl.h[conv] - b.own0 : (ctx->band_own_rows >> level);
  b.h_global = ctx->band_H_global >> level;   // floor-mode pools of a positive height
  return b;
}

// ---- per-layer halo exchange ("halo mode" of a tiled iteration, DESIGN.md section 6).  A band computes only its own
// rows of every activation / gradient tensor; the row above and the row below them, which the next 3x3 kernel reads,
// are the neighbours' boundary own rows and are pulled straight out of the neighbours' workspaces.
struct HaloPlans { Plan up, dn; };
// tensor with C channels at pyramid level `level` (width w_l); off_* = its byte offset in the plan of me / up / down.
// sync_only: publish + wait the stamps without copying (a buffer the neighbours pulled from is about to be rewritten).
int halo_exchange(stb_ctx* ctx, int level, int w_l, int C, size_t off_me, size_t off_up, size_t off_dn,
                  bool sync_only, cudaStream_t s) {
  const CommDev& c = ctx->comm;
  const bool has_up = c.rank > 0, has_dn = c.rank + 1 < c.world;
  const size_t row_bytes = (size_t)w_l * C * 2;
  const int o0 = ctx->band_own0 >> level, r = ctx->band_own_rows >> level;   // interior edges: multiples of 16
  HaloRowArgs a{};
  a.row_bytes = sync_only ? 0 : row_bytes;
  a.seq = ++ctx->halo_seq;
  STB_CHECK(a.seq < 256, STB_ERR_STATE, "too many halo exchanges in one iteration");
  if (has_up) {
    const int up_own0 = (c.rank - 1 > 0 ? COMM_APRON : 0) >> level;
    const int up_last = (c.up_apron_row0 >> level) - 1;   // last own row of the upper band at this level
    STB_CHECK(c.ws[c.rank - 1] != nullptr && up_last >= up_own0 && o0 >= 1, STB_ERR_STATE, "halo: upper neighbour not mapped");
    a.src_up = c.ws[c.rank - 1] + off_up + (size_t)up_last * row_bytes;
    a.dst_up = ctx->ws + off_me + (size_t)(o0 - 1) * row_bytes;
  }
  if (has_dn) {
    STB_CHECK(c.ws[c.rank + 1] != nullptr, STB_ERR_STATE, "halo: lower neighbour not mapped");
    a.src_dn = c.ws[c.rank + 1] + off_dn + (size_t)(COMM_APRON >> level) * row_bytes;
    a.dst_dn = ctx->ws + off_me + (size_t)(o0 + r) * row_bytes;
  }
  return launch_halo_rows(c, a, s);
}

// forward through conv `last_conv` (inclusive); do_tv also produces the TV gradient / loss partials.
// halo != nullptr: per-layer-halo mode of a tiled iteration (own rows only + one exchange per layer).
int forward(stb_ctx* ctx, const Plan& pl, const float* img, int last_conv, bool do_tv, cudaStream_t s,
            const HaloPlans* halo = nullptr) {
  int ntv = 0;
  ctx->prof.begin(PC_CONV0_FWD, s);
  if (do_tv) {
    const BandRows br = band_rows(ctx, pl, 0);
    STB_TRY(launch_tv(img, pl.H, pl.W, br.own0, br.rows, br.h_global, ctx->tv_weight, at<float>(ctx, pl.gtv_off),
                      at<float>(ctx, pl.tvp_off), &ntv, s));
  }
  ctx->n_tv_partials = ntv;
  // conv0 on the tensor cores: Normalize + replicate pad + hi/lo im2col rows built in smem, bias + ReLU epilogue
  STB_TRY(launch_conv0_fwd(img, ctx->wf[0], ctx->bias[0], at<bf16>(ctx, pl.act_off[0]), pl.H, pl.W, s));
  ctx->prof.end(s);
  int np = 0;
  const bf16* cur = at<bf16>(ctx, pl.act_off[0]);
  for (int i = 1; i <= last_conv; ++i) {
    PixelGemmArgs a;
    a.H = pl.h[i]; a.W = pl.w[i]; a.Cin = kCin[i]; a.Cout = kCout[i]; a.mode = 0;
    a.A = cur; a.Bw = ctx->wf[i]; a.out = at<bf16>(ctx, pl.act_off[i]); a.bias = ctx->bias[i];
    cur = a.out;
    size_t x_me = pl.act_off[i], x_up = 0, x_dn = 0;   // the tensor the next conv reads, for the halo exchange
    int x_level = level_of(i), x_w = pl.w[i];
    if (halo) { x_up = halo->up.act_off[i]; x_dn = halo->dn.act_off[i]; }
    if (kPoolAfter[i] && i < last_conv) {  // the 2x2 pool that follows this conv is produced by its epilogue
      if (halo) { x_me = pl.pool_off[np]; x_up = halo->up.pool_off[np]; x_dn = halo->dn.pool_off[np]; ++x_level; x_w = pl.w[i + 1]; }
      a.pool_out = at<bf16>(ctx, pl.pool_off[np++]);
      a.pooling = ctx->pooling;
      cur = a.pool_out;
    }
    if (halo) {  // own rows only (conv0 ran on the whole local image: its halo rows are already there)
      const BandRows br = band_rows(ctx, pl, i);
      a.y_origin = br.own0; a.y_rows = br.rows;
    }
    ctx->prof.begin(PC_CONV_FWD, s);
    STB_TRY(launch_pixel_gemm(a, s));
    ctx->prof.end(s);
    if (halo && i < last_conv) STB_TRY(halo_exchange(ctx, x_level, x_w, kCout[i], x_me, x_up, x_dn, false, s));
  }
  return STB_OK;
}

int style_grams(stb_ctx* ctx, const Plan& pl, cudaStream_t s) {
  float* stats = at<float>(ctx, pl.stats_off);
  ctx->prof.begin(PC_GRAM, s);
  const LayerTable& lt = ctx->layers;
  for (int l = 0; l < lt.n_style; ++l) {
    const int ci = lt.style_conv[l];
    const int C = lt.style_c(l);
    float* S = stats + pl.stats_layer_off[l];
    const BandRows br = band_rows(ctx, pl, ci);
    STB_TRY(launch_gram(at<bf16>(ctx, pl.act_off[ci]) + (size_t)br.own0 * pl.w[ci] * C, (long)br.rows * pl.w[ci], C,
                        at<float>(ctx, pl.gramp_off), pl.gramp_floats, S, S + (size_t)C * C, s));
  }
  ctx->prof.end(s);
  return STB_OK;
}

// deterministic single-block reduction of the partials of every content SSE and of TV into the stats tail:
// out[j] = sum of array j (each summed in the same fixed order), zeros up to `tail` words
struct PartialArrays {
  const float* p[kNumTaps + 1];
  int n[kNumTaps + 1];
  int count, tail;
};
__global__ void reduce_partials_kernel(PartialArrays a, float* __restrict__ out) {
  __shared__ float s_red[kNumTaps + 1][32];
  for (int j = 0; j < a.count; ++j) {
    float v = 0.f;
    for (int i = threadIdx.x; i < a.n[j]; i += blockDim.x) v += a.p[j][i];
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) s_red[j][threadIdx.x >> 5] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int j = 0; j < a.count; ++j) {
      float t = 0.f;
      for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += s_red[j][i];
      out[j] = t;
    }
    for (int j = a.count; j < a.tail; ++j) out[j] = 0.f;
  }
}

// the first loss term of the content-only tap that seeds the backward (no style role there, so no GEMM): d loss /
// d pre-activation = (y > 0) * cscale * (y - t) on rows [row_lo, row_hi) of [rows][w][C], zero elsewhere
__global__ void content_seed_kernel(const bf16* __restrict__ y, const bf16* __restrict__ t, bf16* __restrict__ g,
                                    long n, long row_elems, int row_lo, int row_hi, float cscale) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int row = (int)(i / row_elems);
    const float yv = __bfloat162float(y[i]);
    const float v = (row >= row_lo && row < row_hi) ? cscale * (yv - __bfloat162float(t[i])) : 0.f;
    g[i] = __float2bfloat16(yv > 0.f ? v : 0.f);
  }
}

// step counter and bias corrections live on the device: *step += 1, then the scalars of torch's single-tensor Adam
// (torch/optim/adam.py:413-546) are evaluated in double exactly like the host path does
__global__ void adam_scalars_kernel(long long* step, AdamScalars* out, float lr, float beta1, float beta2,
                                    float adam_eps, float ema_decay) {
  const long long t = *step + 1;
  *step = t;
  *out = make_adam_scalars(t, lr, beta1, beta2, adam_eps, ema_decay);
}

// the iteration counter of the loss ring's stamps on a path without Adam scalars (stb_iterate_lbfgs)
__global__ void advance_step_kernel(long long* step) { *step += 1; }

__global__ void scale_copy_kernel(const float* __restrict__ in, float* __restrict__ out, long n, float scale) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    out[i] = in[i] * scale;
}

// terms = [total, content_k * cw_k / numel_k ..., style_l ..., tvw * tv]; total = their python sum, left to right
// (SumLoss, ST:208/455).  `ring` (optional): pinned HOST memory, slots x 16 floats.  The kernel stores term k into word
// k (k < 8) or k + 1 (k >= 8) of slot (step % slots) and then, after a system-scope fence, the step itself as the
// slot's stamp (word 8): the host polls the stamp instead of synchronising the stream, so the callback of iteration i
// overlaps the backward pass of iteration i.
struct ContentScales { float s[kNumTaps]; int n_content, n_style; };
__global__ void finalize_loss_kernel(const float* __restrict__ scalars, ContentScales cs,
                                     const float* __restrict__ style_terms, float tv_weight,
                                     float* __restrict__ out, float* ring, int ring_slots,
                                     const long long* __restrict__ d_step) {
  if (threadIdx.x == 0) {
    const int nc = cs.n_content, ns = cs.n_style;
    float loss = 0.f;
    for (int k = 0; k < nc; ++k) {
      const float content = scalars[k] * cs.s[k];
      loss = k == 0 ? content : loss + content;
      out[1 + k] = content;
    }
    for (int l = 0; l < ns; ++l) {
      loss += style_terms[l];
      out[1 + nc + l] = style_terms[l];
    }
    const float tv = scalars[nc] * tv_weight;
    loss += tv;
    out[0] = loss;
    out[1 + nc + ns] = tv;
    if (ring != nullptr && d_step != nullptr) {
      const long long step = *d_step;
      volatile float* slot = ring + (size_t)(step % ring_slots) * 16;
      for (int i = 0; i < 2 + nc + ns; ++i) slot[i < 8 ? i : i + 1] = out[i];
      __threadfence_system();
      reinterpret_cast<volatile int*>(slot)[8] = (int)step;
    }
  }
}

// the W2 engine over the style taps of the layer table, in the fixed W2 block at the head of the workspace
int init_w2(stb_ctx* ctx) {
  const LayerTable& lt = ctx->layers;
  int cs[kNumTaps];
  for (int l = 0; l < lt.n_style; ++l) cs[l] = lt.style_c(l);
  return ctx->w2.init(ctx->ws, ctx->w2_bytes, lt.n_style, cs);
}

void comm_release(stb_ctx* ctx) {
  if (ctx->comm_ipc)
    for (int r = 0; r < ctx->comm.world; ++r)
      if (r != ctx->comm.rank && ctx->comm.mbox[r]) cudaIpcCloseMemHandle(ctx->comm.mbox[r]);
  if (ctx->comm_mailbox) cudaFree(ctx->comm_mailbox);
  ctx->comm_mailbox = nullptr;
  uint8_t* keep_ws[COMM_MAX_RANKS];
  std::memcpy(keep_ws, ctx->comm.ws, sizeof(keep_ws));
  ctx->comm = CommDev{};
  std::memcpy(ctx->comm.ws, keep_ws, sizeof(keep_ws));   // the shared workspace outlives a mailbox re-creation
  ctx->comm_ready = ctx->comm_geometry = ctx->comm_ipc = false;
}
void shared_ws_release(stb_ctx* ctx) {
  if (ctx->shared_ws_ipc)
    for (int r = 0; r < COMM_MAX_RANKS; ++r)
      if (ctx->comm.ws[r] && ctx->comm.ws[r] != ctx->shared_ws) cudaIpcCloseMemHandle(ctx->comm.ws[r]);
  for (int r = 0; r < COMM_MAX_RANKS; ++r) ctx->comm.ws[r] = nullptr;
  if (ctx->shared_ws) {
    if (ctx->ws == ctx->shared_ws) { ctx->ws = nullptr; ctx->ws_bytes = 0; ctx->w2_ready = false; ctx->targets_set = false; }
    cudaFree(ctx->shared_ws);
  }
  ctx->shared_ws = nullptr; ctx->shared_ws_bytes = 0; ctx->shared_ws_ipc = false;
}
}  // namespace

extern "C" {

const char* stb_last_error(void) { return last_error_string().c_str(); }

int stb_ctx_create(int device, int pooling, const float* const* conv_w, const float* const* conv_b, void* stream,
                   stb_ctx** out) {
  STB_CHECK(out != nullptr && conv_w != nullptr && conv_b != nullptr, STB_ERR_INVALID, "null argument");
  STB_CHECK(pooling >= 0 && pooling <= 2, STB_ERR_INVALID, "pooling must be STB_POOL_MAX/AVERAGE/L2");
  STB_CUDA_CHECK(cudaSetDevice(device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  stb_ctx* ctx = new stb_ctx();
  ctx->device = device;
  ctx->pooling = pooling;
  const int rc = [&]() -> int {
  size_t bytes = 0;
  for (int i = 0; i < NCONV; ++i) {
    bytes += align_up((size_t)kCout[i] * 4, 256);
    if (i == 0) bytes += align_up((size_t)64 * 27 * 4, 256) + align_up((size_t)9 * 64 * 64 * 2, 256) + 8192 + 512;
    else bytes += 2 * align_up((size_t)9 * kCout[i] * kCin[i] * 2, 256);
  }
  cudaError_t e = cudaMalloc(&ctx->owned, bytes);
  if (e != cudaSuccess) return set_error(STB_ERR_CUDA, "cudaMalloc(%zu): %s", bytes, cudaGetErrorString(e));
  uint8_t* p = static_cast<uint8_t*>(ctx->owned);
  auto take = [&](size_t b) { void* r = p; p += align_up(b, 256); return r; };
  for (int i = 0; i < NCONV; ++i) {
    ctx->bias[i] = (float*)take((size_t)kCout[i] * 4);
    STB_CUDA_CHECK(cudaMemcpyAsync(ctx->bias[i], conv_b[i], (size_t)kCout[i] * 4, cudaMemcpyDeviceToDevice, s));
    if (i == 0) {
      ctx->w0 = (float*)take(64 * 27 * 4);
      STB_CUDA_CHECK(cudaMemcpyAsync(ctx->w0, conv_w[0], 64 * 27 * 4, cudaMemcpyDeviceToDevice, s));
      ctx->wb[0] = (bf16*)take((size_t)32 * 64 * 2);
      STB_TRY(pack_weights_conv0_bwd(ctx->w0, ctx->wb[0], s));
      ctx->wf[0] = (bf16*)take((size_t)64 * 64 * 2);
      STB_TRY(pack_weights_conv0_fwd(ctx->w0, ctx->wf[0], s));
    } else {
      ctx->wf[i] = (bf16*)take((size_t)9 * kCout[i] * kCin[i] * 2);
      ctx->wb[i] = (bf16*)take((size_t)9 * kCout[i] * kCin[i] * 2);
      STB_TRY(pack_weights_fwd(conv_w[i], ctx->wf[i], kCout[i], kCin[i], s));
      STB_TRY(pack_weights_bwd(conv_w[i], ctx->wb[i], kCout[i], kCin[i], s));
    }
  }
  ctx->d_adam = (AdamScalars*)take(256);
  ctx->d_step = (long long*)take(256);
  {
    const char* e = getenv("STB_GRAPH");
    ctx->graphs_enabled = !(e && e[0] == '0');
  }
  ctx->w2_bytes = W2Engine::workspace_bytes();
  STB_CUDA_CHECK(cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
  STB_CUDA_CHECK(cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming));
  STB_CUDA_CHECK(cudaStreamSynchronize(s));
  return STB_OK;
  }();
  if (rc != STB_OK) {  // nothing of a half-built context survives
    stb_ctx_destroy(ctx);
    return rc;
  }
  *out = ctx;
  return STB_OK;
}

void stb_ctx_destroy(stb_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  shared_ws_release(ctx);
  comm_release(ctx);
  if (ctx->owned) cudaFree(ctx->owned);
  if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
  if (ctx->ev_join) cudaEventDestroy(ctx->ev_join);
  ctx->reset_graphs();
  delete ctx;
}

int stb_workspace_bytes(stb_ctx* ctx, int H, int W, size_t* bytes) {
  STB_CHECK(ctx && bytes, STB_ERR_INVALID, "null argument");
  STB_ENTER(ctx);
  STB_TRY(check_size(H, W, 0));
  Plan pl;
  make_plan(ctx, H, W, &pl);
  *bytes = pl.total;
  return STB_OK;
}

int stb_bind_workspace(stb_ctx* ctx, void* ptr, size_t bytes, void* stream) {
  STB_CHECK(ctx != nullptr, STB_ERR_INVALID, "null ctx");
  STB_CHECK(ptr != nullptr && (reinterpret_cast<uintptr_t>(ptr) & 1023) == 0, STB_ERR_INVALID,
            "workspace must be a 1 KiB aligned device pointer");
  STB_CHECK(bytes >= ctx->w2_bytes + 4096, STB_ERR_WORKSPACE, "workspace smaller than the fixed W2 block");
  STB_ENTER(ctx);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  STB_CUDA_CHECK(cudaStreamSynchronize(s));
  ctx->ws = static_cast<uint8_t*>(ptr);
  ctx->ws_bytes = bytes;
  ctx->reset_graphs();
  ctx->targets_set = false;
  STB_TRY(init_w2(ctx));
  ctx->w2_ready = true;
  return STB_OK;
}

int stb_set_layers(stb_ctx* ctx, int n_content, const int* content_layers, int n_style, const int* style_layers) {
  STB_CHECK(ctx != nullptr, STB_ERR_INVALID, "null ctx");
  STB_CHECK(n_content >= 1 && n_content <= kNumTaps && content_layers != nullptr, STB_ERR_INVALID,
            "content_layers must list 1 to %d taps, got %d", kNumTaps, n_content);
  STB_CHECK(n_style >= 0 && n_style <= kNumTaps && (n_style == 0 || style_layers != nullptr), STB_ERR_INVALID,
            "style_layers must list 0 to %d taps, got %d", kNumTaps, n_style);
  LayerTable lt;
  auto to_conv = [](const int* layers, int n, int* conv_out, const char* what) -> int {
    for (int k = 0; k < n; ++k) {
      int t = 0;
      while (t < kNumTaps && kTapLayer[t] != layers[k]) ++t;
      STB_CHECK(t < kNumTaps, STB_ERR_INVALID, "%s: layer %d is not one of the taps 1, 6, 11, 20, 22, 29", what,
                layers[k]);
      for (int j = 0; j < k; ++j)
        STB_CHECK(layers[j] != layers[k], STB_ERR_INVALID, "%s: layer %d is listed twice", what, layers[k]);
      conv_out[k] = kTapConv[t];
    }
    return STB_OK;
  };
  STB_TRY(to_conv(content_layers, n_content, lt.content_conv, "content_layers"));
  STB_TRY(to_conv(style_layers, n_style, lt.style_conv, "style_layers"));
  lt.n_content = n_content;
  lt.n_style = n_style;
  STB_ENTER(ctx);
  ctx->layers = lt;
  ctx->reset_graphs();
  ctx->targets_set = false;
  if (ctx->ws != nullptr) {
    ctx->w2_ready = false;
    STB_TRY(init_w2(ctx));
    ctx->w2_ready = true;
  }
  return STB_OK;
}

int stb_style_stats(stb_ctx* ctx, const float* img, int H, int W, float* const* mean_out, float* const* srm_out,
                    void* stream) {
  STB_CHECK(ctx && img && (ctx->layers.n_style == 0 || (mean_out && srm_out)), STB_ERR_INVALID, "null argument");
  STB_ENTER(ctx);
  const LayerTable& lt = ctx->layers;
  if (lt.n_style == 0) return STB_OK;
  STB_TRY(check_size(H, W, lt.last_style_conv()));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  Plan pl;
  make_plan(ctx, H, W, &pl);
  STB_TRY(ensure_ws(ctx, pl));
  STB_TRY(forward(ctx, pl, img, lt.last_style_conv(), false, s));
  STB_TRY(style_grams(ctx, pl, s));
  const float* stats = at<float>(ctx, pl.stats_off);
  for (int l = 0; l < lt.n_style; ++l) {
    const int C = lt.style_c(l);
    const int ci = lt.style_conv[l];
    // banded contexts return RAW sums over their own rows (the host all-reduces and normalises by the global count)
    const float inv = ctx->band_on ? 1.f : 1.f / ((float)pl.h[ci] * (float)pl.w[ci]);
    const float* S = stats + pl.stats_layer_off[l];
    scale_copy_kernel<<<(C * C + 255) / 256, 256, 0, s>>>(S, srm_out[l], (long)C * C, inv);
    scale_copy_kernel<<<1, 256, 0, s>>>(S + (size_t)C * C, mean_out[l], C, inv);
  }
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

int stb_content_features_ex(stb_ctx* ctx, const float* img, int H, int W, void* const* targets_out, void* stream) {
  STB_CHECK(ctx && img && targets_out, STB_ERR_INVALID, "null argument");
  STB_ENTER(ctx);
  const LayerTable& lt = ctx->layers;
  for (int k = 0; k < lt.n_content; ++k) STB_CHECK(targets_out[k] != nullptr, STB_ERR_INVALID, "null target %d", k);
  STB_TRY(check_size(H, W, lt.last_content_conv()));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  Plan pl;
  make_plan(ctx, H, W, &pl);
  STB_TRY(ensure_ws(ctx, pl));
  STB_TRY(forward(ctx, pl, img, lt.last_content_conv(), false, s));
  for (int k = 0; k < lt.n_content; ++k) {
    const int ci = lt.content_conv[k];
    const size_t bytes = (size_t)pl.h[ci] * pl.w[ci] * kCout[ci] * 2;
    STB_CUDA_CHECK(cudaMemcpyAsync(targets_out[k], at<bf16>(ctx, pl.act_off[ci]), bytes, cudaMemcpyDeviceToDevice, s));
  }
  return STB_OK;
}

int stb_content_features(stb_ctx* ctx, const float* img, int H, int W, void* target_out_bf16, void* stream) {
  STB_CHECK(ctx && target_out_bf16, STB_ERR_INVALID, "null argument");
  STB_CHECK(ctx->layers.is_default(), STB_ERR_STATE, "stb_content_features needs the default layers (use _ex)");
  return stb_content_features_ex(ctx, img, H, W, &target_out_bf16, stream);
}

int stb_set_targets_ex(stb_ctx* ctx, int H, int W, const void* const* content_targets, const float* content_w,
                       const float* const* mean_t, const float* const* srm_t, const float* style_w, float tv_weight,
                       float eps, void* stream) {
  const LayerTable& lt = ctx ? ctx->layers : LayerTable{};
  STB_CHECK(ctx && content_targets && content_w && (lt.n_style == 0 || (mean_t && srm_t && style_w)), STB_ERR_INVALID,
            "null argument");
  for (int k = 0; k < lt.n_content; ++k) STB_CHECK(content_targets[k] != nullptr, STB_ERR_INVALID, "null target %d", k);
  STB_ENTER(ctx);
  STB_TRY(check_size(H, W, NCONV - 1));   // the closure's model holds all six taps (ST:324, 473)
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  Plan pl;
  make_plan(ctx, H, W, &pl);
  STB_TRY(ensure_ws(ctx, pl));
  STB_CHECK(ctx->w2_ready, STB_ERR_STATE, "workspace not bound");
  ctx->reset_graphs();  // weights are baked into the graphs
  for (int k = 0; k < lt.n_content; ++k) {
    const int ci = lt.content_conv[k];
    const size_t cbytes = (size_t)pl.h[ci] * pl.w[ci] * kCout[ci] * 2;
    STB_CUDA_CHECK(cudaMemcpyAsync(at<bf16>(ctx, pl.ctarget_off[k]), content_targets[k], cbytes,
                                   cudaMemcpyDeviceToDevice, s));
    ctx->content_w[k] = content_w[k];
  }
  float* stats = at<float>(ctx, pl.stats_off);
  for (int l = 0; l < lt.n_style; ++l) {
    W2Layer& L = ctx->w2.host_layers[l];
    const int C = lt.style_c(l);
    const int ci = lt.style_conv[l];
    L.eps = eps;
    L.weight = style_w[l];
    L.npix = (float)band_rows(ctx, pl, ci).h_global * (float)pl.w[ci];
    L.S_raw = stats + pl.stats_layer_off[l];
    L.sums = L.S_raw + (size_t)C * C;
    STB_CUDA_CHECK(cudaMemcpyAsync(L.mean_t, mean_t[l], (size_t)C * 4, cudaMemcpyDeviceToDevice, s));
    STB_CUDA_CHECK(cudaMemcpyAsync(L.srm_t, srm_t[l], (size_t)C * C * 4, cudaMemcpyDeviceToDevice, s));
  }
  STB_TRY(ctx->w2.upload_layers(s));
  STB_TRY(ctx->w2.build_targets(s));
  if (ctx->band_on)  // TV gradient of the halo rows belongs to the neighbouring band: keep it zero here
    STB_CUDA_CHECK(cudaMemsetAsync(at<float>(ctx, pl.gtv_off), 0, (size_t)3 * H * W * 4, s));
  ctx->tv_weight = tv_weight;
  ctx->tH = H; ctx->tW = W;
  ctx->targets_set = true;
  return STB_OK;
}

int stb_set_targets(stb_ctx* ctx, int H, int W, const void* content_target_bf16, float content_weight,
                    const float* const* mean_t, const float* const* srm_t, const float* style_w, float tv_weight,
                    float eps, void* stream) {
  STB_CHECK(ctx && content_target_bf16, STB_ERR_INVALID, "null argument");
  STB_CHECK(ctx->layers.is_default(), STB_ERR_STATE, "stb_set_targets needs the default layers (use _ex)");
  return stb_set_targets_ex(ctx, H, W, &content_target_bf16, &content_weight, mean_t, srm_t, style_w, tv_weight, eps,
                            stream);
}

int stb_loss_terms(stb_ctx* ctx, float* out, int capacity, int* n_terms, void* stream) {
  STB_CHECK(ctx && n_terms && (out || capacity == 0) && capacity >= 0, STB_ERR_INVALID, "bad argument");
  STB_ENTER(ctx);
  STB_CHECK(ctx->targets_set, STB_ERR_STATE, "stb_set_targets must precede stb_loss_terms");
  const int n = 2 + ctx->layers.n_content + ctx->layers.n_style;
  *n_terms = n;
  if (capacity == 0) return STB_OK;
  Plan pl;
  make_plan(ctx, ctx->tH, ctx->tW, &pl);
  STB_CUDA_CHECK(cudaMemcpyAsync(out, at<float>(ctx, pl.loss_off), sizeof(float) * std::min(n, capacity),
                                 cudaMemcpyDeviceToHost, static_cast<cudaStream_t>(stream)));
  return STB_OK;
}

}  // extern "C"

namespace {

// phase 1: forward + this context's (band-local) statistics into the stats block
int iterate_fwd(stb_ctx* ctx, const Plan& pl, const float* img, cudaStream_t s, const HaloPlans* halo) {
  const LayerTable& lt = ctx->layers;
  STB_TRY(forward(ctx, pl, img, lt.last_conv(), true, s, halo));
  STB_TRY(style_grams(ctx, pl, s));
  PartialArrays parts{};
  ctx->prof.begin(PC_SSE, s);
  for (int k = 0; k < lt.n_content; ++k) {
    const int ci = lt.content_conv[k], C = kCout[ci];
    const BandRows b = band_rows(ctx, pl, ci);
    const size_t off = (size_t)b.own0 * pl.w[ci] * C;
    parts.p[k] = at<float>(ctx, pl.ssep_off) + (size_t)k * kSsePartials;
    STB_TRY(launch_sse(at<bf16>(ctx, pl.act_off[ci]) + off, at<bf16>(ctx, pl.ctarget_off[k]) + off,
                       (long)b.rows * pl.w[ci] * C, const_cast<float*>(parts.p[k]), &parts.n[k], s));
  }
  parts.p[lt.n_content] = at<float>(ctx, pl.tvp_off);
  parts.n[lt.n_content] = ctx->n_tv_partials;
  parts.count = lt.n_content + 1;
  parts.tail = (int)lt.stats_tail();
  reduce_partials_kernel<<<1, 1024, 0, s>>>(parts, at<float>(ctx, pl.stats_off) + pl.stats_scalars);
  ctx->prof.end(s);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

// Adam + clamp + EMA fused into the epilogue of conv0's dgrad (d_adam: the device scalars of this step)
struct FusedAdam { float *exp_avg, *exp_avg_sq, *ema; const AdamScalars* d_adam; };

// phase 2: W2 losses on the (globally reduced) statistics, backward to the image, optional fused update.
// publish_loss: the loss kernel also writes the loss ring (stb_set_loss_ring) under the device step counter.
int iterate_bwd(stb_ctx* ctx, const Plan& pl, float* img, const FusedAdam* update, bool publish_loss, float* grad_out,
                float* loss_out_host8, cudaStream_t s, const HaloPlans* halo) {
  const int H = pl.H, W = pl.W;
  const LayerTable& lt = ctx->layers;
  // 2 * content weight / numel of content tap k (global numel under tiling): the scale of its dgrad injection
  auto content_numel = [&](int k) {
    const int ci = lt.content_conv[k];
    return (long)band_rows(ctx, pl, ci).h_global * pl.w[ci] * kCout[ci];
  };
  float* loss_dev = at<float>(ctx, pl.loss_off);
  ctx->prof.begin(PC_W2, s);
  STB_TRY(ctx->w2.forward_backward(loss_dev + 16, s));
  ctx->prof.end(s);
  // every loss term is known here (content SSE and TV from the forward, the style terms from the W2 forward): assemble
  // and publish the loss BEFORE the backward pass, so a host callback can consume it while the device works on
  ContentScales cs{};
  cs.n_content = lt.n_content; cs.n_style = lt.n_style;
  for (int k = 0; k < lt.n_content; ++k) cs.s[k] = ctx->content_w[k] / (float)content_numel(k);
  ctx->prof.begin(PC_FINALIZE, s);
  finalize_loss_kernel<<<1, 32, 0, s>>>(at<float>(ctx, pl.stats_off) + pl.stats_scalars, cs, loss_dev + 16,
                                        ctx->tv_weight, loss_dev, publish_loss ? ctx->ring_dev : nullptr,
                                        ctx->ring_slots, ctx->d_step);
  ctx->prof.end(s);
  if (loss_out_host8)
    STB_CUDA_CHECK(cudaMemcpyAsync(loss_out_host8, loss_dev, 8 * sizeof(float), cudaMemcpyDeviceToHost, s));

  bf16* g[2] = {at<bf16>(ctx, pl.g_off[0]), at<bf16>(ctx, pl.g_off[1])};
  int cur = 0;
  const int last = lt.last_conv();
  {  // the deepest tap: d loss / d pre-activation of its conv, own rows only.  With a style role it is
     // mask * (F Gs / N + gmu / N) [+ the content injection], a pixel GEMM on the tap alone; content only: the seed kernel
    const BandRows br = band_rows(ctx, pl, last);
    const int C = kCout[last], ls = lt.style_at(last), kc = lt.content_at(last);
    ctx->prof.begin(PC_CONV_BWD, s);
    if (ls >= 0) {
      const W2Layer& L = ctx->w2.host_layers[ls];
      PixelGemmArgs a;
      a.H = pl.h[last]; a.W = pl.w[last]; a.Cin = 0; a.Cout = C; a.C2 = C; a.mode = 1;
      a.A2 = at<bf16>(ctx, pl.act_off[last]) + (size_t)br.own0 * pl.w[last] * C;
      a.a2_row0 = br.own0; a.a2_rows = br.rows; a.row_lo = br.own0; a.row_hi = br.own0 + br.rows;
      a.B2 = L.gs_bf16; a.bias = L.gmu_bias;
      a.mask_src = at<bf16>(ctx, pl.act_off[last]); a.out = g[cur];
      if (kc >= 0) {
        a.ctarget = at<bf16>(ctx, pl.ctarget_off[kc]);
        a.cscale = 2.f * ctx->content_w[kc] / (float)content_numel(kc);
      }
      if (halo) { a.y_origin = br.own0; a.y_rows = br.rows; }
      STB_TRY(launch_pixel_gemm(a, s));
    } else {
      const long row_elems = (long)pl.w[last] * C, n = (long)pl.h[last] * row_elems;
      long blocks = (n + 255) / 256;
      if (blocks > 16l * num_sms()) blocks = 16l * num_sms();
      content_seed_kernel<<<(unsigned)blocks, 256, 0, s>>>(
          at<bf16>(ctx, pl.act_off[last]), at<bf16>(ctx, pl.ctarget_off[kc]), g[cur], n, row_elems, br.own0,
          br.own0 + br.rows, 2.f * ctx->content_w[kc] / (float)content_numel(kc));
      STB_CUDA_CHECK(cudaGetLastError());
    }
    ctx->prof.end(s);
    if (halo)
      STB_TRY(halo_exchange(ctx, level_of(last), pl.w[last], C, pl.g_off[cur], halo->up.g_off[cur],
                            halo->dn.g_off[cur], false, s));
  }
  for (int i = last; i >= 1; --i) {
    // g[cur] = gradient w.r.t. conv i pre-activation, [h_i][w_i][Cout_i]; produce gradient for conv i-1
    PixelGemmArgs a;
    a.H = pl.h[i]; a.W = pl.w[i]; a.Cin = kCout[i]; a.Cout = kCin[i];
    a.A = g[cur]; a.Bw = ctx->wb[i]; a.out = g[cur ^ 1];
    const BandRows bi = band_rows(ctx, pl, i);
    if (halo) { a.y_origin = bi.own0; a.y_rows = bi.rows; }
    if (kPoolAfter[i - 1]) {
      a.mode = 2;
      ctx->prof.begin(PC_CONV_BWD, s);
      STB_TRY(launch_pixel_gemm(a, s));
      ctx->prof.end(s);
      cur ^= 1;
      ctx->prof.begin(PC_POOL_BWD, s);
      if (!halo) {
        STB_TRY(launch_pool_bwd(ctx->pooling, g[cur], at<bf16>(ctx, pl.act_off[i - 1]), g[cur ^ 1], pl.h[i - 1],
                                pl.w[i - 1], kCout[i - 1], s));
      } else {
        // g[cur ^ 1] is the buffer the neighbours pulled their halo rows from one exchange ago: make sure they are done
        STB_TRY(halo_exchange(ctx, level_of(i), pl.w[i], kCout[i - 1], pl.g_off[cur], halo->up.g_off[cur],
                              halo->dn.g_off[cur], true, s));
        const BandRows bp = band_rows(ctx, pl, i - 1);   // own rows before the pool
        const int C = kCout[i - 1];
        STB_TRY(launch_pool_bwd(ctx->pooling, g[cur] + (size_t)bi.own0 * pl.w[i] * C,
                                at<bf16>(ctx, pl.act_off[i - 1]) + (size_t)bp.own0 * pl.w[i - 1] * C,
                                g[cur ^ 1] + (size_t)bp.own0 * pl.w[i - 1] * C, bp.rows, pl.w[i - 1], C, s));
      }
      ctx->prof.end(s);
      cur ^= 1;
      if (halo)
        STB_TRY(halo_exchange(ctx, level_of(i - 1), pl.w[i - 1], kCout[i - 1], pl.g_off[cur], halo->up.g_off[cur],
                              halo->dn.g_off[cur], false, s));
    } else {
      a.mode = 1;
      a.mask_src = at<bf16>(ctx, pl.act_off[i - 1]);
      const BandRows br = band_rows(ctx, pl, i - 1);
      a.row_lo = br.own0; a.row_hi = br.own0 + br.rows;
      const int ls = lt.style_at(i - 1), kc = lt.content_at(i - 1);
      if (ls >= 0) {
        const W2Layer& L = ctx->w2.host_layers[ls];
        a.C2 = lt.style_c(ls);
        a.A2 = at<bf16>(ctx, pl.act_off[i - 1]) + (size_t)br.own0 * pl.w[i - 1] * a.C2;
        a.a2_row0 = br.own0; a.a2_rows = br.rows;
        a.B2 = L.gs_bf16; a.bias = L.gmu_bias;
      }
      if (kc >= 0) {
        a.ctarget = at<bf16>(ctx, pl.ctarget_off[kc]);
        a.cscale = 2.f * ctx->content_w[kc] / (float)content_numel(kc);
      }
      ctx->prof.begin(PC_CONV_BWD, s);
      STB_TRY(launch_pixel_gemm(a, s));
      ctx->prof.end(s);
      cur ^= 1;
      if (halo)
        STB_TRY(halo_exchange(ctx, level_of(i - 1), pl.w[i - 1], kCin[i], pl.g_off[cur], halo->up.g_off[cur],
                              halo->dn.g_off[cur], false, s));
    }
  }
  // conv0 backward: interior pixels on the tensor cores (1x1 GEMM + col2im) with the optimiser step as epilogue;
  // the border pixels (adjoint of the replicate pad) and their update in SIMT
  const FusedAdam u = update ? *update : FusedAdam{};
  ctx->prof.begin(PC_CONV0_BWD_ADAM, s);
  STB_TRY(launch_conv0_bwd_interior(g[cur], ctx->wb[0], at<float>(ctx, pl.gtv_off), img, u.exp_avg, u.exp_avg_sq,
                                    u.ema, grad_out, H, W, u.d_adam, update != nullptr, s));
  STB_TRY(launch_conv0_bwd_adam(g[cur], true, ctx->w0, at<float>(ctx, pl.gtv_off), img, u.exp_avg, u.exp_avg_sq, u.ema,
                                grad_out, H, W, u.d_adam, update != nullptr, s));
  ctx->prof.end(s);
  STB_CUDA_CHECK(cudaGetLastError());
  return STB_OK;
}

}  // namespace

// ---- CUDA graphs: an iteration (or one of its multi-GPU phases) is ~50-110 launches with fixed arguments; replaying
// a captured graph removes the per-launch host cost and the tensor-map encodes (matters most at the small pyramid
// levels and when the image is tiled over many GPUs).  `key` holds everything that is baked into the launches.
template <typename Run>
int run_graphed(stb_ctx* ctx, GraphSlotId slot, const stb_ctx::GraphKey& key, bool allowed, cudaStream_t s, Run&& run) {
  const bool legacy = (s == nullptr || s == cudaStreamLegacy || s == cudaStreamPerThread);
  if (!ctx->graphs_enabled || ctx->prof.on || legacy || !allowed) return run();
  stb_ctx::GraphSlot& g = ctx->gslot[slot];
  if (!(key == g.key)) {
    g.reset();
    g.key = key;
  }
  if (g.exec) {
    STB_CUDA_CHECK(cudaGraphLaunch(g.exec, s));
    ctx->graph_replays += 1;
    ctx->kernels_replayed += g.kernel_nodes;
    return STB_OK;
  }
  if (++g.hits < 3) return run();  // eager first (lazy one-time setup must not happen inside a capture)
  cudaGraph_t graph = nullptr;
  if (cudaStreamBeginCapture(s, cudaStreamCaptureModeRelaxed) != cudaSuccess) {
    ctx->graph_note = std::string("cudaStreamBeginCapture failed: ") + cudaGetErrorString(cudaGetLastError());
    ctx->graphs_enabled = false;
    return run();
  }
  const int rc = run();
  const cudaError_t ce = cudaStreamEndCapture(s, &graph);
  if (rc != STB_OK || ce != cudaSuccess || graph == nullptr ||
      cudaGraphInstantiate(&g.exec, graph, 0) != cudaSuccess) {
    ctx->graph_note = std::string("graph capture/instantiate failed (rc ") + std::to_string(rc) + ", " +
                      cudaGetErrorString(ce) + " / " + cudaGetErrorString(cudaGetLastError()) + ")";
    if (graph) cudaGraphDestroy(graph);
    g.exec = nullptr;
    ctx->graphs_enabled = false;  // eager launches from here on for this context; visible through stb_graph_status
    return run();
  }
  {  // how many kernel launches one replay stands for
    size_t n = 0;
    if (cudaGraphGetNodes(graph, nullptr, &n) == cudaSuccess && n > 0) {
      std::vector<cudaGraphNode_t> nodes(n);
      if (cudaGraphGetNodes(graph, nodes.data(), &n) == cudaSuccess)
        for (size_t i = 0; i < n; ++i) {
          cudaGraphNodeType t;
          if (cudaGraphNodeGetType(nodes[i], &t) == cudaSuccess && t == cudaGraphNodeTypeKernel) g.kernel_nodes += 1;
        }
    }
  }
  cudaGraphDestroy(graph);
  STB_CUDA_CHECK(cudaGraphLaunch(g.exec, s));
  ctx->graph_replays += 1;
  ctx->kernels_replayed += g.kernel_nodes;
  return STB_OK;
}

namespace stb {
// the test library's banded L-BFGS hook (api_test.cu) runs on a context's comm connection and geometry
const CommDev* ctx_comm(const stb_ctx* ctx) { return ctx->comm_ready && ctx->comm_geometry ? &ctx->comm : nullptr; }
}  // namespace stb

// ---- the iteration entry points.  Each records one variant of the launch sequence
//   [comm phase 0 + halo pull] -> forward + statistics -> [all-reduce of the statistics] -> step kernel ->
//   W2 + backward -> [comm phase 2 -> update -> comm phase 3]
// (brackets: a band's iteration with the exchanges inside, comm.cu), or the untiled L-BFGS step after the backward.
namespace {

enum StepKernel { STEP_NONE, STEP_ADAM_SCALARS, STEP_ADVANCE };   // both advance the device step counter
enum Update { UPDATE_NONE, UPDATE_ADAM_FUSED, UPDATE_ADAM_SEAM, UPDATE_LBFGS, UPDATE_LBFGS_BANDED };
struct Variant {
  const char* name;   // the entry point, for the error texts
  GraphSlotId slot;
  bool fwd, bwd;      // records the forward / the backward half (stb_iterate_fwd / stb_iterate_bwd record one each)
  bool banded;
  StepKernel step;
  Update update;      // ADAM_FUSED: in the epilogue of conv0's dgrad; ADAM_SEAM / LBFGS_BANDED: after the seam exchange
};
constexpr Variant kIterate{"stb_iterate", GS_ITERATE, true, true, false, STEP_ADAM_SCALARS, UPDATE_ADAM_FUSED};
constexpr Variant kClosure{"stb_iterate", GS_ITERATE, true, true, false, STEP_NONE, UPDATE_NONE};   // never graphed
constexpr Variant kFwd{"stb_iterate_fwd", GS_ITERATE_FWD, true, false, false, STEP_NONE, UPDATE_NONE};
constexpr Variant kBwd{"stb_iterate_bwd", GS_ITERATE_BWD, false, true, false, STEP_NONE, UPDATE_NONE};
constexpr Variant kLbfgs{"stb_iterate_lbfgs", GS_ITERATE_LBFGS, true, true, false, STEP_ADVANCE, UPDATE_LBFGS};
constexpr Variant kBanded{"stb_iterate_banded", GS_ITERATE_BANDED, true, true, true, STEP_ADAM_SCALARS,
                          UPDATE_ADAM_SEAM};
constexpr Variant kLbfgsBanded{"stb_iterate_lbfgs_banded", GS_ITERATE_LBFGS_BANDED, true, true, true, STEP_ADVANCE,
                               UPDATE_LBFGS_BANDED};

// the caller's arguments in the order of the C ABI (null / 0 where the entry point has no such argument)
struct IterArgs {
  float *img, *exp_avg, *exp_avg_sq, *ema;
  int64_t step;
  float lr, beta1, beta2, adam_eps, ema_decay;
  float *grad_out, *loss_out_host8;
  void* state;   // L-BFGS
  size_t state_bytes;
};

// the optimizer state the update reads; a band's L-BFGS state holds its own rows
int check_optimizer_state(const stb_ctx* ctx, const Variant& v, const IterArgs& a) {
  if (v.update == UPDATE_ADAM_FUSED || v.update == UPDATE_ADAM_SEAM)
    STB_CHECK(a.exp_avg && a.exp_avg_sq && a.ema && a.step >= 1, STB_ERR_INVALID, "bad optimizer state");
  if (v.update == UPDATE_LBFGS || v.update == UPDATE_LBFGS_BANDED) {
    STB_CHECK(a.step >= 1, STB_ERR_INVALID, "step must be >= 1");
    STB_CHECK((reinterpret_cast<uintptr_t>(a.state) & 255) == 0 && (reinterpret_cast<uintptr_t>(a.img) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(a.ema) & 15) == 0,
              STB_ERR_INVALID, "state must be 256-byte aligned, img and ema 16-byte aligned");
    const int rows = v.banded ? ctx->band_own_rows : ctx->tH;
    const size_t need = lbfgs_state_bytes(3l * rows * ctx->tW);
    STB_CHECK(a.state_bytes >= need, STB_ERR_INVALID,
              "L-BFGS state of %zu bytes is too small for %d rows x %d (needs %zu)", a.state_bytes, rows, ctx->tW, need);
  }
  return STB_OK;
}

// state, workspace and argument checks of an entry point, before anything is launched
int check_iteration(stb_ctx* ctx, const Variant& v, const IterArgs& a, Plan* pl) {
  if (v.banded) {
    STB_CHECK(ctx->targets_set && ctx->band_on, STB_ERR_STATE, "stb_set_band + stb_set_targets must precede %s",
              v.name);
    STB_CHECK(ctx->comm_ready && ctx->comm_geometry, STB_ERR_STATE, "stb_comm_connect_* + stb_comm_set_geometry first");
  } else {
    STB_CHECK(ctx->targets_set, STB_ERR_STATE, "stb_set_targets must precede %s", v.name);
    STB_CHECK(v.update == UPDATE_NONE || !ctx->band_on, STB_ERR_STATE,
              "%s updates the whole image but the context has a band set (stb_iterate_banded / "
              "stb_iterate_lbfgs_banded iterate a band)", v.name);
    STB_TRY(check_optimizer_state(ctx, v, a));
  }
  make_plan(ctx, ctx->tH, ctx->tW, pl);
  STB_TRY(ensure_ws(ctx, *pl));
  if (!v.banded) return STB_OK;
  const CommDev& c = ctx->comm;
  STB_CHECK(c.h_local == pl->H && c.W == pl->W && c.own0 == ctx->band_own0 && c.own_rows == ctx->band_own_rows,
            STB_ERR_STATE, "comm geometry (%dx%d, own %d+%d) does not match the band (%dx%d, own %d+%d)", c.h_local,
            c.W, c.own0, c.own_rows, pl->H, pl->W, ctx->band_own0, ctx->band_own_rows);
  STB_TRY(check_optimizer_state(ctx, v, a));
  STB_CHECK(!ctx->halo_mode || (ctx->ws == ctx->shared_ws && ctx->shared_ws != nullptr), STB_ERR_STATE,
            "halo mode needs the library-owned workspace bound (stb_comm_alloc_workspace)");
  return STB_OK;
}

// graphable = false: eager launches, the graph slot is left alone
int iterate(stb_ctx* ctx, const Variant& v, const IterArgs& a, bool graphable, void* stream) {
  STB_ENTER(ctx);
  Plan pl;
  STB_TRY(check_iteration(ctx, v, a, &pl));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (v.step != STEP_NONE) {
    // the device step counter must read step-1 before this iteration (it is carried across scales like ST:461-462)
    if (ctx->dev_step_mirror != a.step - 1) {
      const long long prev = a.step - 1;
      STB_CUDA_CHECK(cudaMemcpyAsync(ctx->d_step, &prev, sizeof(prev), cudaMemcpyHostToDevice, s));
      STB_CUDA_CHECK(cudaStreamSynchronize(s));  // `prev` is a stack variable; this path runs once per scale at most
    }
    ctx->dev_step_mirror = a.step;
  }
  const CommDev& c = ctx->comm;
  HaloPlans hp;
  const HaloPlans* halo = nullptr;
  if (v.banded && ctx->halo_mode) {
    // per-layer-halo mode: the neighbours' buffers sit at the offsets of THEIR plans (edge bands have one apron less)
    make_plan(ctx, c.rank > 0 ? c.up_h_local : pl.H, pl.W, &hp.up);
    make_plan(ctx, c.rank + 1 < c.world ? c.dn_h_local : pl.H, pl.W, &hp.dn);
    halo = &hp;
  }
  const long n = 3l * pl.H * pl.W;
  float* grad = v.banded ? reinterpret_cast<float*>(c.mbox[c.rank] + c.off_grad)
                : v.update == UPDATE_LBFGS ? lbfgs_grad_buffer(a.state, n) : a.grad_out;
  const FusedAdam fused{a.exp_avg, a.exp_avg_sq, a.ema, ctx->d_adam};
  // the loss ring's stamp is the device step counter: the calls that advance it write the ring, and so does every call
  // on a band
  const bool publish_loss = v.step != STEP_NONE || ctx->band_on;
  auto run = [&]() -> int {
    ctx->halo_seq = 0;
    if (v.fwd) {
      if (v.banded) {
        STB_TRY(launch_comm_phase(c, 0, s));
        STB_TRY(launch_halo_pull(c, a.img, s));
      }
      STB_TRY(iterate_fwd(ctx, pl, a.img, s, halo));
      if (v.banded) STB_TRY(launch_stats_allreduce(c, at<float>(ctx, pl.stats_off), pl.stats_floats, s));
    }
    if (v.step == STEP_ADAM_SCALARS)
      adam_scalars_kernel<<<1, 1, 0, s>>>(ctx->d_step, ctx->d_adam, a.lr, a.beta1, a.beta2, a.adam_eps, a.ema_decay);
    else if (v.step == STEP_ADVANCE)
      advance_step_kernel<<<1, 1, 0, s>>>(ctx->d_step);
    if (v.bwd)
      STB_TRY(iterate_bwd(ctx, pl, a.img, v.update == UPDATE_ADAM_FUSED ? &fused : nullptr, publish_loss, grad,
                          a.loss_out_host8, s, halo));
    if (v.update == UPDATE_LBFGS) return launch_lbfgs_step(a.state, n, a.img, a.ema, a.ema_decay, s);
    if (!v.banded) return STB_OK;
    STB_TRY(launch_comm_phase(c, 2, s));
    if (v.update == UPDATE_ADAM_SEAM)
      STB_TRY(launch_adam_seam(c, a.img, a.exp_avg, a.exp_avg_sq, a.ema, ctx->d_adam, halo ? 0 : 1, s));
    else
      STB_TRY(launch_lbfgs_step_banded(a.state, c, a.img, a.ema, a.ema_decay, halo ? 0 : 1, s));
    return launch_comm_phase(c, 3, s);
  };
  stb_ctx::GraphKey key;
  std::memset(&key, 0, sizeof(key));   // compared bytewise
  key.H = pl.H; key.W = pl.W; key.ws = ctx->ws; key.img = a.img; key.exp_avg = a.exp_avg; key.exp_avg_sq = a.exp_avg_sq;
  key.ema = a.ema; key.grad_out = a.grad_out; key.state = a.state; key.loss = a.loss_out_host8;
  key.lr = a.lr; key.b1 = a.beta1; key.b2 = a.beta2; key.eps = a.adam_eps; key.decay = a.ema_decay;
  return run_graphed(ctx, v.slot, key, graphable, s, run);
}

}  // namespace

extern "C" {

// One pass of ST:480-486.  apply_update = 0 evaluates loss / gradient only (test hook, L-BFGS closure).
int stb_iterate_ex(stb_ctx* ctx, float* img, float* exp_avg, float* exp_avg_sq, float* ema, int64_t step, float lr,
                   float beta1, float beta2, float adam_eps, float ema_decay, int apply_update, float* grad_out,
                   float* loss_out_host8, void* stream) {
  STB_CHECK(ctx && img, STB_ERR_INVALID, "null argument");
  const IterArgs a{img, exp_avg, exp_avg_sq, ema, step, lr, beta1, beta2, adam_eps, ema_decay, grad_out, loss_out_host8};
  return iterate(ctx, apply_update ? kIterate : kClosure, a, apply_update && grad_out == nullptr, stream);
}

// ---- spatial tiling across GPUs (SURVEY.md section 8e).  A band's iteration is stb_iterate_banded; stb_iterate_fwd /
// stb_iterate_bwd are the closure split in two, with the statistics block (stb_stats_block) readable and writable
// between the halves
int stb_set_band(stb_ctx* ctx, int enabled, int H_global, int own_row0, int own_rows) {
  STB_CHECK(ctx != nullptr, STB_ERR_INVALID, "null ctx");
  if (enabled) {
    STB_CHECK(H_global > 0 && own_row0 >= 0 && own_rows > 0 && own_row0 % 16 == 0, STB_ERR_INVALID,
              "band rows must start on a multiple of 16 (four floor-mode pools), got own_row0=%d", own_row0);
  }
  ctx->band_on = enabled != 0;
  ctx->band_H_global = H_global; ctx->band_own0 = own_row0; ctx->band_own_rows = own_rows;
  ctx->targets_set = false;
  return STB_OK;
}

int stb_stats_block(stb_ctx* ctx, int H, int W, float** dev_ptr, size_t* n_floats) {
  STB_CHECK(ctx && dev_ptr && n_floats, STB_ERR_INVALID, "null argument");
  Plan pl;
  make_plan(ctx, H, W, &pl);
  STB_TRY(ensure_ws(ctx, pl));
  *dev_ptr = at<float>(ctx, pl.stats_off);
  *n_floats = pl.stats_floats;
  return STB_OK;
}

int stb_iterate_fwd(stb_ctx* ctx, const float* img, void* stream) {
  STB_CHECK(ctx && img, STB_ERR_INVALID, "null argument");
  return iterate(ctx, kFwd, IterArgs{const_cast<float*>(img)}, true, stream);   // the forward only reads img
}

int stb_iterate_bwd(stb_ctx* ctx, float* img, float* grad_out, float* loss_out_host8, void* stream) {
  STB_CHECK(ctx && img && grad_out, STB_ERR_INVALID, "null argument");
  IterArgs a{img};
  a.grad_out = grad_out;
  a.loss_out_host8 = loss_out_host8;
  return iterate(ctx, kBwd, a, true, stream);
}

// Per-scale warm start on the device (SURVEY.md 8f row 1): F.interpolate(in[1,C,H,W], (Ho,Wo), mode, align_corners=
// False) of the image (bicubic, clamp; ST:420) and of the Adam moments (exp_avg bicubic, exp_avg_sq bilinear + relu;
// ST:285-295).  mode: 0 bilinear, 1 bicubic; post: 0 none, 1 relu, 2 clamp to [0,1].
int stb_resize(const float* in, int C, int H, int W, float* out, int Ho, int Wo, int mode, int post, void* stream) {
  return launch_resize(in, C, H, W, out, Ho, Wo, mode, post, static_cast<cudaStream_t>(stream));
}

// Device snapshot of the averaged image for saving (get_image, AsyncImageWriter): one pass from the EMA's planar
// storage to interleaved uint8 / uint16, outside every iteration graph.
int stb_snapshot(const float* value, int H, int W, double denom, int kind, void* out, void* stream) {
  return launch_snapshot(value, H, W, denom, kind, out, static_cast<cudaStream_t>(stream));
}

// Source images (SURVEY.md 8f row 1, ST:417, 437): the content and style images are uploaded once as uint8 and every
// scale's tensors come from them by Pillow's bicubic resize restated on the device (csrc/resample.cu).
int stb_resample_tmp_bytes(int Hs, int Ws, int Ho, int Wo, int row0, int rows, size_t* bytes) {
  return resample_tmp_bytes(Hs, Ws, Ho, Wo, row0, rows, bytes);
}

int stb_resample_rgb8(const uint8_t* src, int Hs, int Ws, int Ho, int Wo, int row0, int rows, const int32_t* kx,
                      const int32_t* bx, int ksize_x, const int32_t* ky, const int32_t* by, int ksize_y, void* tmp,
                      size_t tmp_bytes, float* out, void* stream) {
  return launch_resample_rgb8(src, Hs, Ws, Ho, Wo, row0, rows, kx, bx, ksize_x, ky, by, ksize_y, tmp, tmp_bytes, out,
                              static_cast<cudaStream_t>(stream));
}

int stb_iterate(stb_ctx* ctx, float* img, float* exp_avg, float* exp_avg_sq, float* ema, int64_t step, float lr,
                float beta1, float beta2, float adam_eps, float ema_decay, float* loss_out_host8, void* stream) {
  return stb_iterate_ex(ctx, img, exp_avg, exp_avg_sq, ema, step, lr, beta1, beta2, adam_eps, ema_decay, 1, nullptr,
                        loss_out_host8, stream);
}

// ---- optimizer='lbfgs' (ST:464-465, SURVEY.md 8f row 4): closure + the L-BFGS step of lbfgs.cu + EMA, one graph
int stb_lbfgs_state_bytes(int H, int W, size_t* bytes) {
  STB_CHECK(bytes != nullptr && H > 0 && W > 0, STB_ERR_INVALID, "bad argument");
  *bytes = lbfgs_state_bytes(3l * H * W);
  return STB_OK;
}

int stb_lbfgs_reset(void* state, int H, int W, void* stream) {
  STB_CHECK(state != nullptr && H > 0 && W > 0, STB_ERR_INVALID, "bad argument");
  STB_CHECK((reinterpret_cast<uintptr_t>(state) & 255) == 0, STB_ERR_INVALID, "L-BFGS state must be 256-byte aligned");
  return launch_lbfgs_reset(state, static_cast<cudaStream_t>(stream));
}

int stb_iterate_lbfgs(stb_ctx* ctx, float* img, float* ema, void* state, size_t state_bytes, int64_t step,
                      float ema_decay, float* loss_out_host8, void* stream) {
  STB_CHECK(ctx && img && ema && state, STB_ERR_INVALID, "null argument");
  IterArgs a{img, nullptr, nullptr, ema, step};
  a.ema_decay = ema_decay; a.loss_out_host8 = loss_out_host8; a.state = state; a.state_bytes = state_bytes;
  return iterate(ctx, kLbfgs, a, true, stream);
}

// Per-kernel-class device timing (CUDA events on the launching stream).  enable: 1 starts recording spans for
// subsequent calls; stb_profile_read synchronises the recorded events, returns accumulated milliseconds and span
// counts per class (PC_* order: conv0_fwd_tv, conv_fwd, pool_fwd, gram, sse, w2, conv_bwd, pool_bwd,
// conv0_bwd_adam, finalize) and clears the record.
int stb_profile_enable(stb_ctx* ctx, int enable) {
  STB_CHECK(ctx != nullptr, STB_ERR_INVALID, "null ctx");
  ctx->prof.on = enable != 0;
  ctx->prof.spans.clear();
  ctx->prof.used = 0;
  return STB_OK;
}

int stb_profile_read(stb_ctx* ctx, float* ms_out, int* count_out, int n_classes) {
  STB_CHECK(ctx && ms_out && count_out && n_classes >= PC_COUNT, STB_ERR_INVALID, "bad argument");
  for (int i = 0; i < n_classes; ++i) { ms_out[i] = 0.f; count_out[i] = 0; }
  for (const auto& sp : ctx->prof.spans) {
    if (sp.e1 < 0) continue;
    STB_CUDA_CHECK(cudaEventSynchronize(ctx->prof.pool[sp.e1]));
    float ms = 0.f;
    STB_CUDA_CHECK(cudaEventElapsedTime(&ms, ctx->prof.pool[sp.e0], ctx->prof.pool[sp.e1]));
    ms_out[sp.cls] += ms;
    count_out[sp.cls] += 1;
  }
  ctx->prof.spans.clear();
  ctx->prof.used = 0;
  return STB_OK;
}

// ---- tiled iteration with the exchanges inside the library (comm.cu): ONE stream-ordered sequence, one CUDA graph
//   begin (iteration stamp, wait for the neighbours' halo) -> halo pull -> forward + band-local statistics ->
//   publish / all-reduce of the statistics over peer memory -> W2 + backward -> gradient stamp -> seam reduce +
//   Adam + clamp + EMA + outbox fill -> halo stamp.
// Mailbox = a cudaMalloc block of THIS library (CUDA IPC needs the allocation base); everything else stays torch-owned.
int stb_comm_create(stb_ctx* ctx, int rank, int world, int max_h_local, int max_W, void* ipc_handle_out64,
                    void** mailbox_out) {
  STB_ENTER(ctx);
  STB_CHECK(world >= 1 && world <= COMM_MAX_RANKS && rank >= 0 && rank < world, STB_ERR_INVALID,
            "rank %d / world %d (at most %d ranks)", rank, world, COMM_MAX_RANKS);
  STB_CHECK(max_h_local >= 16 && max_W >= 16, STB_ERR_INVALID, "bad mailbox capacity %dx%d", max_h_local, max_W);
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  STB_CUDA_CHECK(cudaDeviceSynchronize());
  comm_release(ctx);
  ctx->reset_graphs();
  size_t off[5];
  // stats slots for the largest layer table, so that stb_set_layers never has to re-create a mailbox
  ctx->comm_bytes = comm_mailbox_bytes(stats_floats_max(), max_h_local, max_W, off);
  STB_CUDA_CHECK(cudaMalloc(&ctx->comm_mailbox, ctx->comm_bytes));
  STB_CUDA_CHECK(cudaMemset(ctx->comm_mailbox, 0, ctx->comm_bytes));
  STB_CUDA_CHECK(cudaDeviceSynchronize());
  ctx->comm.rank = rank; ctx->comm.world = world;
  {
    const char* e = getenv("STB_COMM_TIMEOUT_S");
    const double sec = e ? atof(e) : 30.0;
    ctx->comm.timeout_ns = (unsigned long long)((sec > 0.1 ? sec : 0.1) * 1e9);
  }
  ctx->comm.off_stats[0] = off[0]; ctx->comm.off_stats[1] = off[1]; ctx->comm.off_grad = off[2];
  ctx->comm.off_outbox[0] = off[3]; ctx->comm.off_outbox[1] = off[4];
  ctx->comm.mbox[rank] = static_cast<uint8_t*>(ctx->comm_mailbox);
  ctx->comm_max_h = max_h_local; ctx->comm_max_w = max_W;
  if (ipc_handle_out64) {
    cudaIpcMemHandle_t h;
    STB_CUDA_CHECK(cudaIpcGetMemHandle(&h, ctx->comm_mailbox));
    std::memcpy(ipc_handle_out64, &h, sizeof(h));
  }
  if (mailbox_out) *mailbox_out = ctx->comm_mailbox;
  // every kernel of an iteration must be loaded before a peer-wait kernel can be resident (see comm_preload)
  STB_TRY(comm_preload()); STB_TRY(preload_conv_kernels()); STB_TRY(preload_gram_kernels());
  STB_TRY(preload_w2_kernels()); STB_TRY(preload_conv0_kernels()); STB_TRY(preload_image_kernels());
  STB_TRY(preload_resample_kernels());
  cudaFuncAttributes fa;
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(reduce_partials_kernel)));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(content_seed_kernel)));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(adam_scalars_kernel)));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(finalize_loss_kernel)));
  STB_CUDA_CHECK(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(advance_step_kernel)));
  return STB_OK;
}

// handles: world x 64 bytes (cudaIpcMemHandle_t of every rank's mailbox, rank order; own entry ignored)
int stb_comm_connect_ipc(stb_ctx* ctx, const void* handles) {
  STB_ENTER(ctx);
  STB_CHECK(ctx->comm_mailbox && handles, STB_ERR_STATE, "stb_comm_create first");
  for (int r = 0; r < ctx->comm.world; ++r) {
    if (r == ctx->comm.rank) continue;
    cudaIpcMemHandle_t h;
    std::memcpy(&h, static_cast<const uint8_t*>(handles) + 64 * r, sizeof(h));
    void* p = nullptr;
    STB_CUDA_CHECK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    ctx->comm.mbox[r] = static_cast<uint8_t*>(p);
  }
  ctx->comm_ipc = true;
  ctx->comm_ready = true;
  ctx->comm.pdl = 1;   // one process per GPU
  return STB_OK;
}

// same process (several contexts / streams: StyleTransfer(devices=[a, b]), or the single-GPU emulation of the tests):
// plain device pointers
int stb_comm_connect_local(stb_ctx* ctx, void* const* mailboxes) {
  STB_ENTER(ctx);
  STB_CHECK(ctx->comm_mailbox && mailboxes, STB_ERR_STATE, "stb_comm_create first");
  int dev[COMM_MAX_RANKS];
  for (int r = 0; r < ctx->comm.world; ++r) {
    STB_CHECK(mailboxes[r] != nullptr, STB_ERR_INVALID, "null mailbox of rank %d", r);
    dev[r] = ctx->device;
    if (r == ctx->comm.rank) STB_CHECK(mailboxes[r] == ctx->comm_mailbox, STB_ERR_INVALID, "own mailbox mismatch");
    else {
      cudaPointerAttributes pa;
      STB_CUDA_CHECK(cudaPointerGetAttributes(&pa, mailboxes[r]));
      dev[r] = pa.device;
      if (dev[r] != ctx->device) {
        cudaError_t e = cudaDeviceEnablePeerAccess(dev[r], 0);
        if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
        else STB_CUDA_CHECK(e);
      }
    }
    ctx->comm.mbox[r] = static_cast<uint8_t*>(mailboxes[r]);
  }
  // early release is safe only when every rank owns its GPU (see CommDev::pdl): ranks sharing a device keep it off
  int distinct = 1;
  for (int a = 0; a < ctx->comm.world; ++a)
    for (int b = a + 1; b < ctx->comm.world; ++b) distinct = distinct && dev[a] != dev[b];
  ctx->comm_ready = true;
  ctx->comm.pdl = distinct;
  return STB_OK;
}

// ---- per-layer-halo mode: the workspace is a cudaMalloc block of the library that the neighbours map (CUDA IPC) and
// pull single boundary rows from.  stb_comm_alloc_workspace allocates + zeroes + binds it (like stb_bind_workspace);
// stb_comm_connect_ws_* hands in every rank's handle / pointer (rank order; only the neighbours are mapped) and switches
// stb_iterate_banded to "own rows only + one row exchange per layer".  Without it the 80-row aprons are recomputed.
int stb_comm_alloc_workspace(stb_ctx* ctx, size_t bytes, void* ipc_handle_out64, void** ptr_out, void* stream) {
  STB_ENTER(ctx);
  STB_CHECK(bytes >= ctx->w2_bytes + 4096, STB_ERR_WORKSPACE, "workspace smaller than the fixed W2 block");
  STB_CUDA_CHECK(cudaDeviceSynchronize());
  ctx->halo_mode = false;
  shared_ws_release(ctx);
  STB_CUDA_CHECK(cudaMalloc(&ctx->shared_ws, bytes));
  STB_CUDA_CHECK(cudaMemset(ctx->shared_ws, 0, bytes));   // rows a band never computes are read by nobody, but stay finite
  STB_CUDA_CHECK(cudaDeviceSynchronize());
  ctx->shared_ws_bytes = bytes;
  if (ipc_handle_out64) {
    cudaIpcMemHandle_t h;
    STB_CUDA_CHECK(cudaIpcGetMemHandle(&h, ctx->shared_ws));
    std::memcpy(ipc_handle_out64, &h, sizeof(h));
  }
  if (ptr_out) *ptr_out = ctx->shared_ws;
  return stb_bind_workspace(ctx, ctx->shared_ws, bytes, stream);
}

static int connect_ws(stb_ctx* ctx, const void* handles, void* const* pointers) {
  STB_CHECK(ctx->shared_ws && ctx->comm_mailbox, STB_ERR_STATE, "stb_comm_create + stb_comm_alloc_workspace first");
  const int rank = ctx->comm.rank, world = ctx->comm.world;
  for (int r = 0; r < world; ++r) {
    if (r == rank) { ctx->comm.ws[r] = static_cast<uint8_t*>(ctx->shared_ws); continue; }
    if (r != rank - 1 && r != rank + 1) continue;   // only the neighbours' rows are ever read
    void* p = nullptr;
    if (handles) {
      cudaIpcMemHandle_t h;
      std::memcpy(&h, static_cast<const uint8_t*>(handles) + 64 * r, sizeof(h));
      STB_CUDA_CHECK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    } else {
      p = pointers[r];
      STB_CHECK(p != nullptr, STB_ERR_INVALID, "null workspace pointer of rank %d", r);
      cudaPointerAttributes pa;
      STB_CUDA_CHECK(cudaPointerGetAttributes(&pa, p));
      if (pa.device != ctx->device) {
        cudaError_t e = cudaDeviceEnablePeerAccess(pa.device, 0);
        if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
        else STB_CUDA_CHECK(e);
      }
    }
    ctx->comm.ws[r] = static_cast<uint8_t*>(p);
  }
  ctx->shared_ws_ipc = handles != nullptr;
  ctx->reset_graphs();
  return STB_OK;
}
int stb_comm_connect_ws_ipc(stb_ctx* ctx, const void* handles) {
  STB_ENTER(ctx);
  STB_CHECK(handles != nullptr, STB_ERR_INVALID, "null handles");
  return connect_ws(ctx, handles, nullptr);
}
int stb_comm_connect_ws_local(stb_ctx* ctx, void* const* pointers) {
  STB_ENTER(ctx);
  STB_CHECK(pointers != nullptr, STB_ERR_INVALID, "null pointers");
  return connect_ws(ctx, nullptr, pointers);
}
// drop the shared workspace and its mappings (the host barriers before any rank frees memory a neighbour still maps)
int stb_comm_release_workspace(stb_ctx* ctx, int unmap_only) {
  STB_ENTER(ctx);
  STB_CUDA_CHECK(cudaDeviceSynchronize());
  ctx->reset_graphs();
  ctx->halo_mode = false;
  if (unmap_only) {
    if (ctx->shared_ws_ipc)
      for (int r = 0; r < COMM_MAX_RANKS; ++r)
        if (ctx->comm.ws[r] && ctx->comm.ws[r] != ctx->shared_ws) { cudaIpcCloseMemHandle(ctx->comm.ws[r]); ctx->comm.ws[r] = nullptr; }
    return STB_OK;
  }
  shared_ws_release(ctx);
  return STB_OK;
}

// unmap the peers' mailboxes (before any rank frees / re-creates its own; the host barriers in between)
int stb_comm_disconnect(stb_ctx* ctx) {
  STB_ENTER(ctx);
  STB_CUDA_CHECK(cudaDeviceSynchronize());
  ctx->reset_graphs();
  if (ctx->comm_ipc)
    for (int r = 0; r < ctx->comm.world; ++r)
      if (r != ctx->comm.rank && ctx->comm.mbox[r]) {
        STB_CUDA_CHECK(cudaIpcCloseMemHandle(ctx->comm.mbox[r]));
        ctx->comm.mbox[r] = nullptr;
      }
  ctx->comm_ipc = false;
  ctx->comm_ready = false;
  return STB_OK;
}

// geometry of this band and of its neighbours for the current scale (rows in LOCAL coordinates of each rank)
int stb_comm_set_geometry(stb_ctx* ctx, int W, int h_local, int own0, int own_rows, int up_h_local,
                          int up_apron_row0, int dn_h_local, int halo_rows) {
  STB_ENTER(ctx);
  STB_CHECK(ctx->comm_mailbox, STB_ERR_STATE, "stb_comm_create first");
  STB_CHECK(h_local <= ctx->comm_max_h && W <= ctx->comm_max_w && up_h_local <= ctx->comm_max_h &&
                dn_h_local <= ctx->comm_max_h, STB_ERR_WORKSPACE, "band %dx%d exceeds the mailbox capacity %dx%d",
            h_local, W, ctx->comm_max_h, ctx->comm_max_w);
  const bool has_up = ctx->comm.rank > 0, has_dn = ctx->comm.rank + 1 < ctx->comm.world;
  STB_CHECK(own_rows >= COMM_APRON && own0 == (has_up ? COMM_APRON : 0) &&
                h_local == own0 + own_rows + (has_dn ? COMM_APRON : 0), STB_ERR_INVALID,
            "band geometry: h_local=%d own0=%d own_rows=%d (aprons are %d rows)", h_local, own0, own_rows, COMM_APRON);
  if (has_up) STB_CHECK(up_apron_row0 + COMM_APRON == up_h_local, STB_ERR_INVALID, "upper neighbour geometry");
  // the row kernels of the exchange walk a band with 32-bit indices
  STB_CHECK(3l * h_local * W < (1l << 31), STB_ERR_INVALID, "band of %d x %d pixels is too large", h_local, W);
  ctx->comm.W = W; ctx->comm.h_local = h_local; ctx->comm.own0 = own0; ctx->comm.own_rows = own_rows;
  ctx->comm.up_h_local = up_h_local; ctx->comm.up_apron_row0 = up_apron_row0; ctx->comm.dn_h_local = dn_h_local;
  // halo_rows = 1: own rows only + one boundary-row pull per layer (needs the peer-mapped workspace); 0: recomputed aprons
  STB_CHECK(!halo_rows || ctx->comm.ws[ctx->comm.rank] != nullptr, STB_ERR_STATE,
            "halo-row mode needs stb_comm_alloc_workspace + stb_comm_connect_ws_*");
  ctx->halo_mode = halo_rows != 0;
  ctx->comm_geometry = true;
  // the banded graphs bake in the halo mode and the neighbours' heights
  ctx->gslot[GS_ITERATE_BANDED].reset();
  ctx->gslot[GS_ITERATE_LBFGS_BANDED].reset();
  return STB_OK;
}

// zero the iteration stamps of the own mailbox.  The host must barrier over all ranks BEFORE (nobody still reads the
// old stamps) and AFTER (nobody polls a mailbox that is not reset yet).
int stb_comm_reset(stb_ctx* ctx, void* stream) {
  STB_ENTER(ctx);
  STB_CHECK(ctx->comm_mailbox, STB_ERR_STATE, "stb_comm_create first");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  STB_CUDA_CHECK(cudaMemsetAsync(ctx->comm_mailbox, 0, 4096, s));
  STB_CUDA_CHECK(cudaStreamSynchronize(s));
  return STB_OK;
}

int stb_iterate_banded(stb_ctx* ctx, float* img, float* exp_avg, float* exp_avg_sq, float* ema, int64_t step, float lr,
                       float beta1, float beta2, float adam_eps, float ema_decay, float* loss_out_host8,
                       void* stream) {
  STB_CHECK(ctx && img && exp_avg && exp_avg_sq && ema && step >= 1, STB_ERR_INVALID, "bad argument");
  const IterArgs a{img, exp_avg, exp_avg_sq, ema, step, lr, beta1, beta2, adam_eps, ema_decay, nullptr, loss_out_host8};
  return iterate(ctx, kBanded, a, true, stream);
}

// optimizer='lbfgs' on a band: the sequence of stb_iterate_banded up to the gradient stamp, then the banded L-BFGS step
// of lbfgs.cu (seam gather, cross-rank reductions, own-row update + outbox fill) and the halo stamp.  The state holds
// this band's own rows only: stb_lbfgs_state_bytes(own_rows, W).
int stb_iterate_lbfgs_banded(stb_ctx* ctx, float* img, float* ema, void* state, size_t state_bytes, int64_t step,
                             float ema_decay, float* loss_out_host8, void* stream) {
  STB_CHECK(ctx && img && ema && state, STB_ERR_INVALID, "null argument");
  IterArgs a{img, nullptr, nullptr, ema, step};
  a.ema_decay = ema_decay; a.loss_out_host8 = loss_out_host8; a.state = state; a.state_bytes = state_bytes;
  return iterate(ctx, kLbfgsBanded, a, true, stream);
}

// Sync-free loss read-back (SURVEY.md 8f row 2).  host_ring: PINNED host memory of slots x 16 floats (NULL: off).
// Every updating iteration then stores {loss, content, style1..5, tv} into slot (step % slots) and finally the step as
// the slot's int32 stamp (word 8) -- written by the loss kernel itself right after the W2 forward, i.e. before the
// backward pass: the host polls the stamp, no stream synchronisation.
int stb_set_loss_ring(stb_ctx* ctx, float* host_ring, int slots) {
  STB_ENTER(ctx);
  ctx->reset_graphs();
  ctx->ring_dev = nullptr; ctx->ring_slots = 0;
  if (host_ring == nullptr) return STB_OK;
  STB_CHECK(slots >= 2, STB_ERR_INVALID, "loss ring needs at least 2 slots");
  void* dptr = nullptr;
  STB_CUDA_CHECK(cudaHostGetDevicePointer(&dptr, host_ring, 0));
  ctx->ring_dev = static_cast<float*>(dptr);
  ctx->ring_slots = slots;
  return STB_OK;
}

// 1: iterations replay as CUDA graphs; 0: eager launches (why: stb_last_error-style text in note_out, optional)
int stb_graph_status(stb_ctx* ctx, char* note_out, size_t note_bytes) {
  STB_CHECK(ctx != nullptr, STB_ERR_INVALID, "null ctx");
  if (note_out && note_bytes > 0) {
    std::strncpy(note_out, ctx->graph_note.c_str(), note_bytes - 1);
    note_out[note_bytes - 1] = 0;
  }
  bool any = false;
  for (const auto& g : ctx->gslot) any = any || g.exec != nullptr;
  return ctx->graphs_enabled ? (any ? 1 : 2) : 0;  // 2: enabled, nothing captured yet
}

// Kernel launches issued through graph replays so far (counted from the captured graphs, not assumed): replays of every
// graph, kernels those replays launched, and the kernel nodes of the graphs of stb_iterate, stb_iterate_fwd,
// stb_iterate_bwd and stb_iterate_banded (0 where nothing is captured; the L-BFGS graphs have no entry).
int stb_launch_count(stb_ctx* ctx, int64_t* graph_replays, int64_t* kernels_replayed, int* kernels_per_graph4) {
  STB_CHECK(ctx != nullptr, STB_ERR_INVALID, "null ctx");
  if (graph_replays) *graph_replays = ctx->graph_replays;
  if (kernels_replayed) *kernels_replayed = ctx->kernels_replayed;
  if (kernels_per_graph4)
    for (int i = GS_ITERATE; i <= GS_ITERATE_BANDED; ++i) kernels_per_graph4[i] = ctx->gslot[i].kernel_nodes;
  return STB_OK;
}

// diagnostics (STB_W2_TRACE=1): the %globaltimer stamps CTA 0 of the W2 chain kernel wrote for the rounds of the last
// iteration (8 words per round, see w2_chain_kernel); rounds_out receives the number of rounds.
int stb_debug_w2_trace(stb_ctx* ctx, unsigned long long* host_out, size_t words, int* rounds_out) {
  STB_ENTER(ctx);
  STB_CHECK(ctx->w2_ready && host_out && words >= (size_t)W2_TRACE_WORDS, STB_ERR_INVALID, "need %d words", W2_TRACE_WORDS);
  STB_CUDA_CHECK(cudaDeviceSynchronize());
  STB_CUDA_CHECK(cudaMemcpy(host_out, ctx->w2.d_trace, W2_TRACE_WORDS * 8, cudaMemcpyDeviceToHost));
  if (rounds_out) *rounds_out = (int)ctx->w2.rounds.size();
  return STB_OK;
}

// test hook: copy an internal activation (post-ReLU output of conv `conv_index`, bf16 NHWC) of the last forward
int stb_debug_activation(stb_ctx* ctx, int H, int W, int conv_index, void* out_bf16, size_t out_bytes, void* stream) {
  STB_CHECK(ctx && out_bf16 && conv_index >= 0 && conv_index <= ctx->layers.last_conv(), STB_ERR_INVALID,
            "bad argument (conv %d: the forward runs through conv %d)", conv_index, ctx ? ctx->layers.last_conv() : 0);
  Plan pl;
  make_plan(ctx, H, W, &pl);
  STB_TRY(ensure_ws(ctx, pl));
  const size_t bytes = (size_t)pl.h[conv_index] * pl.w[conv_index] * kCout[conv_index] * 2;
  STB_CHECK(out_bytes >= bytes, STB_ERR_INVALID, "output buffer too small (%zu < %zu)", out_bytes, bytes);
  STB_CUDA_CHECK(cudaMemcpyAsync(out_bf16, at<bf16>(ctx, pl.act_off[conv_index]), bytes, cudaMemcpyDeviceToDevice,
                                 static_cast<cudaStream_t>(stream)));
  return STB_OK;
}

}  // extern "C"
