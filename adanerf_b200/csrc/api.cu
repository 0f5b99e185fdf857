// C ABI + host-side context of the H100 AdaNeRF renderer (see include/adanerf_b200.h).
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <optional>
#include <string>
#include <vector>

#include "../../include/adanerf_b200.h"
#include "../../include/adanerf_b200_views.h"
#include "export_loader.h"
#include "flip.cuh"
#include "iwssim.cuh"
#include "mlp.cuh"
#include "ptx.cuh"
#include "stages.cuh"

using namespace adn;

namespace {

struct HostTensor {
  std::vector<float> data;
  int64_t rows = 0, cols = 0;
};

// Memory the context owns: grown by ensure(), freed with the context.  Device memory, or page-locked host memory.
struct Buf {
  enum Kind { kDevice, kPinned };
  void* p = nullptr;
  size_t cap = 0;
  Kind kind;
  explicit Buf(Kind k = kDevice) : kind(k) {}
  Buf(const Buf&) = delete;
  Buf& operator=(const Buf&) = delete;
  ~Buf() { release(); }
  cudaError_t release() {
    const cudaError_t e = !p ? cudaSuccess : kind == kPinned ? cudaFreeHost(p) : cudaFree(p);
    p = nullptr;
    cap = 0;
    return e;
  }
  template <class T> T* as() const { return static_cast<T*>(p); }
};

struct Net {
  bool ready = false;
  int n_in = 0, n_out = 0;
  int depth = 0, width = 0, skip = -1;   // the shape build_net0 / build_net1 inferred from the tensors (adn_net_shape)
  MlpProgram prog{};
  Buf wblob;
  std::map<std::string, HostTensor> tensors;  // kept so "mlp0_terms" can re-pack
};

}  // namespace

struct adn_ctx {
  int device = 0;
  int num_sms = 132;
  adn_scene scene{};
  SceneDev sc{};
  Buf zlut;                       // [128] world depth of the cell centres (log warp)
  Buf zlut_cells;                 // the same tables for D = 32, 64 and 256 depth cells, one after another (cell_table)
  Buf zlut_dense;                 // [dense_K]
  int dense_K = 0;
  Buf zlin;                       // linear_depths(K) of every K = 1..128, the table of K at K (K - 1) / 2 (sampler 2)
  Net net[2];
  int mlp0_terms = 3;
  int n_feat0 = 90;               // sampling-net input features: 6 + 6 (n_freq_pos0 + n_freq_dir0)
  bool fuse_encoder = true;       // stage 3 inside the shading kernel (non-NDC scenes): no [M, n_in]-sized tile buffer
  int64_t chunk_rays = 0;
  bool profile = false;
  int64_t sample_budget = 0;      // B of adn_set_option "sample_budget" (0 = off)
  bool last_budget = false;       // the last render chose its threshold on the device (in budget_thr)
  float last_thr = 0.0f;          // the last render's threshold argument
  bool prof_budget = false;       // the profiled render timed the selection with stage 2 (ev[7] -> ev[3])
  bool sampling_view = false;     // adn_set_option "sampling_view": renders draw the sampling net's view (stages 0-1 + view)
  bool last_view = false;         // the last render drew the view (it counts no samples)
  bool prof_view = false;         // the profiled render drew the view (slots 2-4 unused, the view kernel in slot 5)
  int sampler = 0;                // adn_set_option "sampler": 0 = FromClassifiedDepthAdaptive, 1 = FromClassifiedDepth (fixed K),
                                  // 2 = LinearlySpacedZNearZFar (no sampling net)
  bool prof_linear = false;       // the profiled render ran sampler 2 (rays in slot 0, slot 1 unused)
  int pdf_transform = kPdfSigmoid;   // adn_set_option "pdf_transform": what FromClassifiedDepth applies to raw0 first
  // scratch
  Buf raw0_pad;                   // D < 128: the sampling MLP's rows at its 128-column stride, before the copy to raw0 [N, D]
  Buf tiles0, raw0, ray_o, ray_d, ray_dirs, count, offset, rayidx, zbuf, zpbuf, tiles1, raw1, s2scratch, rgba, metric, flip, iwssim;
  Buf dirs, rgb, nsamples;        // device side of the *_host entry points
  Buf budget_keys, budget_work, budget_thr;   // sample budget: candidate keys, histograms + select state, t*
  BudgetGroup group;              // adn_set_budget_group: the reducer that sums the selection's histograms across members
  Buf total;                      // long long: samples of the last stage 2
  Buf watchdog{Buf::kPinned};     // int flag in mapped pinned host memory: still readable after a device trap
  int* d_err = nullptr;           // device view of watchdog
  Stage2Sync s2sync;              // epoch / ticket base of s2scratch (no per-launch memset)
  // pinned staging for the *_host entry points
  Buf h_in{Buf::kPinned}, h_out{Buf::kPinned}, h_ns{Buf::kPinned};
  // caller buffers page-locked in place at the caller's explicit request (adn_register_host_buffer): the *_host entry
  // points DMA straight from / to them; everything else goes through the context's pinned staging buffers
  struct Reg { const void* p = nullptr; size_t bytes = 0; };
  std::vector<Reg> regs;
  cudaStream_t own_stream = nullptr;
  // issue order across streams (CallOrder): recorded after the last enqueue of every call, waited on before the first
  // enqueue of the next one
  cudaEvent_t order = nullptr;
  cudaEvent_t ev[8] = {};
  adn_stats stats{};
  std::string last_error;
};

namespace {

const char* kStatusText[] = {"ok", "invalid argument", "CUDA error", "no usable sm_90 device", "weights not set",
                             "I/O error", "device watchdog tripped"};

adn_status fail(adn_ctx* ctx, adn_status s, const std::string& msg) {
  if (ctx) ctx->last_error = msg;
  return s;
}
adn_status cuda_fail(adn_ctx* ctx, cudaError_t e, const char* where) {
  return fail(ctx, ADN_ERR_CUDA, std::string(where) + ": " + cudaGetErrorString(e));
}
// A budgeted call on a context in a budget group takes part in the group's reductions even when it has no rays.
bool joins_group(const adn_ctx* ctx) { return ctx && ctx->sample_budget > 0 && ctx->group.fn; }
// The status of a selection whose group reduction failed (launch_budget_threshold stopped enqueueing).
adn_status group_fail(adn_ctx* ctx, const char* who) {
  return fail(ctx, ADN_ERR_CUDA, std::string(who) + ": the budget group's reducer returned " + std::to_string(ctx->group.status) +
                                     " in select round " + std::to_string(ctx->group.failed_round));
}
#define ADN_CUDA(ctx, call)                                   \
  do {                                                        \
    cudaError_t e__ = (call);                                 \
    if (e__ != cudaSuccess) return cuda_fail(ctx, e__, #call); \
  } while (0)

// Makes the calls on one context execute in the order they were made, whatever stream each names.  They share the
// context's scratch (tiles, raw0 / raw1, the stage-2 look-back state and tickets, the budget state) and often each other's
// outputs, so two calls in flight on different streams would overwrite what the other still reads.  begin(): the call's
// stream waits on ctx->order, recorded by the previous call after its last enqueue; the guard records it again when the call
// returns, on an error return after a partial enqueue too.  The wait is made even when the stream is the previous call's: it
// costs one driver call, and a stream handle can be destroyed and handed out again.  One guard per entry point, after
// cudaSetDevice (a null stream is the legacy stream of the current device).
//
// A stream that is capturing a CUDA graph is refused before anything is enqueued: stage 2 takes its launch epoch and ticket
// base from host state (Stage2Sync), so a replayed launch would run with stale ones.
class CallOrder {
 public:
  CallOrder(adn_ctx* ctx, cudaStream_t st) : ctx_(ctx), st_(st) {}
  CallOrder(const CallOrder&) = delete;
  CallOrder& operator=(const CallOrder&) = delete;
  ~CallOrder() {
    if (armed_) cudaEventRecord(ctx_->order, st_);
  }
  adn_status begin(const char* who) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    const cudaError_t e = cudaStreamIsCapturing(st_, &cs);
    if (e != cudaSuccess) cudaGetLastError();   // e.g. the legacy stream while another stream captures: treat as capturing
    if (e != cudaSuccess || cs != cudaStreamCaptureStatusNone)
      return fail(ctx_, ADN_ERR_INVALID, std::string(who) + ": the stream is capturing a CUDA graph; calls cannot be captured "
                                                            "(stage 2's launch epoch and tickets are host state)");
    ADN_CUDA(ctx_, cudaStreamWaitEvent(st_, ctx_->order, 0));
    armed_ = true;
    return ADN_OK;
  }

 private:
  adn_ctx* ctx_;
  cudaStream_t st_;
  bool armed_ = false;
};

// Grows b to at least `bytes` (device buffers with some slack); the old contents are not kept.
adn_status ensure(adn_ctx* ctx, Buf& b, size_t bytes) {
  if (bytes <= b.cap) return ADN_OK;
  ADN_CUDA(ctx, b.release());
  const bool pinned = b.kind == Buf::kPinned;
  const size_t want = pinned ? bytes : bytes + bytes / 8 + 256;
  ADN_CUDA(ctx, pinned ? cudaMallocHost(&b.p, want) : cudaMalloc(&b.p, want));
  b.cap = want;
  return ADN_OK;
}

// True when [p, p + bytes) can be the source / target of an asynchronous copy at full speed: inside a range the caller
// registered with adn_register_host_buffer (whose lifetime the caller vouches for), or memory the caller allocated
// page-locked itself (cudaMallocHost / torch pin_memory).  The library never registers memory behind the caller's back:
// a buffer that is freed and re-allocated at the same address would keep a stale registration (ADVICE r1).
bool pin_in_place(adn_ctx* ctx, const void* p, size_t bytes) {
  const char* lo = static_cast<const char*>(p);
  for (const adn_ctx::Reg& r : ctx->regs)
    if (lo >= static_cast<const char*>(r.p) && lo + bytes <= static_cast<const char*>(r.p) + r.bytes) return true;
  cudaPointerAttributes attr{};
  if (cudaPointerGetAttributes(&attr, p) == cudaSuccess && attr.type == cudaMemoryTypeHost) return true;
  cudaGetLastError();
  return false;
}

// ---- bf16 helpers (host) -------------------------------------------------------------------
inline uint16_t f2bf(float f) {  // round to nearest even
  uint32_t u;
  std::memcpy(&u, &f, 4);
  if ((u & 0x7FFFFFFFu) > 0x7F800000u) return uint16_t((u >> 16) | 0x40);
  u += 0x7FFFu + ((u >> 16) & 1u);
  return uint16_t(u >> 16);
}
inline float bf2f(uint16_t h) {
  uint32_t u = uint32_t(h) << 16;
  float f;
  std::memcpy(&f, &u, 4);
  return f;
}

struct Seg {
  int col0, valid;
};

// Packs one layer's weights W [n_out, k_in] into the ring-stage stream, in the order the MLP kernel consumes it: for each
// 128-row N half, for each K block (Seg):
//   nsplit == 1: a [128 x 64] K-major SWIZZLE_128B bf16 tile;
//   nsplit == 2: for each pair of K steps that holds one (L.k_cnt), a [128 x 32] K-major SWIZZLE_64B tile of the hi
//   terms followed by the same tile of the lo terms (16 KB a stage).  A K block with no K step gets no stage, e.g. the
//   sampling net's second input block at 30 inputs; at 90 inputs it gets one.
// layer_stages(L, nsplit) stages in all.
void pack_layer(const float* W, int n_out, int k_in, const std::vector<Seg>& segs, int nsplit, const MlpLayer& L,
                std::vector<uint8_t>& blob) {
  const int n_half = (n_out + 127) / 128;
  const int cols = nsplit == 2 ? 16 * stage_k_steps(nsplit) : 64;   // K columns of one stage
  const uint32_t half = kBlkBytes / 2;                                // one [128 x 32] tile (nsplit == 2)
  for (int nh = 0; nh < n_half; ++nh) {
    for (size_t b = 0; b < segs.size(); ++b) {
      const Seg& sg = segs[b];
      const int n_st = nsplit == 2 ? (L.k_cnt[b] + stage_k_steps(nsplit) - 1) / stage_k_steps(nsplit) : 1;
      for (int s = 0; s < n_st; ++s) {
        const size_t base = blob.size();
        blob.resize(base + size_t(nsplit) * (nsplit == 2 ? half : kBlkBytes), 0);
        for (int n = 0; n < 128; ++n) {
          const int row = nh * 128 + n;
          for (int kk = 0; kk < cols; ++kk) {
            const int c = s * cols + kk;   // column inside the K block
            float w = 0.0f;
            if (row < n_out && c < sg.valid && sg.col0 + c < k_in) w = W[size_t(row) * k_in + sg.col0 + c];
            const uint16_t hi = f2bf(w);
            if (nsplit == 2) {
              const uint32_t off = sw64_offset(uint32_t(n), uint32_t(kk));
              const uint16_t lo = f2bf(w - bf2f(hi));
              std::memcpy(&blob[base + off], &hi, 2);
              std::memcpy(&blob[base + half + off], &lo, 2);
            } else {
              std::memcpy(&blob[base + sw128_offset(uint32_t(n), uint32_t(kk))], &hi, 2);
            }
          }
        }
      }
    }
  }
}

size_t push_floats(std::vector<float>& f, const float* src, size_t n) {
  while (f.size() % 4) f.push_back(0.0f);
  const size_t off = f.size();
  f.insert(f.end(), src, src + n);
  while (f.size() % 4) f.push_back(0.0f);
  return off;
}

const HostTensor* find(const Net& n, const std::string& name) {
  auto it = n.tensors.find(name);
  return it == n.tensors.end() ? nullptr : &it->second;
}

adn_status upload(adn_ctx* ctx, Net& net, const std::vector<uint8_t>& wblob, const std::vector<float>& fblob) {
  if (fblob.size() > size_t(kSideFloats))
    return fail(ctx, ADN_ERR_INVALID, "network has " + std::to_string(fblob.size()) + " fp32 side parameters (biases and heads), more than " +
                                          std::to_string(kSideFloats) + " fit in shared memory");
  std::memset(net.prog.side, 0, sizeof(net.prog.side));
  std::memcpy(net.prog.side, fblob.data(), fblob.size() * 4);
  adn_status s = ensure(ctx, net.wblob, wblob.size());   // the callers synchronised: no kernel still reads the old blob
  if (s != ADN_OK) return s;
  ADN_CUDA(ctx, cudaMemcpy(net.wblob.p, wblob.data(), wblob.size(), cudaMemcpyHostToDevice));
  return ADN_OK;
}

// The layer programs of the two networks are derived here, from the tensor shapes, and nowhere else in the library.
//
// Sampling net: BaseNet without skips (src/models.py:71-76,183-195): layers.{i}.weight/bias, D = 1-12 layers, n_in <= 128
// inputs, every hidden layer W = 128 or 256 wide, 32, 64, 128 or 256 outputs (the depth cells, multiDepthFeatures); 32 and
// 64 outputs are padded to one 128-row N half with zero weights and biases, so the kernel writes rows of 128 columns.
// Layer 0 reads the two input blocks, every other layer the W/64 hidden blocks (split precision: in shared memory,
// overwritten in place by its epilogue; plain bf16: in registers).
adn_status build_net0(adn_ctx* ctx) {
  Net& net = ctx->net[0];
  auto bad = [&](const std::string& msg) { return fail(ctx, ADN_ERR_INVALID, "sampling net: " + msg); };
  int D = 0;
  while (find(net, "layers." + std::to_string(D) + ".weight")) ++D;
  if (D < 1 || D > kMaxLayers) return bad("need layers.0.weight .. (1-12 layers)");
  const int nsplit = ctx->mlp0_terms == 3 ? 2 : 1;
  const int width = int(find(net, "layers.0.weight")->rows);   // the hidden width W (the output width of a 1-layer net)
  MlpProgram P{};
  P.n_layers = D;
  std::vector<uint8_t> wblob;
  std::vector<float> fblob;
  int prev = -1;
  for (int l = 0; l < D; ++l) {
    const std::string name = "layers." + std::to_string(l);
    const HostTensor* W = find(net, name + ".weight");
    const HostTensor* B = find(net, name + ".bias");
    if (!B || int64_t(B->data.size()) != W->rows) return bad(name + ".bias is missing or not [" + std::to_string(W->rows) + "]");
    const int n_out = int(W->rows), k_in = int(W->cols);
    const bool last = (l == D - 1);
    if (l == 0) {
      if (k_in < 1 || k_in > 128) return bad(name + ".weight has " + std::to_string(k_in) + " input columns; the input width must be 1-128");
      net.n_in = k_in;
    } else if (k_in != prev) {
      return bad(name + ".weight has " + std::to_string(k_in) + " input columns but layers." + std::to_string(l - 1) + " has " +
                 std::to_string(prev) + " outputs: layer widths must chain (BaseNet skips are not supported)");
    }
    if (!last && n_out != width)
      return bad(name + ".weight has " + std::to_string(n_out) + " outputs; every hidden layer must be as wide as layers.0 (" +
                 std::to_string(width) + ")");
    if (!last && n_out != 128 && n_out != 256)
      return bad(name + ".weight has " + std::to_string(n_out) + " outputs; the hidden width must be 128 or 256");
    if (last && n_out != 32 && n_out != 64 && n_out != 128 && n_out != 256)
      return bad(name + ".weight has " + std::to_string(n_out) + " outputs; the output width (the depth cells D, "
                 "multiDepthFeatures) must be 32, 64, 128 or 256");
    prev = n_out;
    MlpLayer& L = P.layers[l];
    std::vector<Seg> segs;
    if (l == 0) {
      segs = {{0, std::min(64, k_in)}, {64, std::max(0, k_in - 64)}};
    } else {
      for (int c = 0; c < k_in; c += 64) segs.push_back({c, 64});
    }
    L.n_kb = uint8_t(segs.size());
    (l == 0 ? L.in_first : L.n_hid) = L.n_kb;
    for (size_t i = 0; i < segs.size(); ++i) {
      // 16-wide K steps that hold data; block 0 keeps at least one (it initialises the accumulator)
      L.k_cnt[i] = uint8_t(std::max(i == 0 ? 1 : 0, (segs[i].valid + 15) / 16));
    }
    L.n_half = uint8_t((n_out + 127) / 128);
    L.flags = last ? uint8_t(LF_FINAL_RAW) : uint8_t(LF_RELU | LF_OUT_ACT);
    L.w_off = uint32_t(wblob.size());
    pack_layer(W->data.data(), n_out, k_in, segs, nsplit, L, wblob);
    std::vector<float> bias(size_t(L.n_half) * 128, 0.0f);   // zero rows past D = 32 / 64 outputs
    std::copy(B->data.begin(), B->data.end(), bias.begin());
    L.bias_off = uint32_t(push_floats(fblob, bias.data(), bias.size()));
    if (last) {
      net.n_out = n_out;
      P.out_cols = int(L.n_half) * 128;   // D < 128: rows padded to one 128-row half (zero weights and biases)
    }
  }
  P.in = sampling_tiles(net.n_in, nsplit);
  P.in_nblk0 = P.in.n_blk;
  net.prog = P;
  adn_status s = upload(ctx, net, wblob, fblob);
  if (s != ADN_OK) return s;
  net.depth = D;
  net.width = width;
  net.skip = -1;
  net.ready = true;
  return ADN_OK;
}

// Shading net: NeRF(D, W, skips, use_viewdirs=True) (src/models.py:199-277) with the scene's encoding: kP = 3 + 6 P position
// and kV = 3 + 6 D direction features (input_ch / input_ch_views, models.py:216-224; 63 + 27 for posEnc 10-4).  D = 1-10
// pts_linears (D + feature + view layer <= kMaxLayers), W = 128 or 256, the view branch W/2.  A skip after pts layer i
// shows as pts_linears.{i+1} reading W + kP columns, cat[pts, h] (models.py:226-228, 260-261); at most one.  The program,
// the input blocks P (one, or two when kP > 64; then V) in shared memory and the W/64 hidden blocks in the consumers'
// registers:
//   pts layer 0 reads P; the skip consumer reads P, then the hidden blocks; the other pts layers read the hidden blocks; the
//   last pts layer also forms alpha (LF_ALPHA_DOT); feature_linear: W -> W without activation; views_linears.0 on
//   cat[feature, V] -> W/2 reads the hidden blocks, then V, with rgb_linear in its epilogue.
// At W = 128 the view layer's 64 outputs are padded to the kernel's 128 rows with zero weights, zero biases and zero
// rgb_linear columns: ReLU(0) = 0 adds nothing to the rgb dot products, so the result is exact.
adn_status build_net1(adn_ctx* ctx) {
  Net& net = ctx->net[1];
  const int kP = 3 + 6 * ctx->sc.n_freq_pos, kV = 3 + 6 * ctx->sc.n_freq_dir;
  const std::string enc = "posEnc " + (ctx->scene.n_freq_pos < 0 && ctx->scene.n_freq_dir < 0
                                           ? std::string("none")
                                           : std::to_string(ctx->sc.n_freq_pos) + "-" + std::to_string(ctx->sc.n_freq_dir));
  auto bad = [&](const std::string& msg) { return fail(ctx, ADN_ERR_INVALID, "shading net: " + msg); };
  auto shape = [](int64_t r, int64_t c) { return "[" + std::to_string(r) + ", " + std::to_string(c) + "]"; };
  const HostTensor* w0 = find(net, "pts_linears.0.weight");
  if (!w0 || w0->cols != kP)
    return bad("pts_linears.0.weight must be [W, " + std::to_string(kP) + "] (" + enc + ")" +
               (w0 ? ", not " + shape(w0->rows, w0->cols) : std::string(", missing")));
  const int W = int(w0->rows);
  if (W != 128 && W != 256) return bad("pts_linears.0.weight has " + std::to_string(W) + " rows; the width W must be 128 or 256");
  int D = 0;
  while (find(net, "pts_linears." + std::to_string(D) + ".weight")) ++D;
  if (D > kMaxLayers - 2) return bad("pts_linears.0 .. " + std::to_string(D - 1) + ": " + std::to_string(D) + " layers, at most 10 are supported");
  const HostTensor *pw[kMaxLayers], *pb[kMaxLayers];
  int skip = -1;
  for (int i = 0; i < D; ++i) {
    const std::string name = "pts_linears." + std::to_string(i);
    pw[i] = find(net, name + ".weight");
    pb[i] = find(net, name + ".bias");
    if (pw[i]->rows != W) return bad(name + ".weight has " + std::to_string(pw[i]->rows) + " rows; every pts layer must be W = " + std::to_string(W) + " wide");
    if (i > 0 && pw[i]->cols == W + kP) {
      if (skip >= 0)
        return bad(name + ".weight reads cat[pts, h] after the skip at layer " + std::to_string(skip) + "; at most one skip is supported");
      skip = i - 1;
    } else if (i > 0 && pw[i]->cols != W) {
      return bad(name + ".weight has " + std::to_string(pw[i]->cols) + " input columns; expect W = " + std::to_string(W) +
                 " or W + " + std::to_string(kP) + " = " + std::to_string(W + kP) + " (a skip, " + enc + ")");
    }
    if (!pb[i] || int64_t(pb[i]->data.size()) != W) return bad(name + ".bias is missing or not [" + std::to_string(W) + "]");
  }
  struct Want {
    const char* name;
    int64_t rows, cols;
  };
  const Want want[4] = {{"feature_linear", W, W}, {"alpha_linear", 1, W}, {"views_linears.0", W / 2, W + kV}, {"rgb_linear", 3, W / 2}};
  const HostTensor *hw[4], *hb[4];
  for (int j = 0; j < 4; ++j) {
    const std::string name(want[j].name);
    hw[j] = find(net, name + ".weight");
    hb[j] = find(net, name + ".bias");
    if (!hw[j] || hw[j]->rows != want[j].rows || hw[j]->cols != want[j].cols)
      return bad(name + ".weight must be " + shape(want[j].rows, want[j].cols) + " for W = " + std::to_string(W) + " (" + enc + ")" +
                 (hw[j] ? ", not " + shape(hw[j]->rows, hw[j]->cols) : std::string(", missing")));
    if (!hb[j] || int64_t(hb[j]->data.size()) != want[j].rows) return bad(name + ".bias is missing or not [" + std::to_string(want[j].rows) + "]");
  }
  const HostTensor *fw = hw[0], *fb = hb[0], *aw = hw[1], *ab = hb[1], *vw = hw[2], *vb = hb[2], *rw = hw[3], *rb = hb[3];
  net.n_in = kP + kV;
  net.n_out = 4;
  const int nh = W / 64;                       // hidden activation blocks 1 .. nh
  MlpProgram P{};
  P.n_layers = D + 2;
  std::vector<uint8_t> wblob;
  std::vector<float> fblob;
  for (int l = 0; l < D + 2; ++l) {
    MlpLayer& L = P.layers[l];
    std::vector<Seg> segs;
    auto read_p = [&] {
      for (int c = 0; c < kP; c += 64) segs.push_back({c, std::min(64, kP - c)});
      L.in_first = uint8_t(shading_p_blocks(kP));
    };
    auto read_hidden = [&](int col0) {
      for (int b = 0; b < nh; ++b) segs.push_back({col0 + 64 * b, 64});
      L.n_hid = uint8_t(nh);
    };
    const HostTensor *Wt, *B;
    L.n_half = uint8_t(W / 128);
    if (l < D) {
      if (l == 0) {
        read_p();
      } else if (l == skip + 1) {   // cat[pts, h]
        read_p();
        read_hidden(kP);
      } else {
        read_hidden(0);
      }
      L.flags = LF_RELU | LF_OUT_ACT | (l == D - 1 ? LF_ALPHA_DOT : 0);
      Wt = pw[l];
      B = pb[l];
    } else if (l == D) {  // feature_linear: no activation (models.py:265)
      read_hidden(0);
      L.flags = LF_OUT_ACT;
      Wt = fw;
      B = fb;
    } else {  // views_linears.0 on cat[feature, views] (models.py:266-269) + rgb_linear in the epilogue
      read_hidden(0);
      segs.push_back({W, kV});
      L.in_last = 1;
      L.flags = LF_RELU | LF_FINAL_RGB;
      L.n_half = 1;
      Wt = vw;
      B = vb;
    }
    L.n_kb = uint8_t(segs.size());
    for (size_t i = 0; i < segs.size(); ++i) L.k_cnt[i] = uint8_t((segs[i].valid + 15) / 16);
    L.w_off = uint32_t(wblob.size());
    pack_layer(Wt->data.data(), int(Wt->rows), int(Wt->cols), segs, 1, L, wblob);
    std::vector<float> bias(size_t(L.n_half) * 128, 0.0f);   // zero rows past the view layer's W/2 outputs
    std::copy(B->data.begin(), B->data.end(), bias.begin());
    L.bias_off = uint32_t(push_floats(fblob, bias.data(), bias.size()));
  }
  std::vector<float> rgb_w(3 * 128, 0.0f);   // rgb_linear at the kernel's row stride of 128
  for (int k = 0; k < 3; ++k) std::copy_n(rw->data.data() + size_t(k) * (W / 2), W / 2, rgb_w.data() + k * 128);
  P.alpha_w_off = uint32_t(push_floats(fblob, aw->data.data(), size_t(W)));
  P.alpha_b_off = uint32_t(push_floats(fblob, ab->data.data(), 1));
  P.rgb_w_off = uint32_t(push_floats(fblob, rgb_w.data(), rgb_w.size()));
  P.rgb_b_off = uint32_t(push_floats(fblob, rb->data.data(), 3));
  P.in = shading_tiles(kP, kV);
  P.in_nblk0 = shading_p_blocks(kP);   // P; V is the block after it
  P.out_cols = 4;
  net.prog = P;
  adn_status s = upload(ctx, net, wblob, fblob);
  if (s != ADN_OK) return s;
  net.depth = D;
  net.width = W;
  net.skip = skip;
  net.ready = true;
  return ADN_OK;
}

// ndc_rays' projection constants -1 / (W / (2 focal)), -1 / (H / (2 focal)): python doubles that are rounded once when
// they meet the fp32 tensors (src/nerf_raymarch_common.py:77-82).  focal <= 0: 0.5 W / tan(fov / 2) (src/datasets.py:181-182,
// adanerf_real_time_viewer/src/featureset.cpp:83-84).
void set_ndc_projection(adn_ctx* ctx, int W, int H, float focal_in) {
  const double focal = focal_in > 0.0f ? double(focal_in) : 0.5 * double(W) / std::tan(0.5 * double(ctx->scene.fov));
  ctx->sc.ndc_cw = float(-1.0 / (double(W) / (2.0 * focal)));
  ctx->sc.ndc_ch = float(-1.0 / (double(H) / (2.0 * focal)));
}

// The K depths of LinearlySpacedZNearZFar.generate with det = True (nerf_raymarch_common.py:310-326), which the thr == 0
// branch of FromClassifiedDepthAdaptive.generate (:708-720) shares, in torch's fp32 steps: t = linspace(0, 1, K + 1)[k] +
// 0.5 / K, with ATen's CPU linspace (k step below the half-way index, fma(-step, K - k, 1) from it on), z = z_near (1 - t) +
// z_far t, then LogTransform.to_world with the pow in double.  NDC scenes (the NoDepthRange samplers, :276-289 / :797-805)
// keep z.
std::vector<float> linear_depths(const adn_scene& sc, int K) {
  std::vector<float> lut(K);
  const double max_v = double(sc.depth_range[1]) - double(sc.depth_range[0]);
  const float step = 1.0f / float(K);
  for (int k = 0; k < K; ++k) {
    const float lin = (k < (K + 1) / 2) ? float(k) * step : std::fma(-step, float(K - k), 1.0f);
    const float t = lin + float(0.5 / K);
    const float z = sc.z_near * (1.0f - t) + sc.z_far * t;
    const float w = float(std::pow(max_v + 1.0, double(z)));
    lut[k] = sc.use_ndc ? z : (w - 1.0f) + sc.depth_range[0];
  }
  return lut;
}

adn_status ensure_dense_lut(adn_ctx* ctx, int K) {
  if (ctx->dense_K == K) return ADN_OK;
  const std::vector<float> lut = linear_depths(ctx->scene, K);
  adn_status s = ensure(ctx, ctx->zlut_dense, sizeof(float) * K);
  if (s != ADN_OK) return s;
  ADN_CUDA(ctx, cudaMemcpy(ctx->zlut_dense.p, lut.data(), sizeof(float) * K, cudaMemcpyHostToDevice));
  ctx->dense_K = K;
  return ADN_OK;
}

PoseDev make_pose(const float* pose, const float* rot) {
  PoseDev p;
  std::memcpy(p.pose, pose, 12);
  std::memcpy(p.rot, rot, 36);
  return p;
}

// The pinhole rays of image rows [row0, row0 + rows) of a W x H frame; none when that window does not fit the frame.
std::optional<CameraRays> camera_rays(const adn_ctx* ctx, int W, int H, int row0, int rows) {
  if (!ctx || W < 1 || H < 1 || row0 < 0 || rows < 0 || row0 + rows > H) return std::nullopt;
  // src/util/raygeneration.py:10-26 with focal = 0.5*W/tan(fov/2) (src/datasets.py:181-182), float64
  CameraRays c;
  const double fov = double(ctx->scene.fov);
  const double focal = 0.5 * W / std::tan(0.5 * fov);
  const double x_dist = std::tan(fov / 2) * focal;
  const double y_dist = x_dist * (double(H) / double(W));
  c.x_pp = x_dist / (W / 2.0);
  c.y_pp = y_dist / (H / 2.0);
  c.start_x = -(x_dist - c.x_pp / 2);
  c.start_y = -(y_dist - c.y_pp / 2);
  c.focal = focal;
  c.W = W;
  c.H = H;
  c.row0 = row0;
  return c;
}

int64_t pad128(int64_t n) { return (n + 127) / 128 * 128; }

// D, the depth cells of raw0 (multiDepthFeatures): the sampling net's outputs, 128 while none is set.
int depth_cells(const adn_ctx* ctx) { return ctx->net[0].ready ? ctx->net[0].n_out : 128; }

// The adaptive depth table of D cells: zlut at D = 128, else its slice of zlut_cells (32, then 64, then 256 entries).
const float* cell_table(const adn_ctx* ctx, int D) {
  if (D == 128) return ctx->zlut.as<float>();
  return ctx->zlut_cells.as<float>() + (D == 32 ? 0 : D == 64 ? 32 : 96);
}

// The adaptive depth table of D cells as adn_create uploads it: LogTransform.to_world((c + 0.5) / D)
// (depth_transformations.py:37-48, nerf_raymarch_common.py:738-742), pow in double, the rest in fp32; on NDC scenes
// (FromClassifiedDepthAdaptiveNoDepthRange, :826-833) the cell centre itself.  (c + 0.5) * (1 / D) is exact for D a power of 2.
std::vector<float> cell_depths(const adn_scene& sc, int D) {
  std::vector<float> lut(D);
  const double max_v = double(sc.depth_range[1]) - double(sc.depth_range[0]);
  for (int i = 0; i < D; ++i) {
    const float z = (float(i) + 0.5f) * (1.0f / float(D));
    const float w = float(std::pow(max_v + 1.0, double(z)));
    lut[i] = sc.use_ndc ? z : (w - 1.0f) + sc.depth_range[0];
  }
  return lut;
}

// Runs the sampling MLP into raw0 [rows, D].  At D < 128 the kernel writes rows of 128 columns (the padded N half) into
// ctx->raw0_pad, and a strided copy keeps the first D of each.
adn_status run_mlp0(adn_ctx* ctx, const uint8_t* tiles, float* raw0, long long rows, cudaStream_t st);

adn_status run_mlp(adn_ctx* ctx, int id, const uint8_t* tiles, float* out, const long long* rows_dev, long long rows,
                   cudaStream_t st, const EncodeParams* enc = nullptr) {
  Net& n = ctx->net[id];
  const cudaError_t e = launch_mlp(n.prog, n.wblob.as<uint8_t>(), tiles, out, rows_dev, rows, ctx->d_err, ctx->num_sms, st, enc);
  if (e != cudaSuccess) return cuda_fail(ctx, e, id == 0 ? "launch sampling MLP" : "launch shading MLP");
  ctx->stats.kernel_launches++;
  return ADN_OK;
}

adn_status run_mlp0(adn_ctx* ctx, const uint8_t* tiles, float* raw0, long long rows, cudaStream_t st) {
  const int D = ctx->net[0].n_out;
  if (D >= 128) return run_mlp(ctx, 0, tiles, raw0, nullptr, rows, st);
  adn_status s = ensure(ctx, ctx->raw0_pad, size_t(rows) * 128 * 4);
  if (s != ADN_OK || (s = run_mlp(ctx, 0, tiles, ctx->raw0_pad.as<float>(), nullptr, rows, st)) != ADN_OK) return s;
  ADN_CUDA(ctx, cudaMemcpy2DAsync(raw0, size_t(D) * 4, ctx->raw0_pad.p, 128 * 4, size_t(D) * 4, size_t(rows), cudaMemcpyDeviceToDevice, st));
  return ADN_OK;
}

// One render call: the camera pose, where the rays come from and where each output goes.  A chunk of a call is a call of
// its own (chunk_of).
struct RenderCall {
  const float* pose;                // [3], host ([n_views, 3] for several views)
  const float* rot;                 // [9] row-major, host ([n_views, 9])
  int n_views = 1;                  // > 1: the rays are view-major, n_per_view of each view, and stage 0 / the ray kernels
  int64_t n_per_view = 0;           // take each ray's camera from a ViewTable (views_of)
  int64_t ray0 = 0;                 // the chunk's first ray in the call (several views)
  const float* d_dirs = nullptr;    // the rays [n_rays, 3], or
  std::optional<CameraRays> cam;    // image rows whose pinhole rays are generated on the device
  int64_t n_rays;
  float thr;
  int K;
  float* d_rgb = nullptr;           // [n_rays, 3]
  uint8_t* d_rgba8 = nullptr;       // [n_rays, 4]
  int32_t* d_nsamples = nullptr;    // [n_rays]
  float* d_oracle_w = nullptr;      // [n_rays, D]: the sampling net's output
  adn_aux_outputs aux{};            // all null: none
  cudaStream_t st;
  RenderCall(const float* pose_, const float* rot_, int64_t n_rays_, float thr_, int K_, void* stream)
      : pose(pose_), rot(rot_), n_rays(n_rays_), thr(thr_), K(K_), st(static_cast<cudaStream_t>(stream)) {}
};

// Rays [r0, r0 + chunk) of a call (fewer at its end): the ray source and every output start at ray r0.  D: raw0's row width.
RenderCall chunk_of(const RenderCall& call, int64_t r0, int64_t chunk, int D) {
  RenderCall c = call;
  c.n_rays = std::min(chunk, call.n_rays - r0);
  if (c.d_dirs) c.d_dirs += 3 * r0;
  if (c.n_views > 1) c.ray0 = r0;   // the pixel is the ray's index inside its view; cam->row0 stays 0
  else if (c.cam) c.cam->row0 += int(r0 / c.cam->W);
  if (c.d_rgb) c.d_rgb += 3 * r0;
  if (c.d_rgba8) c.d_rgba8 += 4 * r0;
  if (c.d_nsamples) c.d_nsamples += r0;
  if (c.d_oracle_w) c.d_oracle_w += D * r0;
  for (float** p : {&c.aux.d_weights, &c.aux.d_alpha, &c.aux.d_z_vals})
    if (*p) *p += r0 * c.K;
  for (float** p : {&c.aux.d_depth_map, &c.aux.d_acc_map, &c.aux.d_disp_map, &c.aux.d_depth_est})
    if (*p) *p += r0;
  return c;
}

// Stage 5's optional outputs: the caller's arrays and the scene's depth constants behind depth_est.
Stage5Aux stage5_aux(const adn_ctx* ctx, const adn_aux_outputs& a) {
  const adn_scene& sc = ctx->scene;
  return {a.d_weights, a.d_alpha, a.d_z_vals, a.d_depth_map, a.d_acc_map, a.d_disp_map, a.d_depth_est, sc.use_ndc ? 1 : 0,
          sc.depth_range[0], float(std::log(double(sc.depth_range[1]) - double(sc.depth_range[0]) + 1.0))};
}

// depth_range[1] - depth_range[0] + 1 in double: the base of LogTransform.to_world (the z tables and the fixed-K sampler).
double depth_base(const adn_ctx* ctx) { return double(ctx->scene.depth_range[1]) - double(ctx->scene.depth_range[0]) + 1.0; }

// The camera table of a chunk of a call over several views (null for one view): a kernel parameter of the stage-0 and ray
// kernels, so each launch carries its own copy.
const ViewTable* views_of(const RenderCall& c, ViewTable& t) {
  if (c.n_views <= 1) return nullptr;
  t.ray0 = c.ray0;
  t.n_per_view = c.n_per_view;
  for (int v = 0; v < c.n_views; ++v) t.v[v] = make_pose(c.pose + 3 * v, c.rot + 9 * v);
  return &t;
}

// Stage 0 + the sampling MLP of one chunk, stream ordered.  Writes the chunk's raw0 [n, D] (the caller's
// d_oracle_weights when given, else the context's scratch from ray w on) and its ray origins / directions (scratch from ray
// w on).  w is 0 unless a sample budget keeps the whole call's rows.  timing: record ev[0..2].
adn_status run_stages_0_1(adn_ctx* ctx, const RenderCall& c, int64_t w, bool timing) {
  const Net& n0 = ctx->net[0];
  adn_status s = ensure(ctx, ctx->tiles0, size_t(pad128(c.n_rays) / 128) * n0.prog.in.tile_bytes());
  if (s != ADN_OK) return s;
  float* raw0 = c.d_oracle_w ? c.d_oracle_w : ctx->raw0.as<float>() + int64_t(depth_cells(ctx)) * w;
  uint8_t* tiles0 = ctx->tiles0.as<uint8_t>();
  ViewTable vt{};
  if (timing) cudaEventRecord(ctx->ev[0], c.st);
  // stage 0 (writes the sampling net's packed input tiles)
  ADN_CUDA(ctx, launch_stage0(ctx->sc, make_pose(c.pose, c.rot), c.d_dirs, c.cam ? &*c.cam : nullptr, c.n_rays, nullptr,
                              ctx->ray_o.as<float>() + 3 * w, ctx->ray_d.as<float>() + 3 * w, tiles0, n0.prog.in.n_terms, c.st,
                              views_of(c, vt)));
  ctx->stats.kernel_launches++;
  if (timing) cudaEventRecord(ctx->ev[1], c.st);
  // stage 1
  if ((s = run_mlp0(ctx, tiles0, raw0, c.n_rays, c.st)) != ADN_OK) return s;
  if (timing) cudaEventRecord(ctx->ev[2], c.st);
  return ADN_OK;
}

// Sampler 2's rays of one chunk, in place of stages 0-1: ray_o / ray_d for stage 3 and, on NDC scenes, the composite's NDC
// directions (ray_dirs).  timing: record ev[0..2] (stage 1's slot stays empty).
adn_status run_rays(adn_ctx* ctx, const RenderCall& c, bool timing) {
  ViewTable vt{};
  if (timing) cudaEventRecord(ctx->ev[0], c.st);
  ADN_CUDA(ctx, launch_camera_rays(ctx->sc, make_pose(c.pose, c.rot), c.d_dirs, c.cam ? &*c.cam : nullptr, c.n_rays,
                                   ctx->ray_o.as<float>(), ctx->ray_d.as<float>(),
                                   ctx->scene.use_ndc ? ctx->ray_dirs.as<float>() : nullptr, c.st, views_of(c, vt)));
  ctx->stats.kernel_launches++;
  if (timing) {
    cudaEventRecord(ctx->ev[1], c.st);
    cudaEventRecord(ctx->ev[2], c.st);
  }
  return ADN_OK;
}

// Sampler 2's depth table for K (1-128) in ctx->zlin.
const float* zlin_table(const adn_ctx* ctx, int K) { return ctx->zlin.as<float>() + K * (K - 1) / 2; }

// Stages 2-5 of one chunk, stream ordered: read what run_stages_0_1 (run_rays) wrote for the same chunk and w.  d_thr: stage 2's
// threshold as a device float (sample budget), null = c.thr.  timing: record ev[3..6].
adn_status run_stages_2_5(adn_ctx* ctx, const RenderCall& c, int64_t w, const float* d_thr, bool timing) {
  const int64_t n = c.n_rays;
  const int K = c.K;
  const bool fixed_k = ctx->sampler != 0;   // K samples on every ray and the density composite
  const bool linear = ctx->sampler == 2;    // LinearlySpacedZNearZFar: the depth table, no sampling net
  const bool dense = !fixed_k && c.thr == 0.0f;
  const int64_t cap = n * K;
  adn_status s;
  if ((s = ensure(ctx, ctx->count, size_t(n) * 4)) != ADN_OK) return s;
  if ((s = ensure(ctx, ctx->offset, size_t(n) * 4)) != ADN_OK) return s;
  if (!dense) {
    if ((s = ensure(ctx, ctx->rayidx, size_t(cap) * 4)) != ADN_OK) return s;
    if ((s = ensure(ctx, ctx->zbuf, size_t(cap) * 4)) != ADN_OK) return s;
  }
  if (!dense && !fixed_k) {
    if ((s = ensure(ctx, ctx->zpbuf, size_t(cap) * 4)) != ADN_OK) return s;
    if ((s = ensure(ctx, ctx->s2scratch, stage2_scratch_bytes(n))) != ADN_OK) return s;
  }
  // stage 3 runs inside the shading kernel (its producer warps encode the next tile) unless option fuse_encoder is 0 or
  // the scene is NDC: then stage3_kernel writes the packed tiles that the kernel's producer copies in
  const bool fused_enc = ctx->fuse_encoder && !ctx->scene.use_ndc;
  if (!fused_enc && (s = ensure(ctx, ctx->tiles1, size_t(pad128(cap) / 128) * ctx->net[1].prog.in.tile_bytes())) != ADN_OK) return s;
  if ((s = ensure(ctx, ctx->raw1, size_t(pad128(cap)) * 16)) != ADN_OK) return s;

  const int D = depth_cells(ctx);
  float* raw0 = linear ? nullptr : c.d_oracle_w ? c.d_oracle_w : ctx->raw0.as<float>() + int64_t(D) * w;
  const float* ray_o = ctx->ray_o.as<float>() + 3 * w;
  const float* ray_d = ctx->ray_d.as<float>() + 3 * w;
  int32_t* count = c.d_nsamples ? c.d_nsamples : ctx->count.as<int32_t>();
  int32_t* offset = ctx->offset.as<int32_t>();
  int32_t* rayidx = dense ? nullptr : ctx->rayidx.as<int32_t>();
  float* z = ctx->zbuf.as<float>();
  uint8_t* tiles1 = ctx->tiles1.as<uint8_t>();   // null / stale when the encoder is fused
  float* raw1 = ctx->raw1.as<float>();
  long long* total = ctx->total.as<long long>();

  // stage 2
  if (linear) {
    ADN_CUDA(ctx, launch_linear_sample(n, K, zlin_table(ctx, K), count, offset, rayidx, z, total, c.st));
  } else if (fixed_k) {
    ADN_CUDA(ctx, launch_pdf_sample(raw0, n, K, ctx->pdf_transform, depth_base(ctx), ctx->scene.depth_range[0], count, offset,
                                    rayidx, z, total, c.st));
  } else if (dense) {
    ADN_CUDA(ctx, launch_stage2_dense(n, K, count, offset, total, c.st));
  } else {
    ADN_CUDA(ctx, launch_stage2(raw0, n, c.thr, K, cell_table(ctx, D), count, offset, nullptr, rayidx, z, ctx->zpbuf.as<float>(),
                                total, ctx->s2scratch.p, &ctx->s2sync, c.st, d_thr, D));
  }
  ctx->stats.kernel_launches++;
  if (timing) cudaEventRecord(ctx->ev[3], c.st);
  // stage 3 (+ 4)
  const EncodeParams ep{ray_o, ray_d, rayidx, z, ctx->zlut_dense.as<float>(), K, ctx->sc};   // read when fused_enc
  if (!fused_enc) {
    ADN_CUDA(ctx, launch_stage3(ctx->sc, ray_o, ray_d, rayidx, z, ctx->zlut_dense.as<float>(), K, cap, total, nullptr, tiles1,
                                ctx->num_sms, c.st));
    ctx->stats.kernel_launches++;
  }
  if (timing) cudaEventRecord(ctx->ev[4], c.st);
  // stage 4
  if ((s = run_mlp(ctx, 1, fused_enc ? nullptr : tiles1, raw1, total, cap, c.st, fused_enc ? &ep : nullptr)) != ADN_OK) return s;
  if (timing) cudaEventRecord(ctx->ev[5], c.st);
  // stage 5
  ADN_CUDA(ctx, launch_stage5(raw1, dense ? raw0 : ctx->zpbuf.as<float>(), z, ctx->zlut_dense.as<float>(), offset, count, n, K,
                              dense ? 1 : 0, c.d_rgb, c.d_rgba8, stage5_aux(ctx, c.aux), c.st,
                              !fixed_k ? nullptr : linear && ctx->scene.use_ndc ? ctx->ray_dirs.as<float>() : ray_d));
  ctx->stats.kernel_launches++;
  if (timing) cudaEventRecord(ctx->ev[6], c.st);
  return ADN_OK;
}

// The sampling net's view of one chunk in place of stages 2-5 (option "sampling_view"): reads what run_stages_0_1 wrote
// for the same chunk.  The view counts no samples: d_nsamples is zeroed.  timing: record ev[5..6].
adn_status run_view(adn_ctx* ctx, const RenderCall& c, bool timing) {
  const float* raw0 = c.d_oracle_w ? c.d_oracle_w : ctx->raw0.as<float>();
  if (c.d_nsamples) ADN_CUDA(ctx, cudaMemsetAsync(c.d_nsamples, 0, size_t(c.n_rays) * 4, c.st));
  if (timing) cudaEventRecord(ctx->ev[5], c.st);
  ADN_CUDA(ctx, launch_sampling_view(raw0, c.n_rays, c.d_rgb, c.d_rgba8, c.st));
  ctx->stats.kernel_launches++;
  if (timing) cudaEventRecord(ctx->ev[6], c.st);
  return ADN_OK;
}

// The hot path for every render entry point: stream ordered, no host synchronisation.  The call runs in chunks of rays;
// with a sample budget, stages 0-1 of every chunk, then one threshold for the whole call, then stages 2-5 of every chunk.
// With option "sampling_view", stages 0-1 and the view of every chunk, and no sample budget.
adn_status render(adn_ctx* ctx, const RenderCall& call) {
  const int64_t n_rays = call.n_rays;
  const float thr = call.thr;
  const int K = call.K;
  const bool joins = joins_group(ctx);   // an empty call still joins the selection's reductions
  if (!ctx || !call.pose || !call.rot || n_rays < 0 || (!call.d_rgb && !call.d_rgba8 && !(joins && n_rays == 0)))
    return fail(ctx, ADN_ERR_INVALID, "render: bad arguments");
  const bool linear = ctx->sampler == 2;   // LinearlySpacedZNearZFar: one network, in the shading slot
  if (linear && !ctx->net[1].ready) return fail(ctx, ADN_ERR_NO_WEIGHTS, "render: set the shading network (slot 1) first");
  if (!linear && (!ctx->net[0].ready || !ctx->net[1].ready)) return fail(ctx, ADN_ERR_NO_WEIGHTS, "render: set both networks first");
  if (!linear && ctx->net[0].n_in != ctx->n_feat0)
    return fail(ctx, ADN_ERR_INVALID, "render: sampling net must have " + std::to_string(ctx->n_feat0) + " inputs for this scene's encoding");
  const int D = linear ? 128 : depth_cells(ctx);   // depth cells of raw0 (multiDepthFeatures)
  if (D != 128 && ctx->sampler == 1)
    return fail(ctx, ADN_ERR_INVALID, "render: sampler 1 (FromClassifiedDepth) supports 128 depth cells only; this sampling net has " +
                                          std::to_string(D));
  if (D != 128 && ctx->sampling_view)
    return fail(ctx, ADN_ERR_INVALID, "render: option sampling_view supports 128 depth cells only; this sampling net has " +
                                          std::to_string(D));
  if (linear && ctx->sampling_view)
    return fail(ctx, ADN_ERR_INVALID, "render: sampler 2 (LinearlySpacedZNearZFar) runs no sampling net, so option sampling_view has nothing to draw");
  if (linear && call.d_oracle_w)
    return fail(ctx, ADN_ERR_INVALID, "render: sampler 2 (LinearlySpacedZNearZFar) runs no sampling net; pass d_oracle_weights = NULL");
  if (linear && ctx->sample_budget > 0)
    return fail(ctx, ADN_ERR_INVALID, "render: sampler 2 (LinearlySpacedZNearZFar) places K samples on every ray; it takes no sample_budget");
  const bool fixed_k = ctx->sampler != 0;   // FromClassifiedDepth and LinearlySpacedZNearZFar ignore thr
  if (K < 1 || K > std::min(D, 128) || (!fixed_k && thr < 0.0f))
    return fail(ctx, ADN_ERR_INVALID, "render: need 1 <= K <= " + std::to_string(std::min(D, 128)) + " and thr >= 0" +
                                          (D != 128 ? " (" + std::to_string(D) + " depth cells)" : std::string()));
  if (!fixed_k && thr == 0.0f && K != D)
    return fail(ctx, ADN_ERR_INVALID, "render: dense mode (thr == 0) needs K == " + std::to_string(D) + " (one sample per depth cell)" +
                                          (D > 128 ? "; K is at most 128, so 256 depth cells have no dense mode" : ""));
  const bool view = ctx->sampling_view;
  if (view) {
    const adn_aux_outputs& a = call.aux;
    if (a.d_weights || a.d_alpha || a.d_z_vals || a.d_depth_map || a.d_acc_map || a.d_disp_map || a.d_depth_est)
      return fail(ctx, ADN_ERR_INVALID, "render: option sampling_view draws no auxiliary outputs (pass none)");
    if (reinterpret_cast<uintptr_t>(call.d_oracle_w) & 15u)
      return fail(ctx, ADN_ERR_INVALID, "render: option sampling_view needs 16-byte aligned d_oracle_weights rows");
  }
  const int64_t budget = view ? 0 : ctx->sample_budget;   // the view selects no samples
  if (fixed_k && budget > 0)
    return fail(ctx, ADN_ERR_INVALID, "render: sampler 1 (FromClassifiedDepth) places K samples on every ray; it takes no sample_budget");
  if (ctx->sampler == 1 && ctx->scene.use_ndc)
    return fail(ctx, ADN_ERR_INVALID, "render: sampler 1 (FromClassifiedDepth) is not supported on NDC scenes");
  if (budget > 0 && thr == 0.0f)
    return fail(ctx, ADN_ERR_INVALID, "render: sample_budget needs the adaptive path (thr > 0 is the floor threshold), not dense mode");
  if (budget > 0 && budget < n_rays)
    return fail(ctx, ADN_ERR_INVALID, "render: sample_budget " + std::to_string(budget) + " is below the " + std::to_string(n_rays) +
                                          " rays of the call (every ray keeps at least one sample)");
  if (budget > 0 && n_rays * (K - 1) >= (int64_t(1) << 32))
    return fail(ctx, ADN_ERR_INVALID, "render: sample_budget supports at most 2^32 - 1 candidate samples (N * (K - 1)) per call");
  if (budget > 0 && D == 128 && (reinterpret_cast<uintptr_t>(call.d_oracle_w) & 15u))
    return fail(ctx, ADN_ERR_INVALID, "render: sample_budget needs 16-byte aligned d_oracle_weights rows");
  if (n_rays == 0 && !joins) return ADN_OK;
  if (ctx->scene.use_ndc && n_rays > 0) {
    // image size behind ndc_rays: the frame being rendered (viewer, featureset.cpp:83-84) or the dataset's (features.py:350-351,430)
    if (call.cam) set_ndc_projection(ctx, call.cam->W, call.cam->H, 0.0f);
    else if (ctx->scene.ndc_w > 0 && ctx->scene.ndc_h > 0) set_ndc_projection(ctx, ctx->scene.ndc_w, ctx->scene.ndc_h, ctx->scene.ndc_focal);
    else return fail(ctx, ADN_ERR_INVALID, "render: NDC scene needs ndc_w / ndc_h when rays are passed explicitly");
  }
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  adn_status s;
  if (!fixed_k && thr == 0.0f && (s = ensure_dense_lut(ctx, K)) != ADN_OK) return s;
  int64_t chunk = ctx->chunk_rays;
  if (chunk <= 0) {
    chunk = (int64_t(8) << 20) / K;     // ~8 Mi samples of scratch per chunk
    if (chunk < 8192) chunk = 8192;
  }
  chunk = pad128(chunk);
  if (call.cam && chunk % call.cam->W) chunk = (chunk / call.cam->W + 1) * call.cam->W;  // whole rows per chunk
  if (linear && std::min(chunk, n_rays) * K > INT32_MAX)
    return fail(ctx, ADN_ERR_INVALID, "render: sampler 2 needs N * K < 2^31 per chunk (int32 offsets); lower option chunk_rays");
  ctx->stats.n_rays = n_rays;
  ctx->last_budget = budget > 0;
  ctx->last_thr = thr;
  ctx->last_view = view;
  if (ctx->profile) ctx->prof_budget = budget > 0;
  if (ctx->profile) ctx->prof_view = view;
  if (ctx->profile) ctx->prof_linear = linear;
  // raw0 / ray_o / ray_d: one chunk's worth, or with a sample budget the whole call's (the threshold is chosen over all of
  // raw0 before any chunk runs stage 2)
  const int64_t span = budget > 0 ? n_rays : std::min(chunk, n_rays);
  if (!linear && !call.d_oracle_w && (s = ensure(ctx, ctx->raw0, size_t(span) * D * 4)) != ADN_OK) return s;
  if (!linear && D < 128 && (s = ensure(ctx, ctx->raw0_pad, size_t(std::min(chunk, n_rays)) * 128 * 4)) != ADN_OK) return s;
  if (linear && ctx->scene.use_ndc && (s = ensure(ctx, ctx->ray_dirs, size_t(span) * 12)) != ADN_OK) return s;
  if ((s = ensure(ctx, ctx->ray_o, size_t(span) * 12)) != ADN_OK) return s;
  if ((s = ensure(ctx, ctx->ray_d, size_t(span) * 12)) != ADN_OK) return s;
  if (budget == 0) {
    for (int64_t r0 = 0; r0 < n_rays; r0 += chunk) {
      const RenderCall c = chunk_of(call, r0, chunk, D);
      const bool timing = ctx->profile && r0 == 0;
      if ((s = linear ? run_rays(ctx, c, timing) : run_stages_0_1(ctx, c, 0, timing)) != ADN_OK) return s;
      if ((s = view ? run_view(ctx, c, timing) : run_stages_2_5(ctx, c, 0, nullptr, timing)) != ADN_OK) return s;
    }
    return ADN_OK;
  }
  if ((s = ensure(ctx, ctx->budget_keys, size_t(std::max<int64_t>(1, n_rays * (K - 1))) * 4)) != ADN_OK) return s;
  if ((s = ensure(ctx, ctx->budget_work, budget_work_bytes())) != ADN_OK) return s;
  if ((s = ensure(ctx, ctx->budget_thr, sizeof(float))) != ADN_OK) return s;
  float* d_thr = ctx->budget_thr.as<float>();
  for (int64_t r0 = 0; r0 < n_rays; r0 += chunk)
    if ((s = run_stages_0_1(ctx, chunk_of(call, r0, chunk, D), r0, ctx->profile && r0 == 0)) != ADN_OK) return s;
  if (ctx->profile) cudaEventRecord(ctx->ev[7], call.st);   // the selection is timed with stage 2 of the first chunk
  int launches = 0;
  ADN_CUDA(ctx, launch_budget_threshold(call.d_oracle_w ? call.d_oracle_w : ctx->raw0.as<float>(), n_rays, thr, K, budget,
                                        ctx->budget_keys.as<uint32_t>(), ctx->budget_work.p, d_thr, ctx->num_sms, call.st, &launches,
                                        &ctx->group, D));
  ctx->stats.kernel_launches += launches;
  if (ctx->group.failed_round >= 0) return group_fail(ctx, "render");
  for (int64_t r0 = 0; r0 < n_rays; r0 += chunk)
    if ((s = run_stages_2_5(ctx, chunk_of(call, r0, chunk, D), r0, d_thr, ctx->profile && r0 == 0)) != ADN_OK) return s;
  return ADN_OK;
}

// render() as one call of a device entry point, ordered after the context's earlier calls (CallOrder).
adn_status render_ordered(adn_ctx* ctx, const RenderCall& call, const char* who) {
  if (!ctx) return ADN_ERR_INVALID;
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  CallOrder order(ctx, call.st);
  const adn_status s = order.begin(who);
  return s != ADN_OK ? s : render(ctx, call);
}

adn_status check_device_error(adn_ctx* ctx) {
  int err = 0;
  cudaError_t e = cudaDeviceSynchronize();
  err = *ctx->watchdog.as<volatile int>();
  if (e != cudaSuccess && !err) return cuda_fail(ctx, e, "device synchronize");
  if (err) return fail(ctx, ADN_ERR_KERNEL, "device watchdog: mbarrier wait timed out at site " + std::to_string(err & 0xfff));
  return ADN_OK;
}

// Enqueues the copy of `bytes` from device memory d to the caller's host array h: straight into h when pin_in_place allows,
// otherwise into the pinned staging buffer `stage`, from which the caller copies on once the stream has synchronised
// (*staged).
adn_status copy_out(adn_ctx* ctx, void* h, const void* d, size_t bytes, Buf& stage, cudaStream_t st, bool* staged) {
  adn_status s;
  *staged = !pin_in_place(ctx, h, bytes);
  if (*staged && (s = ensure(ctx, stage, bytes)) != ADN_OK) return s;
  ADN_CUDA(ctx, cudaMemcpyAsync(*staged ? stage.p : h, d, bytes, cudaMemcpyDeviceToHost, st));
  return ADN_OK;
}

// The *_host entry points: the rays are copied in from h_dirs when given (else generated from c.cam), rendered on the
// context's stream, and rgb / n_samples copied out to the caller's arrays.  Returns once they have landed.
adn_status render_host(adn_ctx* ctx, RenderCall c, const float* h_dirs, float* h_rgb, int32_t* h_nsamples) {
  const size_t n = size_t(c.n_rays);
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  c.st = ctx->own_stream;
  CallOrder order(ctx, c.st);
  adn_status s = order.begin("render_host");
  if (s != ADN_OK) return s;
  if (h_dirs) {
    const bool staged = !pin_in_place(ctx, h_dirs, n * 12);
    if ((s = ensure(ctx, ctx->dirs, n * 12)) != ADN_OK || (staged && (s = ensure(ctx, ctx->h_in, n * 12)) != ADN_OK)) return s;
    if (staged) std::memcpy(ctx->h_in.p, h_dirs, n * 12);
    ADN_CUDA(ctx, cudaMemcpyAsync(ctx->dirs.p, staged ? ctx->h_in.p : h_dirs, n * 12, cudaMemcpyHostToDevice, c.st));
    c.d_dirs = ctx->dirs.as<float>();
  }
  if ((s = ensure(ctx, ctx->rgb, n * 12)) != ADN_OK) return s;
  if (h_nsamples && (s = ensure(ctx, ctx->nsamples, n * 4)) != ADN_OK) return s;
  c.d_rgb = ctx->rgb.as<float>();
  c.d_nsamples = h_nsamples ? ctx->nsamples.as<int32_t>() : nullptr;
  if ((s = render(ctx, c)) != ADN_OK) return s;
  bool rgb_staged = false, ns_staged = false;
  if ((s = copy_out(ctx, h_rgb, c.d_rgb, n * 12, ctx->h_out, c.st, &rgb_staged)) != ADN_OK) return s;
  if (h_nsamples && (s = copy_out(ctx, h_nsamples, c.d_nsamples, n * 4, ctx->h_ns, c.st, &ns_staged)) != ADN_OK) return s;
  ADN_CUDA(ctx, cudaStreamSynchronize(c.st));
  if (rgb_staged) std::memcpy(h_rgb, ctx->h_out.p, n * 12);
  if (ns_staged) std::memcpy(h_nsamples, ctx->h_ns.p, n * 4);
  return check_device_error(ctx);
}

// The checks every views entry makes before anything is enqueued: the camera tables and V (at most kMaxViews, the
// ViewTable a kernel parameter holds), N >= 1 rays per view and V N within int64.
adn_status check_views(adn_ctx* ctx, const char* who, int n_views, const float* poses, const float* rots, int64_t n_per_view) {
  const std::string w(who);
  if (!ctx) return ADN_ERR_INVALID;
  if (n_views < 1 || n_views > kMaxViews)
    return fail(ctx, ADN_ERR_INVALID, w + ": n_views must be 1-" + std::to_string(kMaxViews) + ", not " + std::to_string(n_views));
  if (!poses || !rots) return fail(ctx, ADN_ERR_INVALID, w + ": poses and rots must not be null");
  if (n_per_view < 1) return fail(ctx, ADN_ERR_INVALID, w + ": every view needs at least one ray");
  if (n_per_view > INT64_MAX / n_views)
    return fail(ctx, ADN_ERR_INVALID, w + ": n_views * rays per view overflows a 64-bit ray count");
  return ADN_OK;
}

// A views call over the camera entries: V frames of W x H, every pixel of every view.
adn_status render_views_camera(adn_ctx* ctx, const char* who, int n_views, const float* poses, const float* rots, int W, int H,
                               float thr, int K, float* d_rgb, int32_t* d_nsamples, uint8_t* d_rgba8, void* stream) {
  const std::optional<CameraRays> cam = camera_rays(ctx, W, H, 0, H);
  if (ctx && !cam) return fail(ctx, ADN_ERR_INVALID, std::string(who) + ": bad image size");
  adn_status s = check_views(ctx, who, n_views, poses, rots, int64_t(std::max(W, 0)) * std::max(H, 0));
  if (s != ADN_OK) return s;
  RenderCall c(poses, rots, int64_t(W) * H * n_views, thr, K, stream);
  c.cam = cam;
  c.n_views = n_views;
  c.n_per_view = int64_t(W) * H;
  c.d_rgb = d_rgb;
  c.d_nsamples = d_nsamples;
  c.d_rgba8 = d_rgba8;
  return render_ordered(ctx, c, who);
}

}  // namespace

// =================================================================================================
extern "C" {

const char* adn_version(void) { return "adanerf_b200 0.1 (sm_90a)"; }

const char* adn_strerror(adn_status s) {
  if (s < 0 || s > ADN_ERR_KERNEL) return "unknown status";
  return kStatusText[s];
}

const char* adn_last_error(const adn_ctx* ctx) { return ctx ? ctx->last_error.c_str() : "null context"; }

adn_status adn_create(adn_ctx** out, const adn_scene* scene, int device) {
  if (!out || !scene) return ADN_ERR_INVALID;
  *out = nullptr;
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || device < 0 || device >= n_dev) return ADN_ERR_NO_DEVICE;
  cudaDeviceProp prop{};
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return ADN_ERR_NO_DEVICE;
  if (prop.major != 9) return ADN_ERR_NO_DEVICE;  // wgmma / setmaxnreg kernels (sm_90a): Hopper only, no fallback
  // Band counts; a negative one is posEnc none, the same features as 0 bands.  The sampling net's fields default (0) to
  // the shading net's.  The limits are those of the packed tile formats (tiles.cuh): the shading net's position block at
  // most 2 x 64 columns (3 + 6 P), its view block at most 64 (3 + 6 D), the sampling net's 6 + 6 (P0 + D0) at most 128.
  const int nfp = std::max(0, scene->n_freq_pos), nfd = std::max(0, scene->n_freq_dir);
  const int nfp0 = std::max(0, scene->n_freq_pos0 ? scene->n_freq_pos0 : scene->n_freq_pos);
  const int nfd0 = std::max(0, scene->n_freq_dir0 ? scene->n_freq_dir0 : scene->n_freq_dir);
  if (nfp > 20 || nfd > 10 || nfp0 + nfd0 > 20) return ADN_ERR_INVALID;
  if (scene->use_ndc && (scene->ndc_w < 0 || scene->ndc_h < 0)) return ADN_ERR_INVALID;
  adn_ctx* ctx = new adn_ctx();
  ctx->device = device;
  ctx->num_sms = prop.multiProcessorCount;
  ctx->scene = *scene;
  if (cudaSetDevice(device) != cudaSuccess) {
    delete ctx;
    return ADN_ERR_CUDA;
  }
  for (int a = 0; a < 3; ++a) ctx->sc.c[a] = scene->view_cell_center[a];
  // view_cell_radius = ||size/2|| in float64, squared in float64, then rounded to fp32 (features.py:761,786)
  double r2 = 0;
  for (int a = 0; a < 3; ++a) r2 += (double(scene->view_cell_size[a]) / 2.0) * (double(scene->view_cell_size[a]) / 2.0);
  const double r = std::sqrt(r2);
  ctx->sc.r2 = float(r * r);
  ctx->sc.sqrt_max_depth = float(std::sqrt(double(scene->max_depth)));
  ctx->sc.n_freq_pos = nfp;
  ctx->sc.n_freq_dir = nfd;
  ctx->sc.n_freq_pos0 = nfp0;
  ctx->sc.n_freq_dir0 = nfd0;
  ctx->n_feat0 = 6 + 6 * (nfp0 + nfd0);
  ctx->sc.ndc = scene->use_ndc ? 1 : 0;
  if (scene->use_ndc && scene->ndc_w > 0 && scene->ndc_h > 0) set_ndc_projection(ctx, scene->ndc_w, scene->ndc_h, scene->ndc_focal);
  // z LUT of the default 128 depth cells (cell_depths)
  const std::vector<float> lut = cell_depths(*scene, 128);
  // sampler 2's depth tables, one per K, so that no render uploads one
  std::vector<float> zlin;
  for (int K = 1; K <= 128; ++K) {
    const std::vector<float> t = linear_depths(*scene, K);
    zlin.insert(zlin.end(), t.begin(), t.end());
  }
  // the tables of the other depth-cell counts (multiDepthFeatures 32, 64, 256), in cell_table's order
  std::vector<float> zcells;
  for (int D : {32, 64, 256}) {
    const std::vector<float> t = cell_depths(*scene, D);
    zcells.insert(zcells.end(), t.begin(), t.end());
  }
  bool ok = ensure(ctx, ctx->zlut, lut.size() * 4) == ADN_OK &&
            cudaMemcpy(ctx->zlut.p, lut.data(), lut.size() * 4, cudaMemcpyHostToDevice) == cudaSuccess &&
            ensure(ctx, ctx->zlut_cells, zcells.size() * 4) == ADN_OK &&
            cudaMemcpy(ctx->zlut_cells.p, zcells.data(), zcells.size() * 4, cudaMemcpyHostToDevice) == cudaSuccess &&
            ensure(ctx, ctx->zlin, zlin.size() * 4) == ADN_OK &&
            cudaMemcpy(ctx->zlin.p, zlin.data(), zlin.size() * 4, cudaMemcpyHostToDevice) == cudaSuccess &&
            ensure(ctx, ctx->total, sizeof(long long)) == ADN_OK &&
            cudaMemset(ctx->total.p, 0, sizeof(long long)) == cudaSuccess &&
            cudaHostAlloc(&ctx->watchdog.p, sizeof(int), cudaHostAllocMapped) == cudaSuccess &&
            cudaHostGetDevicePointer(&ctx->d_err, ctx->watchdog.p, 0) == cudaSuccess && (*ctx->watchdog.as<int>() = 0, true) &&
            cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking) == cudaSuccess &&
            cudaEventCreateWithFlags(&ctx->order, cudaEventDisableTiming) == cudaSuccess;
  for (int i = 0; ok && i < 8; ++i) ok = cudaEventCreate(&ctx->ev[i]) == cudaSuccess;
  if (!ok) {
    adn_destroy(ctx);
    return ADN_ERR_CUDA;
  }
  *out = ctx;
  return ADN_OK;
}

void adn_destroy(adn_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  for (auto& r : ctx->regs)
    if (r.p) cudaHostUnregister(const_cast<void*>(r.p));
  for (int i = 0; i < 8; ++i)
    if (ctx->ev[i]) cudaEventDestroy(ctx->ev[i]);
  if (ctx->order) cudaEventDestroy(ctx->order);
  if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
  delete ctx;   // frees every Buf on this device
}

adn_status adn_set_weights(adn_ctx* ctx, int net_id, const adn_tensor_desc* tensors, int n_tensors) {
  if (!ctx || (net_id != 0 && net_id != 1) || !tensors || n_tensors < 1) return fail(ctx, ADN_ERR_INVALID, "set_weights: bad arguments");
  if (net_id == 0 && ctx->sampler == 2)
    return fail(ctx, ADN_ERR_INVALID, "set_weights: option sampler 2 (LinearlySpacedZNearZFar) runs no sampling network; "
                                      "set sampler 0 or 1 first");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  ADN_CUDA(ctx, cudaDeviceSynchronize());
  Net& net = ctx->net[net_id];
  net.ready = false;
  net.tensors.clear();
  for (int i = 0; i < n_tensors; ++i) {
    const adn_tensor_desc& t = tensors[i];
    if (!t.name || !t.data || t.rows < 1 || t.cols < 1) return fail(ctx, ADN_ERR_INVALID, "set_weights: bad tensor descriptor");
    HostTensor h;
    const std::string name(t.name);
    const bool is_bias = name.size() > 5 && name.compare(name.size() - 5, 5, ".bias") == 0;
    h.rows = is_bias ? t.rows * t.cols : t.rows;
    h.cols = is_bias ? 1 : t.cols;
    h.data.assign(t.data, t.data + t.rows * t.cols);
    net.tensors[name] = std::move(h);
  }
  return net_id == 0 ? build_net0(ctx) : build_net1(ctx);
}

adn_status adn_set_option(adn_ctx* ctx, const char* name, int64_t value) {
  if (!ctx || !name) return ADN_ERR_INVALID;
  const std::string n(name);
  if (n == "chunk_rays") {
    if (value < 0) return fail(ctx, ADN_ERR_INVALID, "chunk_rays must be >= 0");
    ctx->chunk_rays = value;
    return ADN_OK;
  }
  if (n == "profile") {
    ctx->profile = value != 0;
    return ADN_OK;
  }
  if (n == "sample_budget") {   // B > 0: adaptive renders choose their threshold (>= thr) so that M <= B; 0 (default): off
    if (value < 0) return fail(ctx, ADN_ERR_INVALID, "sample_budget must be >= 0");
    ctx->sample_budget = value;
    return ADN_OK;
  }
  if (n == "sampling_view") {   // 1: renders draw the sampling net's view (the viewer's render-oracle mode); 0 (default): off
    if (value != 0 && value != 1) return fail(ctx, ADN_ERR_INVALID, "sampling_view must be 0 or 1");
    ctx->sampling_view = value != 0;
    return ADN_OK;
  }
  if (n == "sampler") {   // 0 (default): FromClassifiedDepthAdaptive; 1: FromClassifiedDepth (DONeRF's fixed K samples per ray);
                          // 2: LinearlySpacedZNearZFar (NeRF's K evenly spaced samples, no sampling net)
    if (value < 0 || value > 2)
      return fail(ctx, ADN_ERR_INVALID, "sampler must be 0 (adaptive), 1 (FromClassifiedDepth) or 2 (LinearlySpacedZNearZFar)");
    // a context holding a sampling net belongs to a two-network run, whose shading net was trained on that net's samples:
    // rendering it alone as a NeRF would ignore the sampling net and give a picture of nothing the run trained
    if (value == 2 && ctx->net[0].ready)
      return fail(ctx, ADN_ERR_INVALID, "sampler 2 (LinearlySpacedZNearZFar) renders one network from the shading slot, but this "
                                        "context holds a sampling network (a two-network run); use a context without one");
    ctx->sampler = int(value);
    return ADN_OK;
  }
  if (n == "pdf_transform") {   // FromClassifiedDepth's transform of raw0: 1 (default) sigmoid, 2 softmax
    if (value != kPdfSigmoid && value != kPdfSoftmax)
      return fail(ctx, ADN_ERR_INVALID, "pdf_transform must be 1 (sigmoid, BCEWithLogitsLoss) or 2 (softmax, CrossEntropyLoss); "
                                        "0 (no transform) is not supported");
    ctx->pdf_transform = int(value);
    return ADN_OK;
  }
  if (n == "fuse_encoder") {   // 1 (default): positional encoding inside the shading kernel (no tile buffer); 0: stage3_kernel + packed tiles
    ctx->fuse_encoder = value != 0;
    return ADN_OK;
  }
  if (n == "mlp0_terms") {
    if (value != 1 && value != 3) return fail(ctx, ADN_ERR_INVALID, "mlp0_terms must be 1 or 3");
    ctx->mlp0_terms = int(value);
    if (!ctx->net[0].tensors.empty()) {
      ADN_CUDA(ctx, cudaSetDevice(ctx->device));
      ADN_CUDA(ctx, cudaDeviceSynchronize());
      return build_net0(ctx);
    }
    return ADN_OK;
  }
  return fail(ctx, ADN_ERR_INVALID, "unknown option " + n);
}

adn_status adn_set_budget_group(adn_ctx* ctx, adn_budget_reduce_fn fn, void* user) {
  if (!ctx) return ADN_ERR_INVALID;
  ctx->group.fn = fn;
  ctx->group.user = fn ? user : nullptr;
  return ADN_OK;
}

adn_status adn_get_stats(adn_ctx* ctx, adn_stats* out) {
  if (!ctx || !out) return ADN_ERR_INVALID;
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  adn_status s = check_device_error(ctx);   // synchronises; reports a tripped device watchdog with its site
  if (s != ADN_OK) return s;
  long long total = 0;
  ADN_CUDA(ctx, cudaMemcpy(&total, ctx->total.p, sizeof(total), cudaMemcpyDeviceToHost));
  ctx->stats.n_samples = ctx->last_view ? 0 : total;
  if (ctx->profile) {
    for (int i = 0; i < 6; ++i) {
      float ms = 0;
      if ((ctx->prof_view && i >= 2 && i <= 4) || (ctx->prof_linear && i == 1)) {   // the view runs no stages 2-4, sampler 2 no stage 1
        ctx->stats.ms_stage[i] = 0.0f;
        continue;
      }
      // with a sample budget, stage 2's slot starts at the threshold selection (ev[7])
      const cudaEvent_t from = (i == 2 && ctx->prof_budget) ? ctx->ev[7] : ctx->ev[i];
      if (cudaEventElapsedTime(&ms, from, ctx->ev[i + 1]) == cudaSuccess) ctx->stats.ms_stage[i] = ms;
    }
  }
  *out = ctx->stats;
  return ADN_OK;
}

adn_status adn_last_threshold(adn_ctx* ctx, float* thr_out) {
  if (!ctx || !thr_out) return fail(ctx, ADN_ERR_INVALID, "last_threshold: bad arguments");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  adn_status s = check_device_error(ctx);   // synchronises, like adn_get_stats
  if (s != ADN_OK) return s;
  if (ctx->last_budget) ADN_CUDA(ctx, cudaMemcpy(thr_out, ctx->budget_thr.p, sizeof(float), cudaMemcpyDeviceToHost));
  else *thr_out = ctx->last_thr;
  return ADN_OK;
}

adn_status adn_render_rays(adn_ctx* ctx, const float* pose, const float* rot, const float* d_dirs, int64_t n_rays, float thr,
                           int K, float* d_rgb, int32_t* d_nsamples, float* d_oracle_weights, void* stream) {
  if (ctx && n_rays == 0 && !joins_group(ctx)) return ADN_OK;   // empty batch: nothing to read or write
  if (!d_dirs && n_rays != 0) return fail(ctx, ADN_ERR_INVALID, "render_rays: d_dirs is null");
  return adn_render_rays_aux(ctx, pose, rot, d_dirs, n_rays, thr, K, d_rgb, d_nsamples, d_oracle_weights, nullptr, stream);
}

adn_status adn_render_rays_aux(adn_ctx* ctx, const float* pose, const float* rot, const float* d_dirs, int64_t n_rays, float thr,
                               int K, float* d_rgb, int32_t* d_nsamples, float* d_oracle_weights, const adn_aux_outputs* aux,
                               void* stream) {
  if (ctx && n_rays == 0 && !joins_group(ctx)) return ADN_OK;
  if (!d_dirs && n_rays != 0) return fail(ctx, ADN_ERR_INVALID, "render_rays_aux: d_dirs is null");
  RenderCall c(pose, rot, n_rays, thr, K, stream);
  c.d_dirs = d_dirs;
  c.d_rgb = d_rgb;
  c.d_nsamples = d_nsamples;
  c.d_oracle_w = d_oracle_weights;
  if (aux) c.aux = *aux;
  return render_ordered(ctx, c, "render_rays");
}

adn_status adn_render_camera(adn_ctx* ctx, const float* pose, const float* rot, int W, int H, int row0, int rows, float thr,
                             int K, float* d_rgb, int32_t* d_nsamples, void* stream) {
  RenderCall c(pose, rot, int64_t(rows) * W, thr, K, stream);
  c.cam = camera_rays(ctx, W, H, row0, rows);
  if (!c.cam) return fail(ctx, ADN_ERR_INVALID, "render_camera: bad image window");
  c.d_rgb = d_rgb;
  c.d_nsamples = d_nsamples;
  return render_ordered(ctx, c, "render_camera");
}

adn_status adn_render_camera_rgba8(adn_ctx* ctx, const float* pose, const float* rot, int W, int H, int row0, int rows,
                                   float thr, int K, uint8_t* d_rgba8, void* stream) {
  RenderCall c(pose, rot, int64_t(rows) * W, thr, K, stream);
  c.cam = camera_rays(ctx, W, H, row0, rows);
  if (!c.cam) return fail(ctx, ADN_ERR_INVALID, "render_camera: bad image window");
  c.d_rgba8 = d_rgba8;
  return render_ordered(ctx, c, "render_camera_rgba8");
}

adn_status adn_render_camera_surface(adn_ctx* ctx, const float* pose, const float* rot, int W, int H, int row0, int rows,
                                     float thr, int K, unsigned long long surface, void* stream) {
  RenderCall c(pose, rot, int64_t(rows) * W, thr, K, stream);
  c.cam = camera_rays(ctx, W, H, row0, rows);
  if (!c.cam || !surface) return fail(ctx, ADN_ERR_INVALID, "render_camera_surface: bad image window / surface");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  CallOrder order(ctx, c.st);   // the render and the surface write: one call
  adn_status s = order.begin("render_camera_surface");
  if (s != ADN_OK || (s = ensure(ctx, ctx->rgba, size_t(rows) * W * 4)) != ADN_OK) return s;
  c.d_rgba8 = ctx->rgba.as<uint8_t>();
  if ((s = render(ctx, c)) != ADN_OK || rows == 0) return s;
  ADN_CUDA(ctx, launch_rgba_to_surface(c.d_rgba8, W, row0, rows, surface, c.st));
  ctx->stats.kernel_launches++;
  return ADN_OK;
}

adn_status adn_render_views_rays(adn_ctx* ctx, int n_views, const float* poses, const float* rots, const float* d_dirs,
                                 int64_t n_per_view, float thr, int K, float* d_rgb, int32_t* d_nsamples,
                                 float* d_oracle_weights, const adn_aux_outputs* aux, void* stream) {
  adn_status s = check_views(ctx, "render_views_rays", n_views, poses, rots, n_per_view);
  if (s != ADN_OK) return s;
  if (!d_dirs) return fail(ctx, ADN_ERR_INVALID, "render_views_rays: d_dirs is null");
  RenderCall c(poses, rots, n_per_view * n_views, thr, K, stream);
  c.n_views = n_views;
  c.n_per_view = n_per_view;
  c.d_dirs = d_dirs;
  c.d_rgb = d_rgb;
  c.d_nsamples = d_nsamples;
  c.d_oracle_w = d_oracle_weights;
  if (aux) c.aux = *aux;
  return render_ordered(ctx, c, "render_views_rays");
}

adn_status adn_render_views_camera(adn_ctx* ctx, int n_views, const float* poses, const float* rots, int W, int H, float thr,
                                   int K, float* d_rgb, int32_t* d_nsamples, void* stream) {
  return render_views_camera(ctx, "render_views_camera", n_views, poses, rots, W, H, thr, K, d_rgb, d_nsamples, nullptr, stream);
}

adn_status adn_render_views_camera_rgba8(adn_ctx* ctx, int n_views, const float* poses, const float* rots, int W, int H,
                                         float thr, int K, uint8_t* d_rgba8, void* stream) {
  return render_views_camera(ctx, "render_views_camera_rgba8", n_views, poses, rots, W, H, thr, K, nullptr, nullptr, d_rgba8,
                             stream);
}

adn_status adn_register_host_buffer(adn_ctx* ctx, const void* p, size_t bytes) {
  if (!ctx || !p || bytes == 0) return fail(ctx, ADN_ERR_INVALID, "register_host_buffer: bad arguments");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  for (const adn_ctx::Reg& r : ctx->regs)
    if (r.p == p) return fail(ctx, ADN_ERR_INVALID, "register_host_buffer: already registered (unregister first)");
  ADN_CUDA(ctx, cudaHostRegister(const_cast<void*>(p), bytes, cudaHostRegisterDefault));
  ctx->regs.push_back({p, bytes});
  return ADN_OK;
}

adn_status adn_unregister_host_buffer(adn_ctx* ctx, const void* p) {
  if (!ctx || !p) return fail(ctx, ADN_ERR_INVALID, "unregister_host_buffer: bad arguments");
  for (size_t i = 0; i < ctx->regs.size(); ++i)
    if (ctx->regs[i].p == p) {
      ADN_CUDA(ctx, cudaSetDevice(ctx->device));
      ADN_CUDA(ctx, cudaDeviceSynchronize());   // no copy of an earlier call may still target the buffer
      ADN_CUDA(ctx, cudaHostUnregister(const_cast<void*>(p)));
      ctx->regs.erase(ctx->regs.begin() + long(i));
      return ADN_OK;
    }
  return fail(ctx, ADN_ERR_INVALID, "unregister_host_buffer: not registered");
}

adn_status adn_net_dims(adn_ctx* ctx, int net_id, int* n_in, int* n_out) {
  if (!ctx || (net_id != 0 && net_id != 1)) return fail(ctx, ADN_ERR_INVALID, "net_dims: bad arguments");
  if (!ctx->net[net_id].ready) return fail(ctx, ADN_ERR_NO_WEIGHTS, "net_dims: network not set");
  if (n_in) *n_in = ctx->net[net_id].n_in;
  if (n_out) *n_out = ctx->net[net_id].n_out;
  return ADN_OK;
}

adn_status adn_net_shape(adn_ctx* ctx, int net_id, int* depth, int* width, int* skip) {
  if (!ctx || (net_id != 0 && net_id != 1)) return fail(ctx, ADN_ERR_INVALID, "net_shape: bad arguments");
  const Net& n = ctx->net[net_id];
  if (!n.ready) return fail(ctx, ADN_ERR_NO_WEIGHTS, "net_shape: network not set");
  if (depth) *depth = n.depth;
  if (width) *width = n.width;
  if (skip) *skip = n.skip;
  return ADN_OK;
}

adn_status adn_render_rays_host(adn_ctx* ctx, const float* pose, const float* rot, const float* h_dirs, int64_t n_rays,
                                float thr, int K, float* h_rgb, int32_t* h_nsamples) {
  if (!ctx || !h_dirs || !h_rgb || n_rays < 0) return fail(ctx, ADN_ERR_INVALID, "render_rays_host: bad arguments");
  if (n_rays == 0 && !joins_group(ctx)) return ADN_OK;
  return render_host(ctx, RenderCall(pose, rot, n_rays, thr, K, nullptr), h_dirs, h_rgb, h_nsamples);
}

adn_status adn_render_camera_host(adn_ctx* ctx, const float* pose, const float* rot, int W, int H, int row0, int rows,
                                  float thr, int K, float* h_rgb, int32_t* h_nsamples) {
  RenderCall c(pose, rot, int64_t(rows) * W, thr, K, nullptr);
  c.cam = camera_rays(ctx, W, H, row0, rows);
  if (!c.cam || !h_rgb) return fail(ctx, ADN_ERR_INVALID, "render_camera_host: bad arguments");
  if (c.n_rays == 0 && !joins_group(ctx)) return ADN_OK;
  return render_host(ctx, c, nullptr, h_rgb, h_nsamples);
}

// ---- stage-level entry points --------------------------------------------------------------------
adn_status adn_generate_ray_directions(adn_ctx* ctx, int W, int H, int row0, int rows, float* d_dirs, void* stream) {
  const std::optional<CameraRays> cam = camera_rays(ctx, W, H, row0, rows);
  if (!cam || !d_dirs) return fail(ctx, ADN_ERR_INVALID, "generate_ray_directions: bad arguments");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  CallOrder order(ctx, static_cast<cudaStream_t>(stream));
  if (adn_status s = order.begin("generate_ray_directions"); s != ADN_OK) return s;
  ADN_CUDA(ctx, launch_gen_dirs(*cam, int64_t(rows) * W, d_dirs, static_cast<cudaStream_t>(stream)));
  ctx->stats.kernel_launches++;
  return ADN_OK;
}

adn_status adn_stage0_features(adn_ctx* ctx, const float* pose, const float* rot, const float* d_dirs, int64_t n_rays,
                               float* d_x0, float* d_ray_o, float* d_ray_d, void* stream) {
  if (!ctx || !pose || !rot || !d_dirs || n_rays < 0 || (d_ray_o == nullptr) != (d_ray_d == nullptr))
    return fail(ctx, ADN_ERR_INVALID, "stage0: bad arguments");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  CallOrder order(ctx, static_cast<cudaStream_t>(stream));
  if (adn_status s = order.begin("stage0"); s != ADN_OK) return s;
  ADN_CUDA(ctx, launch_stage0(ctx->sc, make_pose(pose, rot), d_dirs, nullptr, n_rays, d_x0, d_ray_o, d_ray_d, nullptr, 0,
                              static_cast<cudaStream_t>(stream)));
  ctx->stats.kernel_launches++;
  return ADN_OK;
}

adn_status adn_mlp0_forward(adn_ctx* ctx, const float* d_x0, int64_t n_rays, float* d_raw0, void* stream) {
  if (!ctx || !d_x0 || !d_raw0 || n_rays < 0) return fail(ctx, ADN_ERR_INVALID, "mlp0_forward: bad arguments");
  if (!ctx->net[0].ready) return fail(ctx, ADN_ERR_NO_WEIGHTS, "mlp0_forward: sampling net not set");
  if (n_rays == 0) return ADN_OK;
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CallOrder order(ctx, st);
  adn_status s = order.begin("mlp0_forward");
  Net& n = ctx->net[0];
  if (s != ADN_OK || (s = ensure(ctx, ctx->tiles0, size_t(pad128(n_rays) / 128) * n.prog.in.tile_bytes())) != ADN_OK) return s;
  ADN_CUDA(ctx, launch_pack_rows(d_x0, n_rays, nullptr, n.n_in, n.prog.in, static_cast<uint8_t*>(ctx->tiles0.p), ctx->num_sms, st));
  ctx->stats.kernel_launches++;
  return run_mlp0(ctx, static_cast<uint8_t*>(ctx->tiles0.p), d_raw0, n_rays, st);
}

adn_status adn_stage2_sample(adn_ctx* ctx, const float* d_raw0, int64_t n_rays, float thr, int K, int32_t* d_count,
                             int32_t* d_offset, int32_t* d_cell, int32_t* d_ray, float* d_z, float* d_zp, int64_t* d_total,
                             void* stream) {
  const int D = ctx ? depth_cells(ctx) : 128;
  if (!ctx || !d_total || n_rays < 0 || K < 1 || K > std::min(D, 128) || !(thr > 0.0f) ||
      (n_rays > 0 && (!d_raw0 || !d_count || !d_offset || !d_ray || !d_z || !d_zp)))
    return fail(ctx, ADN_ERR_INVALID, "stage2: bad arguments (adaptive path needs thr > 0 and 1 <= K <= " +
                                          std::to_string(std::min(D, 128)) + ")");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  CallOrder order(ctx, static_cast<cudaStream_t>(stream));
  adn_status s = order.begin("stage2");
  if (s != ADN_OK || (s = ensure(ctx, ctx->s2scratch, stage2_scratch_bytes(n_rays))) != ADN_OK) return s;
  ADN_CUDA(ctx, launch_stage2(d_raw0, n_rays, thr, K, cell_table(ctx, D), d_count, d_offset, d_cell, d_ray, d_z, d_zp,
                              reinterpret_cast<long long*>(d_total), ctx->s2scratch.p, &ctx->s2sync, static_cast<cudaStream_t>(stream),
                              nullptr, D));
  ctx->stats.kernel_launches++;
  return ADN_OK;
}

adn_status adn_pdf_sample(adn_ctx* ctx, const float* d_raw0, int64_t n_rays, int K, int transform, int32_t* d_count,
                          int32_t* d_offset, int32_t* d_ray, float* d_z) {
  if (!ctx || n_rays < 0 || K < 1 || K > 128 || (n_rays > 0 && (!d_raw0 || !d_z)))
    return fail(ctx, ADN_ERR_INVALID, "pdf_sample: bad arguments (need 1 <= K <= 128, d_raw0 and d_z)");
  if (transform != kPdfSigmoid && transform != kPdfSoftmax)
    return fail(ctx, ADN_ERR_INVALID, "pdf_sample: transform must be 1 (sigmoid) or 2 (softmax)");
  if (n_rays * K > INT32_MAX) return fail(ctx, ADN_ERR_INVALID, "pdf_sample: N * K must stay below 2^31 (int32 offsets)");
  if (n_rays == 0) return ADN_OK;
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  const cudaStream_t st = ctx->own_stream;
  {
    CallOrder order(ctx, st);
    if (adn_status s = order.begin("pdf_sample"); s != ADN_OK) return s;
    ADN_CUDA(ctx, launch_pdf_sample(d_raw0, n_rays, K, transform, depth_base(ctx), ctx->scene.depth_range[0], d_count, d_offset,
                                    d_ray, d_z, nullptr, st));
    ctx->stats.kernel_launches++;
  }
  ADN_CUDA(ctx, cudaStreamSynchronize(st));
  return ADN_OK;
}

adn_status adn_camera_rays(adn_ctx* ctx, const float* pose, const float* rot, const float* d_dirs, int64_t n_rays, float* d_ray_o,
                           float* d_ray_d, float* d_ray_dirs) {
  if (!ctx || !pose || !rot || n_rays < 0 || (n_rays > 0 && (!d_dirs || !d_ray_o || !d_ray_d)))
    return fail(ctx, ADN_ERR_INVALID, "camera_rays: bad arguments (need pose, rot, d_dirs, d_ray_o and d_ray_d)");
  if (ctx->scene.use_ndc && d_ray_dirs) {
    if (ctx->scene.ndc_w <= 0 || ctx->scene.ndc_h <= 0)
      return fail(ctx, ADN_ERR_INVALID, "camera_rays: the NDC directions need the scene's ndc_w / ndc_h");
    set_ndc_projection(ctx, ctx->scene.ndc_w, ctx->scene.ndc_h, ctx->scene.ndc_focal);
  }
  if (n_rays == 0) return ADN_OK;
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  const cudaStream_t st = ctx->own_stream;
  {
    CallOrder order(ctx, st);
    if (adn_status s = order.begin("camera_rays"); s != ADN_OK) return s;
    ADN_CUDA(ctx, launch_camera_rays(ctx->sc, make_pose(pose, rot), d_dirs, nullptr, n_rays, d_ray_o, d_ray_d, d_ray_dirs, st));
    ctx->stats.kernel_launches++;
  }
  ADN_CUDA(ctx, cudaStreamSynchronize(st));
  return ADN_OK;
}

adn_status adn_linear_depths(adn_ctx* ctx, int K, float* d_z) {
  if (!ctx || K < 1 || K > 128 || !d_z) return fail(ctx, ADN_ERR_INVALID, "linear_depths: bad arguments (need 1 <= K <= 128 and d_z)");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  const cudaStream_t st = ctx->own_stream;
  {
    CallOrder order(ctx, st);
    if (adn_status s = order.begin("linear_depths"); s != ADN_OK) return s;
    ADN_CUDA(ctx, cudaMemcpyAsync(d_z, zlin_table(ctx, K), size_t(K) * 4, cudaMemcpyDeviceToDevice, st));
  }
  ADN_CUDA(ctx, cudaStreamSynchronize(st));
  return ADN_OK;
}

adn_status adn_sampling_view(adn_ctx* ctx, const float* d_raw0, int64_t n_rays, float* d_rgb, uint8_t* d_rgba8) {
  if (!ctx || n_rays < 0 || (n_rays > 0 && (!d_raw0 || (!d_rgb && !d_rgba8))))
    return fail(ctx, ADN_ERR_INVALID, "sampling_view: bad arguments");
  if (reinterpret_cast<uintptr_t>(d_raw0) & 15u) return fail(ctx, ADN_ERR_INVALID, "sampling_view: d_raw0 must be 16-byte aligned");
  if (n_rays == 0) return ADN_OK;
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  const cudaStream_t st = ctx->own_stream;
  {
    CallOrder order(ctx, st);
    if (adn_status s = order.begin("sampling_view"); s != ADN_OK) return s;
    ADN_CUDA(ctx, launch_sampling_view(d_raw0, n_rays, d_rgb, d_rgba8, st));
    ctx->stats.kernel_launches++;
  }
  ADN_CUDA(ctx, cudaStreamSynchronize(st));
  return ADN_OK;
}

adn_status adn_budget_threshold(adn_ctx* ctx, const float* d_raw0, int64_t n_rays, float thr_min, int K, int64_t max_samples,
                                float* d_thr, void* stream) {
  const int D = ctx ? depth_cells(ctx) : 128;
  if (!ctx || !d_thr || n_rays < 0 || (n_rays > 0 && !d_raw0) || K < 1 || K > std::min(D, 128) || !(thr_min > 0.0f) || max_samples < n_rays)
    return fail(ctx, ADN_ERR_INVALID, "budget_threshold: bad arguments (need thr_min > 0, 1 <= K <= " + std::to_string(std::min(D, 128)) +
                                          ", max_samples >= n_rays)");
  if (n_rays * (K - 1) >= (int64_t(1) << 32))
    return fail(ctx, ADN_ERR_INVALID, "budget_threshold: at most 2^32 - 1 candidate samples (N * (K - 1))");
  if (D == 128 && (reinterpret_cast<uintptr_t>(d_raw0) & 15u)) return fail(ctx, ADN_ERR_INVALID, "budget_threshold: d_raw0 must be 16-byte aligned");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  CallOrder order(ctx, static_cast<cudaStream_t>(stream));
  adn_status s = order.begin("budget_threshold");
  if (s != ADN_OK || (s = ensure(ctx, ctx->budget_keys, size_t(std::max<int64_t>(1, n_rays * (K - 1))) * 4)) != ADN_OK ||
      (s = ensure(ctx, ctx->budget_work, budget_work_bytes())) != ADN_OK)
    return s;
  int launches = 0;
  ADN_CUDA(ctx, launch_budget_threshold(d_raw0, n_rays, thr_min, K, max_samples, static_cast<uint32_t*>(ctx->budget_keys.p),
                                        ctx->budget_work.p, d_thr, ctx->num_sms, static_cast<cudaStream_t>(stream), &launches,
                                        &ctx->group, D));
  ctx->stats.kernel_launches += launches;
  return ctx->group.failed_round >= 0 ? group_fail(ctx, "budget_threshold") : ADN_OK;
}

adn_status adn_stage3_encode(adn_ctx* ctx, const float* d_ray_o, const float* d_ray_d, const int32_t* d_ray, const float* d_z,
                             int64_t n_samples, float* d_x1, void* stream) {
  if (!ctx || !d_ray_o || !d_ray_d || !d_ray || !d_z || !d_x1 || n_samples < 0) return fail(ctx, ADN_ERR_INVALID, "stage3: bad arguments");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  CallOrder order(ctx, static_cast<cudaStream_t>(stream));
  if (adn_status s = order.begin("stage3"); s != ADN_OK) return s;
  ADN_CUDA(ctx, launch_stage3(ctx->sc, d_ray_o, d_ray_d, d_ray, d_z, nullptr, 1, n_samples, nullptr, d_x1, nullptr, ctx->num_sms,
                              static_cast<cudaStream_t>(stream)));
  ctx->stats.kernel_launches++;
  return ADN_OK;
}

adn_status adn_mlp1_forward(adn_ctx* ctx, const float* d_x1, int64_t n_samples, float* d_raw1, void* stream) {
  if (!ctx || !d_x1 || !d_raw1 || n_samples < 0) return fail(ctx, ADN_ERR_INVALID, "mlp1_forward: bad arguments");
  if (!ctx->net[1].ready) return fail(ctx, ADN_ERR_NO_WEIGHTS, "mlp1_forward: shading net not set");
  if (n_samples == 0) return ADN_OK;
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CallOrder order(ctx, st);
  adn_status s = order.begin("mlp1_forward");
  Net& n = ctx->net[1];
  if (s != ADN_OK || (s = ensure(ctx, ctx->tiles1, size_t(pad128(n_samples) / 128) * n.prog.in.tile_bytes())) != ADN_OK) return s;
  ADN_CUDA(ctx, launch_pack_rows(d_x1, n_samples, nullptr, n.n_in, n.prog.in, static_cast<uint8_t*>(ctx->tiles1.p), ctx->num_sms, st));
  ctx->stats.kernel_launches++;
  return run_mlp(ctx, 1, static_cast<uint8_t*>(ctx->tiles1.p), d_raw1, nullptr, n_samples, st);
}

adn_status adn_stage5_composite_aux(adn_ctx* ctx, const float* d_raw1, const float* d_zp, const float* d_z,
                                    const int32_t* d_offset, const int32_t* d_count, int64_t n_rays, int K, int dense,
                                    float* d_rgb, uint8_t* d_rgba8, const adn_aux_outputs* aux, void* stream) {
  const adn_aux_outputs a = aux ? *aux : adn_aux_outputs{};
  const bool reads_z = a.d_z_vals || a.d_depth_map || a.d_disp_map || a.d_depth_est;
  if (!ctx || n_rays < 0 || K < 1 || K > 128 || (dense && K != 128 && K != depth_cells(ctx)))
    return fail(ctx, ADN_ERR_INVALID, "stage5: bad arguments (dense mode needs K == 128 or K == the sampling net's depth cells)");
  if (n_rays > 0 && (!d_raw1 || !d_zp || (!dense && (!d_offset || !d_count || (reads_z && !d_z)))))
    return fail(ctx, ADN_ERR_INVALID, "stage5: bad arguments");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  CallOrder order(ctx, static_cast<cudaStream_t>(stream));
  adn_status s = order.begin("stage5");
  if (s != ADN_OK || (dense && (s = ensure_dense_lut(ctx, K)) != ADN_OK)) return s;
  ADN_CUDA(ctx, launch_stage5(d_raw1, d_zp, dense ? nullptr : d_z, ctx->zlut_dense.as<float>(), dense ? nullptr : d_offset,
                              d_count, n_rays, K, dense, d_rgb, d_rgba8, stage5_aux(ctx, a), static_cast<cudaStream_t>(stream)));
  ctx->stats.kernel_launches++;
  return ADN_OK;
}

adn_status adn_stage5_density_composite(adn_ctx* ctx, const float* d_raw1, const float* d_z, const float* d_ray_d, int64_t n_rays,
                                        int K, float* d_rgb, uint8_t* d_rgba8, const adn_aux_outputs* aux) {
  if (!ctx || n_rays < 0 || K < 1 || K > 128 || (n_rays > 0 && (!d_raw1 || !d_z || !d_ray_d)))
    return fail(ctx, ADN_ERR_INVALID, "stage5_density: bad arguments (need 1 <= K <= 128, d_raw1, d_z and d_ray_d)");
  if (n_rays == 0) return ADN_OK;
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  const cudaStream_t st = ctx->own_stream;
  {
    CallOrder order(ctx, st);
    if (adn_status s = order.begin("stage5_density"); s != ADN_OK) return s;
    ADN_CUDA(ctx, launch_stage5(d_raw1, nullptr, d_z, nullptr, nullptr, nullptr, n_rays, K, 0, d_rgb, d_rgba8,
                                stage5_aux(ctx, aux ? *aux : adn_aux_outputs{}), st, d_ray_d));
    ctx->stats.kernel_launches++;
  }
  ADN_CUDA(ctx, cudaStreamSynchronize(st));
  return ADN_OK;
}

adn_status adn_stage5_composite(adn_ctx* ctx, const float* d_raw1, const float* d_zp, const float* d_z, const int32_t* d_offset,
                                const int32_t* d_count, int64_t n_rays, int K, float* d_rgb, float* d_weights,
                                float* d_depth_map, void* stream) {
  if (!d_rgb) return fail(ctx, ADN_ERR_INVALID, "stage5: bad arguments");
  adn_aux_outputs aux{};
  aux.d_weights = d_weights;
  aux.d_depth_map = d_depth_map;
  return adn_stage5_composite_aux(ctx, d_raw1, d_zp, d_z, d_offset, d_count, n_rays, K, 0, d_rgb, nullptr, &aux, stream);
}

adn_status adn_image_metrics(adn_ctx* ctx, const float* d_image, const float* d_reference, int64_t n_values, int clamp01,
                             double* mse_out, double* psnr_out, void* stream) {
  if (!ctx || !d_image || !d_reference || n_values < 1 || (!mse_out && !psnr_out))
    return fail(ctx, ADN_ERR_INVALID, "image_metrics: bad arguments");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CallOrder order(ctx, st);
  adn_status s = order.begin("image_metrics");
  if (s != ADN_OK || (s = ensure(ctx, ctx->metric, sizeof(double) * (kMetricBlocks + 1))) != ADN_OK) return s;
  double* part = static_cast<double*>(ctx->metric.p);
  ADN_CUDA(ctx, launch_image_sqdiff(d_image, d_reference, n_values, clamp01, part, part + kMetricBlocks, st));
  ctx->stats.kernel_launches += 2;
  double sum = 0.0;
  ADN_CUDA(ctx, cudaMemcpyAsync(&sum, part + kMetricBlocks, sizeof(double), cudaMemcpyDeviceToHost, st));
  ADN_CUDA(ctx, cudaStreamSynchronize(st));
  const double mse = sum / double(n_values);                       // calculate_mse, src/evaluate.py:49-50
  if (mse_out) *mse_out = mse;
  if (psnr_out) *psnr_out = 10.0 * std::log10(1.0 / mse);         // calculate_psnr, src/evaluate.py:53-54
  return ADN_OK;
}

adn_status adn_image_flip(adn_ctx* ctx, const float* d_image, const float* d_reference, int W, int H, double pixels_per_degree,
                          float* d_flip_map, double* mean_out) {
  if (!ctx || !d_image || !d_reference || (!d_flip_map && !mean_out) || W < 1 || H < 1 || int64_t(W) * H > INT32_MAX)
    return fail(ctx, ADN_ERR_INVALID, "image_flip: bad arguments");
  if (!std::isfinite(pixels_per_degree) || !(pixels_per_degree > 0.0) || pixels_per_degree > kFlipMaxPpd)
    return fail(ctx, ADN_ERR_INVALID, "image_flip: need 0 < pixels_per_degree <= " + std::to_string(kFlipMaxPpd));
  FlipConsts c;
  flip_consts(pixels_per_degree, &c);
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  const cudaStream_t st = ctx->own_stream;
  double sum = 0.0;
  {
    CallOrder order(ctx, st);
    adn_status s = order.begin("image_flip");
    if (s != ADN_OK || (s = ensure(ctx, ctx->flip, flip_scratch_bytes(W, H))) != ADN_OK) return s;
    ADN_CUDA(ctx, launch_flip(d_image, d_reference, W, H, c, ctx->flip.p, d_flip_map, st));
    ctx->stats.kernel_launches += 3;
    ADN_CUDA(ctx, cudaMemcpyAsync(&sum, ctx->flip.p, sizeof(double), cudaMemcpyDeviceToHost, st));
  }
  ADN_CUDA(ctx, cudaStreamSynchronize(st));
  if (mean_out) *mean_out = sum / (double(W) * double(H));
  return ADN_OK;
}

adn_status adn_image_iwssim(adn_ctx* ctx, const float* d_image, const float* d_reference, int W, int H, int layout,
                            double* score_out, double* scale_out) {
  if (!ctx || !d_image || !d_reference || !score_out || W < kIwMinSize || H < kIwMinSize || int64_t(W) * H > INT32_MAX)
    return fail(ctx, ADN_ERR_INVALID, "image_iwssim: bad arguments (W, H >= " + std::to_string(kIwMinSize) + ", W * H < 2^31)");
  if (layout != ADN_IWSSIM_GRAY && layout != ADN_IWSSIM_EVALUATE_RGB)
    return fail(ctx, ADN_ERR_INVALID, "image_iwssim: unknown layout " + std::to_string(layout));
  // the metric's image: H rows of W for gray planes; evaluate.py views its [H*W, 3] buffer as [W, H]
  const IwPlan plan = layout == ADN_IWSSIM_GRAY ? iwssim_plan(H, W) : iwssim_plan(W, H);
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  const cudaStream_t st = ctx->own_stream;
  double res[1 + kIwNsc];
  {
    CallOrder order(ctx, st);
    adn_status s = order.begin("image_iwssim");
    if (s != ADN_OK || (s = ensure(ctx, ctx->iwssim, plan.bytes)) != ADN_OK) return s;
    ADN_CUDA(ctx, launch_iwssim(d_image, d_reference, layout == ADN_IWSSIM_GRAY ? kIwGray : kIwEvaluateRgb, plan, ctx->iwssim.p, st));
    ctx->stats.kernel_launches += 10;
    ADN_CUDA(ctx, cudaMemcpyAsync(res, static_cast<char*>(ctx->iwssim.p) + plan.off_out, sizeof(res), cudaMemcpyDeviceToHost, st));
  }
  ADN_CUDA(ctx, cudaStreamSynchronize(st));
  *score_out = res[0];
  if (scale_out)
    for (int k = 0; k < kIwNsc; ++k) scale_out[k] = res[1 + k];
  return ADN_OK;
}

adn_status adn_probe_export_dir(const char* dir, adn_scene* scene_out, float* thr_out, int* k_out, int* n_tensors_out) {
  if (!dir) return ADN_ERR_INVALID;
  adn::ExportDir ex;
  std::string err;
  if (!adn::load_export_dir(dir, ex, err)) {
    std::fprintf(stderr, "adanerf_b200: %s\n", err.c_str());
    return ADN_ERR_IO;
  }
  if (scene_out) *scene_out = ex.scene;
  if (thr_out) *thr_out = ex.threshold;
  if (k_out) *k_out = ex.num_samples;
  if (n_tensors_out) {
    n_tensors_out[0] = int(ex.nets[0].size());
    n_tensors_out[1] = int(ex.nets[1].size());
  }
  return ADN_OK;
}

adn_status adn_create_from_export_dir(adn_ctx** out, const char* dir, int device, float* thr_out, int* k_out) {
  if (!out || !dir) return ADN_ERR_INVALID;
  *out = nullptr;
  adn::ExportDir ex;
  std::string err;
  if (!adn::load_export_dir(dir, ex, err) || !adn::check_depth_cells(ex, err)) {
    std::fprintf(stderr, "adanerf_b200: %s\n", err.c_str());
    return ADN_ERR_IO;
  }
  adn_ctx* ctx = nullptr;
  adn_status s = adn_create(&ctx, &ex.scene, device);
  if (s != ADN_OK) return s;
  for (int id = 0; id < 2; ++id) {
    if (ex.sampler == 2 && id == 0) continue;   // a one-network export: its net is in slot 1
    std::vector<adn_tensor_desc> descs;
    for (auto& t : ex.nets[id]) descs.push_back({t.name.c_str(), t.data.data(), t.rows, t.cols});
    s = adn_set_weights(ctx, id, descs.data(), int(descs.size()));
    if (s != ADN_OK) {
      std::fprintf(stderr, "adanerf_b200: %s\n", ctx->last_error.c_str());
      adn_destroy(ctx);
      return s;
    }
  }
  if ((ex.sampler == 2 && (s = adn_set_option(ctx, "sampler", 2)) != ADN_OK) ||
      (ex.sampler == 1 && ((s = adn_set_option(ctx, "sampler", 1)) != ADN_OK ||
                           (s = adn_set_option(ctx, "pdf_transform", ex.pdf_transform)) != ADN_OK))) {
    std::fprintf(stderr, "adanerf_b200: %s\n", ctx->last_error.c_str());
    adn_destroy(ctx);
    return s;
  }
  if (thr_out) *thr_out = ex.threshold;
  if (k_out) *k_out = ex.num_samples;
  *out = ctx;
  return ADN_OK;
}

}  // extern "C"
