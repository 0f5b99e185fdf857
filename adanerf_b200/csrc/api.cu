// C ABI + host-side context of the H100 AdaNeRF renderer (see include/adanerf_b200.h).
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/adanerf_b200.h"
#include "export_loader.h"
#include "mlp.cuh"
#include "ptx.cuh"
#include "stages.cuh"

using namespace adn;

namespace {

struct HostTensor {
  std::vector<float> data;
  int64_t rows = 0, cols = 0;
};

struct Net {
  bool ready = false;
  int n_in = 0, n_out = 0;
  MlpProgram prog{};
  uint8_t* d_wblob = nullptr;
  std::map<std::string, HostTensor> tensors;  // kept so "mlp0_terms" can re-pack
};

struct Buf {
  void* p = nullptr;
  size_t cap = 0;
};

}  // namespace

struct adn_ctx {
  int device = 0;
  int num_sms = 132;
  adn_scene scene{};
  SceneDev sc{};
  float* d_zlut = nullptr;        // [128] world depth of the cell centres (log warp)
  float* d_zlut_dense = nullptr;  // [dense_K]
  int dense_K = 0;
  Net net[2];
  int mlp0_terms = 3;
  int n_feat0 = 90;               // sampling-net input features: 6 + 6 (n_freq_pos0 + n_freq_dir0)
  bool fuse_encoder = false;      // stage 3 inside the shading kernel: saves the [M, 90]-sized tile buffer
  int64_t chunk_rays = 0;
  bool profile = false;
  int64_t sample_budget = 0;      // B of adn_set_option "sample_budget" (0 = off)
  bool last_budget = false;       // the last render chose its threshold on the device (in budget_thr)
  float last_thr = 0.0f;          // the last render's threshold argument
  bool prof_budget = false;       // the profiled render timed the selection with stage 2 (ev[7] -> ev[3])
  // scratch
  Buf tiles0, raw0, ray_o, ray_d, dirs, count, offset, rayidx, zbuf, zpbuf, tiles1, raw1, s2scratch, rgb, rgba, metric;
  Buf budget_keys, budget_work, budget_thr;   // sample budget: candidate keys, histograms + select state, t*
  long long* d_total = nullptr;
  int* d_err = nullptr;           // device view of h_err
  int* h_err = nullptr;           // watchdog flag in mapped pinned host memory: still readable after a device trap
  // pinned staging for the *_host entry points
  Stage2Sync s2sync;              // epoch / ticket base of s2scratch (no per-launch memset)
  Buf h_in, h_out, h_ns;
  // caller buffers page-locked in place at the caller's explicit request (adn_register_host_buffer): the *_host entry
  // points DMA straight from / to them; everything else goes through the context's pinned staging buffers
  struct Reg { const void* p = nullptr; size_t bytes = 0; };
  std::vector<Reg> regs;
  cudaStream_t own_stream = nullptr;
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
#define ADN_CUDA(ctx, call)                                   \
  do {                                                        \
    cudaError_t e__ = (call);                                 \
    if (e__ != cudaSuccess) return cuda_fail(ctx, e__, #call); \
  } while (0)

adn_status ensure(adn_ctx* ctx, Buf& b, size_t bytes) {
  if (bytes <= b.cap) return ADN_OK;
  if (b.p) ADN_CUDA(ctx, cudaFree(b.p));
  b.p = nullptr;
  b.cap = 0;
  size_t want = bytes + bytes / 8 + 256;
  ADN_CUDA(ctx, cudaMalloc(&b.p, want));
  b.cap = want;
  return ADN_OK;
}
adn_status ensure_pinned(adn_ctx* ctx, Buf& b, size_t bytes) {
  if (bytes <= b.cap) return ADN_OK;
  if (b.p) ADN_CUDA(ctx, cudaFreeHost(b.p));
  b.p = nullptr;
  b.cap = 0;
  ADN_CUDA(ctx, cudaMallocHost(&b.p, bytes));
  b.cap = bytes;
  return ADN_OK;
}

// True when [p, p + bytes) can be the source / target of an asynchronous copy at full speed: inside a range the caller
// registered with adn_register_host_buffer (whose lifetime the caller vouches for), or memory the caller allocated
// page-locked itself (cudaMallocHost / torch pin_memory).  The library never registers memory behind the caller's back:
// a buffer that is freed and re-allocated at the same address would keep a stale registration (ADVICE r1).
bool pin_in_place(adn_ctx* ctx, int /*slot*/, const void* p, size_t bytes) {
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
// 128-row N half, for each K block (Seg): a [128 x 64] K-major SWIZZLE_128B bf16 tile (hi), followed by the lo tile when
// nsplit == 2.
void pack_layer(const float* W, int n_out, int k_in, const std::vector<Seg>& segs, int nsplit, std::vector<uint8_t>& blob) {
  const int n_half = (n_out + 127) / 128;
  for (int nh = 0; nh < n_half; ++nh) {
    for (const Seg& sg : segs) {
      const size_t base = blob.size();
      blob.resize(base + size_t(nsplit) * kBlkBytes, 0);
      for (int n = 0; n < 128; ++n) {
        const int row = nh * 128 + n;
        for (int kk = 0; kk < 64; ++kk) {
          float w = 0.0f;
          if (row < n_out && kk < sg.valid && sg.col0 + kk < k_in) w = W[size_t(row) * k_in + sg.col0 + kk];
          const uint16_t hi = f2bf(w);
          const uint32_t off = sw128_offset(uint32_t(n), uint32_t(kk));
          std::memcpy(&blob[base + off], &hi, 2);
          if (nsplit == 2) {
            const uint16_t lo = f2bf(w - bf2f(hi));
            std::memcpy(&blob[base + kBlkBytes + off], &lo, 2);
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
  if (fblob.size() > size_t(kSideFloats)) return fail(ctx, ADN_ERR_INVALID, "network has too many fp32 side parameters");
  std::memset(net.prog.side, 0, sizeof(net.prog.side));
  std::memcpy(net.prog.side, fblob.data(), fblob.size() * 4);
  if (net.d_wblob) cudaFree(net.d_wblob);
  net.d_wblob = nullptr;
  ADN_CUDA(ctx, cudaMalloc(&net.d_wblob, wblob.size()));
  ADN_CUDA(ctx, cudaMemcpy(net.d_wblob, wblob.data(), wblob.size(), cudaMemcpyHostToDevice));
  return ADN_OK;
}

// Sampling net: BaseNet without skips (src/models.py:71-76,183-195): layers.{i}.weight/bias.
adn_status build_net0(adn_ctx* ctx) {
  Net& net = ctx->net[0];
  int D = 0;
  while (find(net, "layers." + std::to_string(D) + ".weight")) ++D;
  if (D < 1 || D > kMaxLayers) return fail(ctx, ADN_ERR_INVALID, "sampling net: need layers.0.weight .. (1-12 layers)");
  const int nsplit = ctx->mlp0_terms == 3 ? 2 : 1;
  MlpProgram P{};
  P.n_layers = D;
  std::vector<uint8_t> wblob;
  std::vector<float> fblob;
  int prev = -1;
  for (int l = 0; l < D; ++l) {
    const HostTensor* W = find(net, "layers." + std::to_string(l) + ".weight");
    const HostTensor* B = find(net, "layers." + std::to_string(l) + ".bias");
    if (!B || int64_t(B->data.size()) != W->rows) return fail(ctx, ADN_ERR_INVALID, "sampling net: missing/odd bias");
    const int n_out = int(W->rows), k_in = int(W->cols);
    const bool last = (l == D - 1);
    if (l == 0) {
      if (k_in < 1 || k_in > 128) return fail(ctx, ADN_ERR_INVALID, "sampling net: input width must be <= 128");
      net.n_in = k_in;
    } else if (k_in != prev) {
      return fail(ctx, ADN_ERR_INVALID, "sampling net: layer widths do not chain");
    }
    if (!last && n_out != 256) return fail(ctx, ADN_ERR_INVALID, "sampling net: hidden width must be 256");
    if (last && n_out != 128 && n_out != 256) return fail(ctx, ADN_ERR_INVALID, "sampling net: output width must be 128 or 256");
    prev = n_out;
    MlpLayer& L = P.layers[l];
    std::vector<Seg> segs;
    if (l == 0) {
      segs = {{0, std::min(64, k_in)}, {64, std::max(0, k_in - 64)}};
    } else {
      segs = {{0, 64}, {64, 64}, {128, 64}, {192, 64}};
    }
    L.n_kb = uint8_t(segs.size());
    for (size_t i = 0; i < segs.size(); ++i) {
      L.a_blk[i] = uint8_t(i);
      // 16-wide K steps that hold data; block 0 keeps at least one (it initialises the accumulator)
      L.k_cnt[i] = uint8_t(std::max(i == 0 ? 1 : 0, (segs[i].valid + 15) / 16));
    }
    L.n_half = uint8_t(n_out / 128);
    L.flags = last ? uint8_t(LF_FINAL_RAW) : uint8_t(LF_RELU | LF_OUT_ACT);
    L.out_blk0 = 0;
    L.w_off = uint32_t(wblob.size());
    pack_layer(W->data.data(), n_out, k_in, segs, nsplit, wblob);
    L.bias_off = uint32_t(push_floats(fblob, B->data.data(), B->data.size()));
    if (last) {
      net.n_out = n_out;
      P.out_cols = n_out;
    }
  }
  P.in = sampling_tiles(net.n_in, nsplit);
  P.in_nblk0 = P.in.n_blk;
  net.prog = P;
  adn_status s = upload(ctx, net, wblob, fblob);
  if (s != ADN_OK) return s;
  net.ready = true;
  return ADN_OK;
}

// Shading net: NeRF(D=8, W=256, skips=[4], use_viewdirs=True) (src/models.py:199-277).
adn_status build_net1(adn_ctx* ctx) {
  Net& net = ctx->net[1];
  auto need = [&](const std::string& n, int64_t r, int64_t c) -> const HostTensor* {
    const HostTensor* t = find(net, n);
    if (!t || t->rows != r || t->cols != c) return nullptr;
    return t;
  };
  const HostTensor *pw[8], *pb[8];
  for (int i = 0; i < 8; ++i) {
    const int64_t k = (i == 0) ? 63 : (i == 5 ? 319 : 256);
    pw[i] = need("pts_linears." + std::to_string(i) + ".weight", 256, k);
    pb[i] = find(net, "pts_linears." + std::to_string(i) + ".bias");
    if (!pw[i] || !pb[i] || pb[i]->data.size() != 256)
      return fail(ctx, ADN_ERR_INVALID, "shading net: pts_linears." + std::to_string(i) + " has the wrong shape (expect NeRF 8x256, skip 4, posEnc 10-4)");
  }
  const HostTensor* fw = need("feature_linear.weight", 256, 256);
  const HostTensor* fb = find(net, "feature_linear.bias");
  const HostTensor* aw = need("alpha_linear.weight", 1, 256);
  const HostTensor* ab = find(net, "alpha_linear.bias");
  const HostTensor* vw = need("views_linears.0.weight", 128, 283);
  const HostTensor* vb = find(net, "views_linears.0.bias");
  const HostTensor* rw = need("rgb_linear.weight", 3, 128);
  const HostTensor* rb = find(net, "rgb_linear.bias");
  if (!fw || !fb || !aw || !ab || !vw || !vb || !rw || !rb || fb->data.size() != 256 || ab->data.size() != 1 ||
      vb->data.size() != 128 || rb->data.size() != 3)
    return fail(ctx, ADN_ERR_INVALID, "shading net: feature/alpha/views/rgb tensors missing or wrong shape");
  net.n_in = 90;
  net.n_out = 4;
  MlpProgram P{};
  P.n_layers = 10;
  std::vector<uint8_t> wblob;
  std::vector<float> fblob;
  const std::vector<Seg> segH = {{0, 64}, {64, 64}, {128, 64}, {192, 64}};
  for (int l = 0; l < 10; ++l) {
    MlpLayer& L = P.layers[l];
    std::vector<Seg> segs;
    const HostTensor *W, *B;
    L.out_blk0 = 1;
    L.n_half = 2;
    if (l == 0) {
      segs = {{0, 63}};
      L.a_blk[0] = 0;
      L.flags = LF_RELU | LF_OUT_ACT;
      W = pw[0];
      B = pb[0];
    } else if (l == 5) {
      segs = {{0, 63}, {63, 64}, {127, 64}, {191, 64}, {255, 64}};   // cat[pts, h] (models.py:260-261)
      const uint8_t blk[5] = {0, 1, 2, 3, 4};
      std::memcpy(L.a_blk, blk, 5);
      L.flags = LF_RELU | LF_OUT_ACT | LF_LOAD_IN1_AFTER;
      W = pw[5];
      B = pb[5];
    } else if (l <= 7) {
      segs = segH;
      const uint8_t blk[5] = {1, 2, 3, 4, 0};
      std::memcpy(L.a_blk, blk, 5);
      L.flags = LF_RELU | LF_OUT_ACT | (l == 7 ? LF_ALPHA_DOT : 0);
      W = pw[l];
      B = pb[l];
    } else if (l == 8) {  // feature_linear: no activation (models.py:265)
      segs = segH;
      const uint8_t blk[5] = {1, 2, 3, 4, 0};
      std::memcpy(L.a_blk, blk, 5);
      L.flags = LF_OUT_ACT;
      W = fw;
      B = fb;
    } else {  // views_linears.0 on cat[feature, views] (models.py:266-269) + rgb_linear in the epilogue
      segs = {{0, 64}, {64, 64}, {128, 64}, {192, 64}, {256, 27}};
      const uint8_t blk[5] = {1, 2, 3, 4, 0};
      std::memcpy(L.a_blk, blk, 5);
      L.flags = LF_RELU | LF_FINAL_RGB | LF_WAIT_IN;
      L.n_half = 1;
      W = vw;
      B = vb;
    }
    L.n_kb = uint8_t(segs.size());
    for (size_t i = 0; i < segs.size(); ++i) L.k_cnt[i] = uint8_t((segs[i].valid + 15) / 16);
    L.w_off = uint32_t(wblob.size());
    pack_layer(W->data.data(), int(W->rows), int(W->cols), segs, 1, wblob);
    L.bias_off = uint32_t(push_floats(fblob, B->data.data(), B->data.size()));
  }
  P.alpha_w_off = uint32_t(push_floats(fblob, aw->data.data(), 256));
  P.alpha_b_off = uint32_t(push_floats(fblob, ab->data.data(), 1));
  P.rgb_w_off = uint32_t(push_floats(fblob, rw->data.data(), 3 * 128));
  P.rgb_b_off = uint32_t(push_floats(fblob, rb->data.data(), 3));
  P.in = shading_tiles();
  P.in_nblk0 = 1;   // P; V after layer 5
  P.out_cols = 4;
  net.prog = P;
  adn_status s = upload(ctx, net, wblob, fblob);
  if (s != ADN_OK) return s;
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

adn_status ensure_dense_lut(adn_ctx* ctx, int K) {
  if (ctx->dense_K == K && ctx->d_zlut_dense) return ADN_OK;
  // thr == 0 branch of FromClassifiedDepthAdaptive.generate (nerf_raymarch_common.py:708-720), fp32 steps
  std::vector<float> lut(K);
  const double max_v = double(ctx->scene.depth_range[1]) - double(ctx->scene.depth_range[0]);
  for (int k = 0; k < K; ++k) {
    // torch.linspace(0,1,K+1)[k] + 0.5/K in fp32
    const float step = 1.0f / float(K);
    const float lin = (k < (K + 1) / 2) ? float(k) * step : 1.0f - float(K - k) * step;  // ATen linspace is symmetric
    const float t = lin + float(0.5 / K);
    const float z = ctx->scene.z_near * (1.0f - t) + ctx->scene.z_far * t;
    const float w = float(std::pow(max_v + 1.0, double(z)));
    lut[k] = ctx->scene.use_ndc ? z : (w - 1.0f) + ctx->scene.depth_range[0];   // NoDepthRange: :797-805
  }
  if (ctx->d_zlut_dense) cudaFree(ctx->d_zlut_dense);
  ctx->d_zlut_dense = nullptr;
  ADN_CUDA(ctx, cudaMalloc(&ctx->d_zlut_dense, sizeof(float) * K));
  ADN_CUDA(ctx, cudaMemcpy(ctx->d_zlut_dense, lut.data(), sizeof(float) * K, cudaMemcpyHostToDevice));
  ctx->dense_K = K;
  return ADN_OK;
}

PoseDev make_pose(const float* pose, const float* rot) {
  PoseDev p;
  std::memcpy(p.pose, pose, 12);
  std::memcpy(p.rot, rot, 36);
  return p;
}

CameraRays make_camera(const adn_ctx* ctx, int W, int H, int row0) {
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

adn_status run_mlp(adn_ctx* ctx, int id, const uint8_t* tiles, float* out, const long long* rows_dev, long long rows,
                   cudaStream_t st, const EncodeParams* enc = nullptr) {
  Net& n = ctx->net[id];
  const cudaError_t e = launch_mlp(n.prog, n.d_wblob, tiles, out, rows_dev, rows, ctx->d_err, ctx->num_sms, st, enc);
  if (e != cudaSuccess) return cuda_fail(ctx, e, id == 0 ? "launch sampling MLP" : "launch shading MLP");
  ctx->stats.kernel_launches++;
  return ADN_OK;
}

enum { kStages01 = 1, kStages25 = 2 };

// The hot path for one chunk of rays, stream ordered, no host synchronisation.  `parts`: kStages01 = stage 0 + sampling MLP
// (writes the chunk's raw0 / ray_o / ray_d), kStages25 = stages 2-5 (reads them).  d_thr: stage 2's threshold as a device
// float (sample budget), null = `thr`.
adn_status render_chunk(adn_ctx* ctx, const PoseDev& pd, const float* d_dirs, const CameraRays* cam, int64_t n, float thr,
                        int K, float* d_rgb, uint8_t* d_rgba8, int32_t* d_nsamples, float* raw0, float* ray_o, float* ray_d,
                        const float* d_thr, const Stage5Aux& aux, cudaStream_t st, bool timing, int parts) {
  const bool dense = (thr == 0.0f);
  const int64_t cap = n * K;
  adn_status s;
  Net& n0 = ctx->net[0];
  if (parts & kStages01) {
    if ((s = ensure(ctx, ctx->tiles0, size_t(pad128(n) / 128) * n0.prog.in.tile_bytes())) != ADN_OK) return s;
    uint8_t* tiles0 = static_cast<uint8_t*>(ctx->tiles0.p);
    if (timing) cudaEventRecord(ctx->ev[0], st);
    // stage 0 (writes the sampling net's packed input tiles)
    ADN_CUDA(ctx, launch_stage0(ctx->sc, pd, d_dirs, cam, n, nullptr, ray_o, ray_d, tiles0, n0.prog.in.n_terms, st));
    ctx->stats.kernel_launches++;
    if (timing) cudaEventRecord(ctx->ev[1], st);
    // stage 1
    if ((s = run_mlp(ctx, 0, tiles0, raw0, nullptr, n, st)) != ADN_OK) return s;
    if (timing) cudaEventRecord(ctx->ev[2], st);
  }
  if (!(parts & kStages25)) return ADN_OK;
  if ((s = ensure(ctx, ctx->count, size_t(n) * 4)) != ADN_OK) return s;
  if ((s = ensure(ctx, ctx->offset, size_t(n) * 4)) != ADN_OK) return s;
  if (!dense) {
    if ((s = ensure(ctx, ctx->rayidx, size_t(cap) * 4)) != ADN_OK) return s;
    if ((s = ensure(ctx, ctx->zbuf, size_t(cap) * 4)) != ADN_OK) return s;
    if ((s = ensure(ctx, ctx->zpbuf, size_t(cap) * 4)) != ADN_OK) return s;
    if ((s = ensure(ctx, ctx->s2scratch, stage2_scratch_bytes(n))) != ADN_OK) return s;
  }
  // stage 3 runs inside the shading kernel (encoder warp) unless the variant needs the stand-alone kernel
  const bool fused_enc = ctx->fuse_encoder && !ctx->scene.use_ndc;
  if (!fused_enc && (s = ensure(ctx, ctx->tiles1, size_t(pad128(cap) / 128) * ctx->net[1].prog.in.tile_bytes())) != ADN_OK) return s;
  if ((s = ensure(ctx, ctx->raw1, size_t(pad128(cap)) * 16)) != ADN_OK) return s;

  int32_t* count = d_nsamples ? d_nsamples : static_cast<int32_t*>(ctx->count.p);
  int32_t* offset = static_cast<int32_t*>(ctx->offset.p);
  uint8_t* tiles1 = static_cast<uint8_t*>(ctx->tiles1.p);   // null / stale when the encoder is fused
  float* raw1 = static_cast<float*>(ctx->raw1.p);

  // stage 2
  if (dense) {
    ADN_CUDA(ctx, launch_stage2_dense(n, K, count, offset, ctx->d_total, st));
  } else {
    ADN_CUDA(ctx, launch_stage2(raw0, n, thr, K, ctx->d_zlut, count, offset, nullptr, static_cast<int32_t*>(ctx->rayidx.p),
                                static_cast<float*>(ctx->zbuf.p), static_cast<float*>(ctx->zpbuf.p), ctx->d_total,
                                ctx->s2scratch.p, &ctx->s2sync, st, d_thr));
  }
  ctx->stats.kernel_launches++;
  if (timing) cudaEventRecord(ctx->ev[3], st);
  // stage 3 (+ 4)
  EncodeParams ep;
  if (fused_enc) {
    ep.ray_o = ray_o;
    ep.ray_d = ray_d;
    ep.ray_idx = dense ? nullptr : static_cast<int32_t*>(ctx->rayidx.p);
    ep.z = static_cast<float*>(ctx->zbuf.p);
    ep.zlut_dense = ctx->d_zlut_dense;
    ep.K = K;
    ep.sc = ctx->sc;
  } else {
    ADN_CUDA(ctx, launch_stage3(ctx->sc, ray_o, ray_d, dense ? nullptr : static_cast<int32_t*>(ctx->rayidx.p),
                                static_cast<float*>(ctx->zbuf.p), ctx->d_zlut_dense, K, cap, ctx->d_total, nullptr, tiles1, st));
    ctx->stats.kernel_launches++;
  }
  if (timing) cudaEventRecord(ctx->ev[4], st);
  // stage 4
  if ((s = run_mlp(ctx, 1, fused_enc ? nullptr : tiles1, raw1, ctx->d_total, cap, st, fused_enc ? &ep : nullptr)) != ADN_OK) return s;
  if (timing) cudaEventRecord(ctx->ev[5], st);
  // stage 5
  ADN_CUDA(ctx, launch_stage5(raw1, dense ? raw0 : static_cast<float*>(ctx->zpbuf.p), static_cast<float*>(ctx->zbuf.p),
                              ctx->d_zlut_dense, offset, count, n, K, dense ? 1 : 0, d_rgb, d_rgba8, aux, st));
  ctx->stats.kernel_launches++;
  if (timing) cudaEventRecord(ctx->ev[6], st);
  return ADN_OK;
}

adn_status render_impl(adn_ctx* ctx, const float* pose, const float* rot, const float* d_dirs, const CameraRays* cam,
                       int64_t n_rays, float thr, int K, float* d_rgb, uint8_t* d_rgba8, int32_t* d_nsamples,
                       float* d_oracle_w, cudaStream_t st, const adn_aux_outputs* ax = nullptr) {
  if (!ctx || !pose || !rot || n_rays < 0 || (!d_rgb && !d_rgba8)) return fail(ctx, ADN_ERR_INVALID, "render: bad arguments");
  if (!ctx->net[0].ready || !ctx->net[1].ready) return fail(ctx, ADN_ERR_NO_WEIGHTS, "render: set both networks first");
  if (ctx->net[0].n_in != ctx->n_feat0 || ctx->net[0].n_out != 128)
    return fail(ctx, ADN_ERR_INVALID, "render: sampling net must be " + std::to_string(ctx->n_feat0) + " -> 128 for this scene's encoding");
  if (K < 1 || K > 128 || thr < 0.0f) return fail(ctx, ADN_ERR_INVALID, "render: need 1 <= K <= 128 and thr >= 0");
  if (thr == 0.0f && K != 128) return fail(ctx, ADN_ERR_INVALID, "render: dense mode (thr == 0) needs K == 128 (one sample per depth cell)");
  const int64_t budget = ctx->sample_budget;
  if (budget > 0 && thr == 0.0f)
    return fail(ctx, ADN_ERR_INVALID, "render: sample_budget needs the adaptive path (thr > 0 is the floor threshold), not dense mode");
  if (budget > 0 && budget < n_rays)
    return fail(ctx, ADN_ERR_INVALID, "render: sample_budget " + std::to_string(budget) + " is below the " + std::to_string(n_rays) +
                                          " rays of the call (every ray keeps at least one sample)");
  if (budget > 0 && n_rays * (K - 1) >= (int64_t(1) << 32))
    return fail(ctx, ADN_ERR_INVALID, "render: sample_budget supports at most 2^32 - 1 candidate samples (N * (K - 1)) per call");
  if (budget > 0 && (reinterpret_cast<uintptr_t>(d_oracle_w) & 15u))
    return fail(ctx, ADN_ERR_INVALID, "render: sample_budget needs 16-byte aligned d_oracle_weights rows");
  if (n_rays == 0) return ADN_OK;
  if (ctx->scene.use_ndc) {
    // image size behind ndc_rays: the frame being rendered (viewer, featureset.cpp:83-84) or the dataset's (features.py:350-351,430)
    if (cam) set_ndc_projection(ctx, cam->W, cam->H, 0.0f);
    else if (ctx->scene.ndc_w > 0 && ctx->scene.ndc_h > 0) set_ndc_projection(ctx, ctx->scene.ndc_w, ctx->scene.ndc_h, ctx->scene.ndc_focal);
    else return fail(ctx, ADN_ERR_INVALID, "render: NDC scene needs ndc_w / ndc_h when rays are passed explicitly");
  }
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  adn_status s;
  if (thr == 0.0f && (s = ensure_dense_lut(ctx, K)) != ADN_OK) return s;
  int64_t chunk = ctx->chunk_rays;
  if (chunk <= 0) {
    chunk = (int64_t(8) << 20) / K;     // ~8 Mi samples of scratch per chunk
    if (chunk < 8192) chunk = 8192;
  }
  chunk = pad128(chunk);
  if (cam && chunk % cam->W) chunk = (chunk / cam->W + 1) * cam->W;  // whole rows per chunk
  const PoseDev pd = make_pose(pose, rot);
  ctx->stats.n_rays = n_rays;
  ctx->last_budget = budget > 0;
  ctx->last_thr = thr;
  if (ctx->profile) ctx->prof_budget = budget > 0;
  // raw0 / ray_o / ray_d: one chunk's worth, or with a sample budget the whole call's (the threshold is chosen over all of
  // raw0 before any chunk runs stage 2)
  const int64_t span = budget > 0 ? n_rays : std::min(chunk, n_rays);
  if (!d_oracle_w && (s = ensure(ctx, ctx->raw0, size_t(span) * 128 * 4)) != ADN_OK) return s;
  if ((s = ensure(ctx, ctx->ray_o, size_t(span) * 12)) != ADN_OK) return s;
  if ((s = ensure(ctx, ctx->ray_d, size_t(span) * 12)) != ADN_OK) return s;
  float* raw0 = d_oracle_w ? d_oracle_w : static_cast<float*>(ctx->raw0.p);
  float* ray_o = static_cast<float*>(ctx->ray_o.p);
  float* ray_d = static_cast<float*>(ctx->ray_d.p);
  auto run = [&](int64_t r0, int parts, const float* d_thr) -> adn_status {
    const int64_t n = std::min(chunk, n_rays - r0);
    const int64_t w = budget > 0 ? r0 : 0;   // window of raw0 / ray_o / ray_d
    CameraRays c{};
    if (cam) {
      c = *cam;
      c.row0 = cam->row0 + int(r0 / cam->W);
    }
    Stage5Aux aux;
    if (ax) {   // this chunk's window of the caller's per-ray / per-slot buffers
      aux.weights = ax->d_weights ? ax->d_weights + r0 * K : nullptr;
      aux.alpha = ax->d_alpha ? ax->d_alpha + r0 * K : nullptr;
      aux.z_vals = ax->d_z_vals ? ax->d_z_vals + r0 * K : nullptr;
      aux.depth_map = ax->d_depth_map ? ax->d_depth_map + r0 : nullptr;
      aux.acc_map = ax->d_acc_map ? ax->d_acc_map + r0 : nullptr;
      aux.disp_map = ax->d_disp_map ? ax->d_disp_map + r0 : nullptr;
      aux.depth_est = ax->d_depth_est ? ax->d_depth_est + r0 : nullptr;
      aux.linear_depth = ctx->scene.use_ndc ? 1 : 0;
      aux.dr_min = ctx->scene.depth_range[0];
      aux.log_range = float(std::log(double(ctx->scene.depth_range[1]) - double(ctx->scene.depth_range[0]) + 1.0));
    }
    return render_chunk(ctx, pd, d_dirs ? d_dirs + 3 * r0 : nullptr, cam ? &c : nullptr, n, thr, K, d_rgb ? d_rgb + 3 * r0 : nullptr,
                        d_rgba8 ? d_rgba8 + 4 * r0 : nullptr, d_nsamples ? d_nsamples + r0 : nullptr,
                        d_oracle_w ? d_oracle_w + 128 * r0 : raw0 + 128 * w, ray_o + 3 * w, ray_d + 3 * w, d_thr, aux, st,
                        ctx->profile && r0 == 0, parts);
  };
  if (budget == 0) {
    for (int64_t r0 = 0; r0 < n_rays; r0 += chunk)
      if ((s = run(r0, kStages01 | kStages25, nullptr)) != ADN_OK) return s;
    return ADN_OK;
  }
  // sample budget: stages 0-1 of every chunk, one threshold for the call, stages 2-5 of every chunk
  if ((s = ensure(ctx, ctx->budget_keys, size_t(std::max<int64_t>(1, n_rays * (K - 1))) * 4)) != ADN_OK) return s;
  if ((s = ensure(ctx, ctx->budget_work, budget_work_bytes())) != ADN_OK) return s;
  if ((s = ensure(ctx, ctx->budget_thr, sizeof(float))) != ADN_OK) return s;
  float* d_thr = static_cast<float*>(ctx->budget_thr.p);
  for (int64_t r0 = 0; r0 < n_rays; r0 += chunk)
    if ((s = run(r0, kStages01, nullptr)) != ADN_OK) return s;
  if (ctx->profile) cudaEventRecord(ctx->ev[7], st);   // the selection is timed with stage 2 of the first chunk
  int launches = 0;
  ADN_CUDA(ctx, launch_budget_threshold(raw0, n_rays, thr, K, budget, static_cast<uint32_t*>(ctx->budget_keys.p), ctx->budget_work.p,
                                        d_thr, ctx->num_sms, st, &launches));
  ctx->stats.kernel_launches += launches;
  for (int64_t r0 = 0; r0 < n_rays; r0 += chunk)
    if ((s = run(r0, kStages25, d_thr)) != ADN_OK) return s;
  return ADN_OK;
}

adn_status check_device_error(adn_ctx* ctx) {
  int err = 0;
  cudaError_t e = cudaDeviceSynchronize();
  err = *reinterpret_cast<volatile int*>(ctx->h_err);
  if (e != cudaSuccess && !err) return cuda_fail(ctx, e, "device synchronize");
  if (err) return fail(ctx, ADN_ERR_KERNEL, "device watchdog: mbarrier wait timed out at site " + std::to_string(err & 0xfff));
  return ADN_OK;
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
  if (scene->n_freq_pos != 10 || scene->n_freq_dir != 4) return ADN_ERR_INVALID;  // posEncArgs[1] "10-4" (F = 90)
  const int nfp0 = scene->n_freq_pos0 ? scene->n_freq_pos0 : scene->n_freq_pos;
  const int nfd0 = scene->n_freq_dir0 ? scene->n_freq_dir0 : scene->n_freq_dir;
  if (!((nfp0 == 10 && nfd0 == 4) || (nfp0 == 2 && nfd0 == 2))) return ADN_ERR_INVALID;   // posEncArgs[0] "10-4" or "2-2"
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
  ctx->sc.n_freq_pos = scene->n_freq_pos;
  ctx->sc.n_freq_dir = scene->n_freq_dir;
  ctx->sc.n_freq_pos0 = nfp0;
  ctx->sc.n_freq_dir0 = nfd0;
  ctx->n_feat0 = 6 + 6 * (nfp0 + nfd0);
  ctx->sc.ndc = scene->use_ndc ? 1 : 0;
  if (scene->use_ndc && scene->ndc_w > 0 && scene->ndc_h > 0) set_ndc_projection(ctx, scene->ndc_w, scene->ndc_h, scene->ndc_focal);
  // z LUT: LogTransform.to_world((cell + .5)/128) (depth_transformations.py:37-48), pow in double, rest in fp32
  float lut[128];
  const double max_v = double(scene->depth_range[1]) - double(scene->depth_range[0]);
  for (int i = 0; i < 128; ++i) {
    const float z = (float(i) + 0.5f) * (1.0f / 128.0f);
    const float w = float(std::pow(max_v + 1.0, double(z)));
    // FromClassifiedDepthAdaptiveNoDepthRange (NDC configs): the cell centre itself (nerf_raymarch_common.py:826-833)
    lut[i] = scene->use_ndc ? z : (w - 1.0f) + scene->depth_range[0];
  }
  bool ok = cudaMalloc(&ctx->d_zlut, sizeof(lut)) == cudaSuccess &&
            cudaMemcpy(ctx->d_zlut, lut, sizeof(lut), cudaMemcpyHostToDevice) == cudaSuccess &&
            cudaMalloc(&ctx->d_total, sizeof(long long)) == cudaSuccess &&
            cudaMemset(ctx->d_total, 0, sizeof(long long)) == cudaSuccess &&
            cudaHostAlloc(&ctx->h_err, sizeof(int), cudaHostAllocMapped) == cudaSuccess &&
            cudaHostGetDevicePointer(&ctx->d_err, ctx->h_err, 0) == cudaSuccess && (*ctx->h_err = 0, true) &&
            cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking) == cudaSuccess;
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
  Buf* bufs[] = {&ctx->tiles0, &ctx->raw0,  &ctx->ray_o,  &ctx->ray_d, &ctx->dirs,      &ctx->count, &ctx->offset,
                 &ctx->rayidx, &ctx->zbuf,  &ctx->zpbuf,  &ctx->tiles1, &ctx->raw1,  &ctx->s2scratch, &ctx->rgb,   &ctx->rgba, &ctx->metric,
                 &ctx->budget_keys, &ctx->budget_work, &ctx->budget_thr};
  for (Buf* b : bufs)
    if (b->p) cudaFree(b->p);
  for (auto& r : ctx->regs)
    if (r.p) cudaHostUnregister(const_cast<void*>(r.p));
  Buf* pinned[] = {&ctx->h_in, &ctx->h_out, &ctx->h_ns};
  for (Buf* b : pinned)
    if (b->p) cudaFreeHost(b->p);
  for (int i = 0; i < 2; ++i) {
    if (ctx->net[i].d_wblob) cudaFree(ctx->net[i].d_wblob);
  }
  if (ctx->d_zlut) cudaFree(ctx->d_zlut);
  if (ctx->d_zlut_dense) cudaFree(ctx->d_zlut_dense);
  if (ctx->d_total) cudaFree(ctx->d_total);
  if (ctx->h_err) cudaFreeHost(ctx->h_err);
  for (int i = 0; i < 8; ++i)
    if (ctx->ev[i]) cudaEventDestroy(ctx->ev[i]);
  if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
  delete ctx;
}

adn_status adn_set_weights(adn_ctx* ctx, int net_id, const adn_tensor_desc* tensors, int n_tensors) {
  if (!ctx || (net_id != 0 && net_id != 1) || !tensors || n_tensors < 1) return fail(ctx, ADN_ERR_INVALID, "set_weights: bad arguments");
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
  if (n == "fuse_encoder") {   // 1: positional encoding inside the shading kernel (no tile buffer); 0 (default): stage3_kernel + packed tiles
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

adn_status adn_get_stats(adn_ctx* ctx, adn_stats* out) {
  if (!ctx || !out) return ADN_ERR_INVALID;
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  adn_status s = check_device_error(ctx);   // synchronises; reports a tripped device watchdog with its site
  if (s != ADN_OK) return s;
  long long total = 0;
  ADN_CUDA(ctx, cudaMemcpy(&total, ctx->d_total, sizeof(total), cudaMemcpyDeviceToHost));
  ctx->stats.n_samples = total;
  if (ctx->profile) {
    for (int i = 0; i < 6; ++i) {
      float ms = 0;
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
  if (ctx && n_rays == 0) return ADN_OK;   // empty batch: nothing to read or write
  if (!d_dirs) return fail(ctx, ADN_ERR_INVALID, "render_rays: d_dirs is null");
  return render_impl(ctx, pose, rot, d_dirs, nullptr, n_rays, thr, K, d_rgb, nullptr, d_nsamples, d_oracle_weights,
                     static_cast<cudaStream_t>(stream));
}

adn_status adn_render_rays_aux(adn_ctx* ctx, const float* pose, const float* rot, const float* d_dirs, int64_t n_rays, float thr,
                               int K, float* d_rgb, int32_t* d_nsamples, float* d_oracle_weights, const adn_aux_outputs* aux,
                               void* stream) {
  if (ctx && n_rays == 0) return ADN_OK;
  if (!d_dirs) return fail(ctx, ADN_ERR_INVALID, "render_rays_aux: d_dirs is null");
  return render_impl(ctx, pose, rot, d_dirs, nullptr, n_rays, thr, K, d_rgb, nullptr, d_nsamples, d_oracle_weights,
                     static_cast<cudaStream_t>(stream), aux);
}

adn_status adn_render_camera(adn_ctx* ctx, const float* pose, const float* rot, int W, int H, int row0, int rows, float thr,
                             int K, float* d_rgb, int32_t* d_nsamples, void* stream) {
  if (!ctx || W < 1 || H < 1 || row0 < 0 || rows < 0 || row0 + rows > H) return fail(ctx, ADN_ERR_INVALID, "render_camera: bad image window");
  const CameraRays cam = make_camera(ctx, W, H, row0);
  return render_impl(ctx, pose, rot, nullptr, &cam, int64_t(rows) * W, thr, K, d_rgb, nullptr, d_nsamples, nullptr,
                     static_cast<cudaStream_t>(stream));
}

adn_status adn_render_camera_rgba8(adn_ctx* ctx, const float* pose, const float* rot, int W, int H, int row0, int rows,
                                   float thr, int K, uint8_t* d_rgba8, void* stream) {
  if (!ctx || W < 1 || H < 1 || row0 < 0 || rows < 0 || row0 + rows > H) return fail(ctx, ADN_ERR_INVALID, "render_camera: bad image window");
  const CameraRays cam = make_camera(ctx, W, H, row0);
  return render_impl(ctx, pose, rot, nullptr, &cam, int64_t(rows) * W, thr, K, nullptr, d_rgba8, nullptr, nullptr,
                     static_cast<cudaStream_t>(stream));
}

adn_status adn_render_camera_surface(adn_ctx* ctx, const float* pose, const float* rot, int W, int H, int row0, int rows,
                                     float thr, int K, unsigned long long surface, void* stream) {
  if (!ctx || W < 1 || H < 1 || row0 < 0 || rows < 0 || row0 + rows > H || !surface)
    return fail(ctx, ADN_ERR_INVALID, "render_camera_surface: bad image window / surface");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  adn_status s = ensure(ctx, ctx->rgba, size_t(rows) * W * 4);
  if (s != ADN_OK) return s;
  uint8_t* px = static_cast<uint8_t*>(ctx->rgba.p);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  s = adn_render_camera_rgba8(ctx, pose, rot, W, H, row0, rows, thr, K, px, stream);
  if (s != ADN_OK) return s;
  ADN_CUDA(ctx, launch_rgba_to_surface(px, W, row0, rows, surface, st));
  ctx->stats.kernel_launches++;
  return ADN_OK;
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

adn_status adn_render_rays_host(adn_ctx* ctx, const float* pose, const float* rot, const float* h_dirs, int64_t n_rays,
                                float thr, int K, float* h_rgb, int32_t* h_nsamples) {
  if (!ctx || !h_dirs || !h_rgb || n_rays < 0) return fail(ctx, ADN_ERR_INVALID, "render_rays_host: bad arguments");
  if (n_rays == 0) return ADN_OK;
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  adn_status s;
  if ((s = ensure(ctx, ctx->dirs, size_t(n_rays) * 12)) != ADN_OK) return s;
  if ((s = ensure(ctx, ctx->rgb, size_t(n_rays) * 12)) != ADN_OK) return s;
  if ((s = ensure(ctx, ctx->count, size_t(n_rays) * 4)) != ADN_OK) return s;
  if ((s = ensure_pinned(ctx, ctx->h_in, size_t(n_rays) * 12)) != ADN_OK) return s;
  if ((s = ensure_pinned(ctx, ctx->h_out, size_t(n_rays) * 12)) != ADN_OK) return s;
  if (h_nsamples && (s = ensure_pinned(ctx, ctx->h_ns, size_t(n_rays) * 4)) != ADN_OK) return s;
  cudaStream_t st = ctx->own_stream;
  const bool in_pinned = pin_in_place(ctx, 0, h_dirs, size_t(n_rays) * 12);
  const bool out_pinned = pin_in_place(ctx, 1, h_rgb, size_t(n_rays) * 12);
  const bool ns_pinned = h_nsamples && pin_in_place(ctx, 2, h_nsamples, size_t(n_rays) * 4);
  const void* src = h_dirs;
  if (!in_pinned) {
    std::memcpy(ctx->h_in.p, h_dirs, size_t(n_rays) * 12);
    src = ctx->h_in.p;
  }
  ADN_CUDA(ctx, cudaMemcpyAsync(ctx->dirs.p, src, size_t(n_rays) * 12, cudaMemcpyHostToDevice, st));
  int32_t* d_ns = nullptr;
  if (h_nsamples) {
    if ((s = ensure(ctx, ctx->rgba, size_t(n_rays) * 4)) != ADN_OK) return s;
    d_ns = static_cast<int32_t*>(ctx->rgba.p);
  }
  s = render_impl(ctx, pose, rot, static_cast<float*>(ctx->dirs.p), nullptr, n_rays, thr, K, static_cast<float*>(ctx->rgb.p),
                  nullptr, d_ns, nullptr, st);
  if (s != ADN_OK) return s;
  ADN_CUDA(ctx, cudaMemcpyAsync(out_pinned ? static_cast<void*>(h_rgb) : ctx->h_out.p, ctx->rgb.p, size_t(n_rays) * 12,
                                cudaMemcpyDeviceToHost, st));
  if (h_nsamples)
    ADN_CUDA(ctx, cudaMemcpyAsync(ns_pinned ? static_cast<void*>(h_nsamples) : ctx->h_ns.p, d_ns, size_t(n_rays) * 4,
                                  cudaMemcpyDeviceToHost, st));
  ADN_CUDA(ctx, cudaStreamSynchronize(st));
  if (!out_pinned) std::memcpy(h_rgb, ctx->h_out.p, size_t(n_rays) * 12);
  if (h_nsamples && !ns_pinned) std::memcpy(h_nsamples, ctx->h_ns.p, size_t(n_rays) * 4);
  return check_device_error(ctx);
}

adn_status adn_render_camera_host(adn_ctx* ctx, const float* pose, const float* rot, int W, int H, int row0, int rows,
                                  float thr, int K, float* h_rgb, int32_t* h_nsamples) {
  if (!ctx || !h_rgb || W < 1 || H < 1 || row0 < 0 || rows < 0 || row0 + rows > H) return fail(ctx, ADN_ERR_INVALID, "render_camera_host: bad arguments");
  const int64_t n_rays = int64_t(rows) * W;
  if (n_rays == 0) return ADN_OK;
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  adn_status s;
  if ((s = ensure(ctx, ctx->rgb, size_t(n_rays) * 12)) != ADN_OK) return s;
  if ((s = ensure_pinned(ctx, ctx->h_out, size_t(n_rays) * 12)) != ADN_OK) return s;
  int32_t* d_ns = nullptr;
  if (h_nsamples) {
    if ((s = ensure(ctx, ctx->rgba, size_t(n_rays) * 4)) != ADN_OK) return s;
    if ((s = ensure_pinned(ctx, ctx->h_ns, size_t(n_rays) * 4)) != ADN_OK) return s;
    d_ns = static_cast<int32_t*>(ctx->rgba.p);
  }
  cudaStream_t st = ctx->own_stream;
  const bool out_pinned = pin_in_place(ctx, 1, h_rgb, size_t(n_rays) * 12);
  const bool ns_pinned = h_nsamples && pin_in_place(ctx, 2, h_nsamples, size_t(n_rays) * 4);
  const CameraRays cam = make_camera(ctx, W, H, row0);
  s = render_impl(ctx, pose, rot, nullptr, &cam, n_rays, thr, K, static_cast<float*>(ctx->rgb.p), nullptr, d_ns, nullptr, st);
  if (s != ADN_OK) return s;
  ADN_CUDA(ctx, cudaMemcpyAsync(out_pinned ? static_cast<void*>(h_rgb) : ctx->h_out.p, ctx->rgb.p, size_t(n_rays) * 12,
                                cudaMemcpyDeviceToHost, st));
  if (h_nsamples)
    ADN_CUDA(ctx, cudaMemcpyAsync(ns_pinned ? static_cast<void*>(h_nsamples) : ctx->h_ns.p, d_ns, size_t(n_rays) * 4,
                                  cudaMemcpyDeviceToHost, st));
  ADN_CUDA(ctx, cudaStreamSynchronize(st));
  if (!out_pinned) std::memcpy(h_rgb, ctx->h_out.p, size_t(n_rays) * 12);
  if (h_nsamples && !ns_pinned) std::memcpy(h_nsamples, ctx->h_ns.p, size_t(n_rays) * 4);
  return check_device_error(ctx);
}

// ---- stage-level entry points --------------------------------------------------------------------
adn_status adn_generate_ray_directions(adn_ctx* ctx, int W, int H, int row0, int rows, float* d_dirs, void* stream) {
  if (!ctx || !d_dirs || W < 1 || H < 1 || row0 < 0 || rows < 0 || row0 + rows > H) return fail(ctx, ADN_ERR_INVALID, "generate_ray_directions: bad arguments");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  const CameraRays cam = make_camera(ctx, W, H, row0);
  ADN_CUDA(ctx, launch_gen_dirs(cam, int64_t(rows) * W, d_dirs, static_cast<cudaStream_t>(stream)));
  ctx->stats.kernel_launches++;
  return ADN_OK;
}

adn_status adn_stage0_features(adn_ctx* ctx, const float* pose, const float* rot, const float* d_dirs, int64_t n_rays,
                               float* d_x0, float* d_ray_o, float* d_ray_d, void* stream) {
  if (!ctx || !pose || !rot || !d_dirs || n_rays < 0 || (d_ray_o == nullptr) != (d_ray_d == nullptr))
    return fail(ctx, ADN_ERR_INVALID, "stage0: bad arguments");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
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
  Net& n = ctx->net[0];
  adn_status s = ensure(ctx, ctx->tiles0, size_t(pad128(n_rays) / 128) * n.prog.in.tile_bytes());
  if (s != ADN_OK) return s;
  ADN_CUDA(ctx, launch_pack_rows(d_x0, n_rays, nullptr, n.n_in, n.prog.in, static_cast<uint8_t*>(ctx->tiles0.p), st));
  ctx->stats.kernel_launches++;
  return run_mlp(ctx, 0, static_cast<uint8_t*>(ctx->tiles0.p), d_raw0, nullptr, n_rays, st);
}

adn_status adn_stage2_sample(adn_ctx* ctx, const float* d_raw0, int64_t n_rays, float thr, int K, int32_t* d_count,
                             int32_t* d_offset, int32_t* d_cell, int32_t* d_ray, float* d_z, float* d_zp, int64_t* d_total,
                             void* stream) {
  if (!ctx || !d_total || n_rays < 0 || K < 1 || K > 128 || !(thr > 0.0f) ||
      (n_rays > 0 && (!d_raw0 || !d_count || !d_offset || !d_ray || !d_z || !d_zp)))
    return fail(ctx, ADN_ERR_INVALID, "stage2: bad arguments (adaptive path needs thr > 0)");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  adn_status s = ensure(ctx, ctx->s2scratch, stage2_scratch_bytes(n_rays));
  if (s != ADN_OK) return s;
  ADN_CUDA(ctx, launch_stage2(d_raw0, n_rays, thr, K, ctx->d_zlut, d_count, d_offset, d_cell, d_ray, d_z, d_zp,
                              reinterpret_cast<long long*>(d_total), ctx->s2scratch.p, &ctx->s2sync, static_cast<cudaStream_t>(stream)));
  ctx->stats.kernel_launches++;
  return ADN_OK;
}

adn_status adn_budget_threshold(adn_ctx* ctx, const float* d_raw0, int64_t n_rays, float thr_min, int K, int64_t max_samples,
                                float* d_thr, void* stream) {
  if (!ctx || !d_thr || n_rays < 0 || (n_rays > 0 && !d_raw0) || K < 1 || K > 128 || !(thr_min > 0.0f) || max_samples < n_rays)
    return fail(ctx, ADN_ERR_INVALID, "budget_threshold: bad arguments (need thr_min > 0, 1 <= K <= 128, max_samples >= n_rays)");
  if (n_rays * (K - 1) >= (int64_t(1) << 32))
    return fail(ctx, ADN_ERR_INVALID, "budget_threshold: at most 2^32 - 1 candidate samples (N * (K - 1))");
  if (reinterpret_cast<uintptr_t>(d_raw0) & 15u) return fail(ctx, ADN_ERR_INVALID, "budget_threshold: d_raw0 must be 16-byte aligned");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  adn_status s = ensure(ctx, ctx->budget_keys, size_t(std::max<int64_t>(1, n_rays * (K - 1))) * 4);
  if (s != ADN_OK || (s = ensure(ctx, ctx->budget_work, budget_work_bytes())) != ADN_OK) return s;
  int launches = 0;
  ADN_CUDA(ctx, launch_budget_threshold(d_raw0, n_rays, thr_min, K, max_samples, static_cast<uint32_t*>(ctx->budget_keys.p),
                                        ctx->budget_work.p, d_thr, ctx->num_sms, static_cast<cudaStream_t>(stream), &launches));
  ctx->stats.kernel_launches += launches;
  return ADN_OK;
}

adn_status adn_stage3_encode(adn_ctx* ctx, const float* d_ray_o, const float* d_ray_d, const int32_t* d_ray, const float* d_z,
                             int64_t n_samples, float* d_x1, void* stream) {
  if (!ctx || !d_ray_o || !d_ray_d || !d_ray || !d_z || !d_x1 || n_samples < 0) return fail(ctx, ADN_ERR_INVALID, "stage3: bad arguments");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  ADN_CUDA(ctx, launch_stage3(ctx->sc, d_ray_o, d_ray_d, d_ray, d_z, nullptr, 1, n_samples, nullptr, d_x1, nullptr,
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
  Net& n = ctx->net[1];
  adn_status s = ensure(ctx, ctx->tiles1, size_t(pad128(n_samples) / 128) * n.prog.in.tile_bytes());
  if (s != ADN_OK) return s;
  ADN_CUDA(ctx, launch_pack_rows(d_x1, n_samples, nullptr, n.n_in, n.prog.in, static_cast<uint8_t*>(ctx->tiles1.p), st));
  ctx->stats.kernel_launches++;
  return run_mlp(ctx, 1, static_cast<uint8_t*>(ctx->tiles1.p), d_raw1, nullptr, n_samples, st);
}

adn_status adn_stage5_composite(adn_ctx* ctx, const float* d_raw1, const float* d_zp, const float* d_z, const int32_t* d_offset,
                                const int32_t* d_count, int64_t n_rays, int K, float* d_rgb, float* d_weights,
                                float* d_depth_map, void* stream) {
  if (!ctx || !d_raw1 || !d_zp || !d_offset || !d_count || !d_rgb || n_rays < 0 || K < 1 || K > 128 || (d_depth_map && !d_z))
    return fail(ctx, ADN_ERR_INVALID, "stage5: bad arguments");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  Stage5Aux aux;
  aux.weights = d_weights;
  aux.depth_map = d_depth_map;
  ADN_CUDA(ctx, launch_stage5(d_raw1, d_zp, d_z, nullptr, d_offset, d_count, n_rays, K, 0, d_rgb, nullptr, aux,
                              static_cast<cudaStream_t>(stream)));
  ctx->stats.kernel_launches++;
  return ADN_OK;
}

adn_status adn_image_metrics(adn_ctx* ctx, const float* d_image, const float* d_reference, int64_t n_values, int clamp01,
                             double* mse_out, double* psnr_out, void* stream) {
  if (!ctx || !d_image || !d_reference || n_values < 1 || (!mse_out && !psnr_out))
    return fail(ctx, ADN_ERR_INVALID, "image_metrics: bad arguments");
  ADN_CUDA(ctx, cudaSetDevice(ctx->device));
  adn_status s = ensure(ctx, ctx->metric, sizeof(double) * (kMetricBlocks + 1));
  if (s != ADN_OK) return s;
  double* part = static_cast<double*>(ctx->metric.p);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
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
  if (!adn::load_export_dir(dir, ex, err)) {
    std::fprintf(stderr, "adanerf_b200: %s\n", err.c_str());
    return ADN_ERR_IO;
  }
  adn_ctx* ctx = nullptr;
  adn_status s = adn_create(&ctx, &ex.scene, device);
  if (s != ADN_OK) return s;
  for (int id = 0; id < 2; ++id) {
    std::vector<adn_tensor_desc> descs;
    for (auto& t : ex.nets[id]) descs.push_back({t.name.c_str(), t.data.data(), t.rows, t.cols});
    s = adn_set_weights(ctx, id, descs.data(), int(descs.size()));
    if (s != ADN_OK) {
      std::fprintf(stderr, "adanerf_b200: %s\n", ctx->last_error.c_str());
      adn_destroy(ctx);
      return s;
    }
  }
  if (thr_out) *thr_out = ex.threshold;
  if (k_out) *k_out = ex.num_samples;
  *out = ctx;
  return ADN_OK;
}

}  // extern "C"
