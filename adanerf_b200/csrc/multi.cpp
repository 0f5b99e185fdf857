// Multi-GPU frame renderer over the single-device C ABI + NCCL (see include/adanerf_b200_multi.h).
#include <cuda_runtime.h>
#include <nccl.h>

#include <cstdio>
#include <string>
#include <thread>
#include <vector>

#include "../../include/adanerf_b200_multi.h"
#include "export_loader.h"

namespace {

struct Dev {
  int device = 0;
  adn_ctx* ctx = nullptr;
  ncclComm_t comm = nullptr;
  cudaStream_t render = nullptr, comm_s = nullptr;
  float* band[2] = {nullptr, nullptr};
  int32_t* ns[2] = {nullptr, nullptr};      // the band's per-ray sample counts
  size_t band_cap = 0;                      // floats per buffer
  cudaEvent_t start[2] = {}, rendered[2] = {}, gathered[2] = {};
};

}  // namespace

struct adn_multi {
  std::vector<Dev> devs;
  float* frame[2] = {nullptr, nullptr};     // on devs[0]
  size_t frame_cap = 0;
  long long issued = 0, waited = 0;         // frames enqueued / handed out
  int W[2] = {0, 0}, H[2] = {0, 0};
  int64_t budget = 0;                       // option "sample_budget": samples per frame, over all bands
  bool view = false;                        // option "sampling_view": the bands draw the sampling net's view (no budget)
  std::string err;
};

namespace {

adn_status fail(adn_multi* m, adn_status s, const std::string& msg) {
  if (m) m->err = msg;
  return s;
}
#define MCUDA(m, call)                                                                            \
  do {                                                                                            \
    cudaError_t e__ = (call);                                                                     \
    if (e__ != cudaSuccess) return fail(m, ADN_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e__)); \
  } while (0)
#define MNCCL(m, call)                                                                            \
  do {                                                                                            \
    ncclResult_t r__ = (call);                                                                    \
    if (r__ != ncclSuccess) return fail(m, ADN_ERR_CUDA, std::string(#call) + ": " + ncclGetErrorString(r__)); \
  } while (0)
#define MADN(m, d, call)                                                                          \
  do {                                                                                            \
    adn_status s__ = (call);                                                                      \
    if (s__ != ADN_OK) return fail(m, s__, std::string(#call) + ": " + adn_last_error((d).ctx));  \
  } while (0)

// adn_budget_reduce_fn of a device's context: sums a select round's histogram words over all devices' bands.
int all_reduce_u64(void* user, uint64_t* d_words, int64_t n_words, void* stream) {
  const Dev* d = static_cast<const Dev*>(user);
  return ncclAllReduce(d_words, d_words, size_t(n_words), ncclUint64, ncclSum, d->comm, static_cast<cudaStream_t>(stream)) == ncclSuccess ? 0 : 1;
}

void band_of(int G, int H, int rank, int* row0, int* rows) {
  const int base = H / G, extra = H % G;
  *row0 = rank * base + (rank < extra ? rank : extra);
  *rows = base + (rank < extra ? 1 : 0);
}

}  // namespace

extern "C" {

adn_status adn_multi_create(adn_multi** out, const adn_scene* scene, const int* devices, int n_devices) {
  if (!out || !scene || n_devices < 1 || n_devices > 64) return ADN_ERR_INVALID;
  *out = nullptr;
  adn_multi* m = new adn_multi();
  m->devs.resize(size_t(n_devices));
  std::vector<int> ids(static_cast<size_t>(n_devices));
  for (int r = 0; r < n_devices; ++r) ids[size_t(r)] = devices ? devices[r] : r;
  auto bail = [&](adn_status s) {
    adn_multi_destroy(m);
    return s;
  };
  for (int r = 0; r < n_devices; ++r) {
    Dev& d = m->devs[size_t(r)];
    d.device = ids[size_t(r)];
    adn_status s = adn_create(&d.ctx, scene, d.device);
    if (s != ADN_OK) return bail(s);
    if (cudaSetDevice(d.device) != cudaSuccess || cudaStreamCreateWithFlags(&d.render, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&d.comm_s, cudaStreamNonBlocking) != cudaSuccess)
      return bail(ADN_ERR_CUDA);
    for (int k = 0; k < 2; ++k)
      if (cudaEventCreate(&d.start[k]) != cudaSuccess || cudaEventCreate(&d.rendered[k]) != cudaSuccess ||
          cudaEventCreate(&d.gathered[k]) != cudaSuccess)
        return bail(ADN_ERR_CUDA);
  }
  if (n_devices > 1) {   // one process, one communicator per device (SURVEY.md 8e)
    std::vector<ncclComm_t> comms(static_cast<size_t>(n_devices));
    if (ncclCommInitAll(comms.data(), n_devices, ids.data()) != ncclSuccess) return bail(ADN_ERR_CUDA);
    for (int r = 0; r < n_devices; ++r) m->devs[size_t(r)].comm = comms[size_t(r)];
  }
  *out = m;
  return ADN_OK;
}

adn_status adn_multi_create_from_export_dir(adn_multi** out, const char* dir, const int* devices, int n_devices, float* thr_out,
                                            int* k_out) {
  if (!out || !dir) return ADN_ERR_INVALID;
  adn::ExportDir ex;
  std::string err;
  if (!adn::load_export_dir(dir, ex, err) || !adn::check_depth_cells(ex, err)) {
    std::fprintf(stderr, "adanerf_b200: %s\n", err.c_str());
    return ADN_ERR_IO;
  }
  adn_status s = adn_multi_create(out, &ex.scene, devices, n_devices);
  if (s != ADN_OK) return s;
  for (int id = 0; id < 2; ++id) {
    if (ex.sampler == 2 && id == 0) continue;   // a one-network export: its net is in slot 1
    std::vector<adn_tensor_desc> descs;
    for (auto& t : ex.nets[id]) descs.push_back({t.name.c_str(), t.data.data(), t.rows, t.cols});
    s = adn_multi_set_weights(*out, id, descs.data(), int(descs.size()));
    if (s != ADN_OK) {
      std::fprintf(stderr, "adanerf_b200: %s\n", (*out)->err.c_str());
      adn_multi_destroy(*out);
      *out = nullptr;
      return s;
    }
  }
  // a FromClassifiedDepth export: every band renders with the fixed-K sampler and the export's transform
  // a LinearlySpacedZNearZFar export: every band renders K evenly spaced samples with the one network
  if ((ex.sampler == 2 && (s = adn_multi_set_option(*out, "sampler", 2)) != ADN_OK) ||
      (ex.sampler == 1 && ((s = adn_multi_set_option(*out, "sampler", 1)) != ADN_OK ||
                           (s = adn_multi_set_option(*out, "pdf_transform", ex.pdf_transform)) != ADN_OK))) {
    std::fprintf(stderr, "adanerf_b200: %s\n", (*out)->err.c_str());
    adn_multi_destroy(*out);
    *out = nullptr;
    return s;
  }
  if (thr_out) *thr_out = ex.threshold;
  if (k_out) *k_out = ex.num_samples;
  return ADN_OK;
}

void adn_multi_destroy(adn_multi* m) {
  if (!m) return;
  for (Dev& d : m->devs) {
    cudaSetDevice(d.device);
    cudaDeviceSynchronize();
  }
  for (Dev& d : m->devs) {
    cudaSetDevice(d.device);
    if (d.comm) ncclCommDestroy(d.comm);
    for (int k = 0; k < 2; ++k) {
      if (d.band[k]) cudaFree(d.band[k]);
      if (d.ns[k]) cudaFree(d.ns[k]);
      if (d.start[k]) cudaEventDestroy(d.start[k]);
      if (d.rendered[k]) cudaEventDestroy(d.rendered[k]);
      if (d.gathered[k]) cudaEventDestroy(d.gathered[k]);
    }
    if (d.render) cudaStreamDestroy(d.render);
    if (d.comm_s) cudaStreamDestroy(d.comm_s);
    if (d.ctx) adn_destroy(d.ctx);
  }
  if (!m->devs.empty()) {
    cudaSetDevice(m->devs[0].device);
    for (int k = 0; k < 2; ++k)
      if (m->frame[k]) cudaFree(m->frame[k]);
  }
  delete m;
}

const char* adn_multi_last_error(const adn_multi* m) { return m ? m->err.c_str() : "null"; }
int adn_multi_devices(const adn_multi* m) { return m ? int(m->devs.size()) : 0; }

adn_status adn_multi_set_weights(adn_multi* m, int net_id, const adn_tensor_desc* tensors, int n_tensors) {
  if (!m) return ADN_ERR_INVALID;
  for (Dev& d : m->devs) MADN(m, d, adn_set_weights(d.ctx, net_id, tensors, n_tensors));
  return ADN_OK;
}

adn_status adn_multi_set_option(adn_multi* m, const char* name, int64_t value) {
  if (!m || !name) return ADN_ERR_INVALID;
  for (Dev& d : m->devs) MADN(m, d, adn_set_option(d.ctx, name, value));
  if (std::string(name) == "sample_budget") {
    // B holds for the frame: on several devices every band's selection sums its histograms with the other bands' (NCCL)
    m->budget = value;
    const bool group = value > 0 && m->devs.size() > 1;
    for (Dev& d : m->devs) MADN(m, d, adn_set_budget_group(d.ctx, group ? all_reduce_u64 : nullptr, &d));
  }
  if (std::string(name) == "sampling_view") m->view = value != 0;
  return ADN_OK;
}

void adn_multi_band(const adn_multi* m, int H, int rank, int* row0, int* rows) {
  int a = 0, b = 0;
  if (m && rank >= 0 && rank < int(m->devs.size())) band_of(int(m->devs.size()), H, rank, &a, &b);
  if (row0) *row0 = a;
  if (rows) *rows = b;
}

adn_status adn_multi_render_camera(adn_multi* m, const float* pose, const float* rot, int W, int H, float thr, int K) {
  if (!m || !pose || !rot || W < 1 || H < 1) return fail(m, ADN_ERR_INVALID, "multi_render_camera: bad arguments");
  if (m->issued - m->waited >= 2) return fail(m, ADN_ERR_INVALID, "multi_render_camera: two frames already in flight (adn_multi_wait_frame first)");
  const int G = int(m->devs.size());
  const int slot = int(m->issued & 1);
  const size_t frame_floats = size_t(W) * H * 3;
  const int64_t n_rays = int64_t(W) * H;
  // what a band cannot see for itself is refused here, before any device enqueues: a band that failed before its first
  // reduction would leave the others waiting in theirs.  The sampling net's view applies no budget.
  const int64_t budget = m->view ? 0 : m->budget;
  if (budget > 0 && thr == 0.0f)
    return fail(m, ADN_ERR_INVALID, "multi_render_camera: sample_budget needs the adaptive path (thr > 0), not dense mode");
  if (budget > 0 && budget < n_rays)
    return fail(m, ADN_ERR_INVALID, "multi_render_camera: sample_budget " + std::to_string(budget) + " is below the " +
                                        std::to_string(n_rays) + " rays of the frame (every ray keeps at least one sample)");
  if (budget > 0 && n_rays * (K - 1) >= (int64_t(1) << 32))
    return fail(m, ADN_ERR_INVALID, "multi_render_camera: sample_budget supports at most 2^32 - 1 candidate samples (W * H * (K - 1)) per frame");
  const bool grouped = budget > 0 && G > 1;
  Dev& d0 = m->devs[0];
  if (frame_floats > m->frame_cap) {   // (re)allocate both frame buffers: only when idle
    if (m->issued != m->waited) return fail(m, ADN_ERR_INVALID, "multi_render_camera: frame size changed with a frame in flight");
    MCUDA(m, cudaSetDevice(d0.device));
    for (int k = 0; k < 2; ++k) {
      if (m->frame[k]) MCUDA(m, cudaFree(m->frame[k]));
      m->frame[k] = nullptr;
      MCUDA(m, cudaMalloc(&m->frame[k], frame_floats * sizeof(float)));
    }
    m->frame_cap = frame_floats;
  }
  for (int r = 0; r < G; ++r) {
    Dev& d = m->devs[size_t(r)];
    int row0, rows;
    band_of(G, H, r, &row0, &rows);
    const size_t n = size_t(rows) * W * 3;
    MCUDA(m, cudaSetDevice(d.device));
    if (n > d.band_cap) {
      if (m->issued != m->waited) return fail(m, ADN_ERR_INVALID, "multi_render_camera: frame size changed with a frame in flight");
      for (int k = 0; k < 2; ++k) {
        if (d.band[k]) MCUDA(m, cudaFree(d.band[k]));
        if (d.ns[k]) MCUDA(m, cudaFree(d.ns[k]));
        d.band[k] = nullptr;
        d.ns[k] = nullptr;
        MCUDA(m, cudaMalloc(&d.band[k], n * sizeof(float)));
        MCUDA(m, cudaMalloc(&d.ns[k], n / 3 * sizeof(int32_t)));
      }
      d.band_cap = n;
    }
  }
  // every device renders its band (its own rays from pose / rot / row window: no input scatter), enqueued from a host
  // thread of its own: a band's budget selection issues NCCL collectives, which one thread cannot issue for several
  // devices outside a group call.  Under a budget a device with no rows still makes its empty call, to take part.
  struct Enqueued {
    adn_status s = ADN_OK;
    std::string msg;
  };
  std::vector<Enqueued> res(static_cast<size_t>(G));
  auto enqueue = [&](int r) {
    Dev& d = m->devs[size_t(r)];
    Enqueued& out = res[size_t(r)];
    auto cuda = [&](cudaError_t e, const char* what) {
      if (e != cudaSuccess) {
        out.s = ADN_ERR_CUDA;
        out.msg = std::string(what) + ": " + cudaGetErrorString(e);
      }
      return e == cudaSuccess;
    };
    int row0, rows;
    band_of(G, H, r, &row0, &rows);
    // the band buffer of this slot was the source of the gather two frames ago
    if (!cuda(cudaSetDevice(d.device), "cudaSetDevice") || !cuda(cudaStreamWaitEvent(d.render, d.gathered[slot], 0), "cudaStreamWaitEvent") ||
        !cuda(cudaEventRecord(d.start[slot], d.render), "cudaEventRecord"))
      return;
    if (rows > 0 || grouped) {
      out.s = adn_render_camera(d.ctx, pose, rot, W, H, row0, rows, thr, K, d.band[slot], d.ns[slot], d.render);
      if (out.s != ADN_OK) {
        out.msg = std::string("adn_render_camera on device ") + std::to_string(d.device) + ": " + adn_last_error(d.ctx);
        return;
      }
    }
    if (cuda(cudaEventRecord(d.rendered[slot], d.render), "cudaEventRecord"))
      cuda(cudaStreamWaitEvent(d.comm_s, d.rendered[slot], 0), "cudaStreamWaitEvent");
  };
  if (G == 1) {
    enqueue(0);
  } else {
    std::vector<std::thread> threads;
    for (int r = 0; r < G; ++r) threads.emplace_back(enqueue, r);
    for (std::thread& t : threads) t.join();
  }
  for (const Enqueued& e : res)
    if (e.s != ADN_OK) return fail(m, e.s, e.msg);
  // ONE gather of the RGB tiles on the first device: grouped send / recv over NVLink; the first device's own band is a
  // device-to-device copy on its communication stream
  {
    int row0, rows;
    band_of(G, H, 0, &row0, &rows);
    MCUDA(m, cudaSetDevice(d0.device));
    if (rows > 0)
      MCUDA(m, cudaMemcpyAsync(m->frame[slot] + size_t(row0) * W * 3, d0.band[slot], size_t(rows) * W * 3 * sizeof(float),
                               cudaMemcpyDeviceToDevice, d0.comm_s));
  }
  if (G > 1) {
    MNCCL(m, ncclGroupStart());
    ncclResult_t res = ncclSuccess;
    for (int r = 1; r < G && res == ncclSuccess; ++r) {
      Dev& d = m->devs[size_t(r)];
      int row0, rows;
      band_of(G, H, r, &row0, &rows);
      const size_t n = size_t(rows) * W * 3;
      if (n == 0) continue;
      res = ncclSend(d.band[slot], n, ncclFloat, 0, d.comm, d.comm_s);
      if (res == ncclSuccess) res = ncclRecv(m->frame[slot] + size_t(row0) * W * 3, n, ncclFloat, r, d0.comm, d0.comm_s);
    }
    const ncclResult_t end = ncclGroupEnd();   // the group is closed on every path
    if (res != ncclSuccess) return fail(m, ADN_ERR_CUDA, std::string("ncclSend / ncclRecv: ") + ncclGetErrorString(res));
    MNCCL(m, end);
  }
  for (int r = 0; r < G; ++r) {
    Dev& d = m->devs[size_t(r)];
    MCUDA(m, cudaSetDevice(d.device));
    MCUDA(m, cudaEventRecord(d.gathered[slot], d.comm_s));
  }
  m->W[slot] = W;
  m->H[slot] = H;
  ++m->issued;
  return ADN_OK;
}

adn_status adn_multi_wait_frame(adn_multi* m, const float** d_frame, float* h_rgb) {
  if (!m) return ADN_ERR_INVALID;
  if (m->issued == m->waited) return fail(m, ADN_ERR_INVALID, "multi_wait_frame: no frame in flight");
  const int slot = int(m->waited & 1);
  for (Dev& d : m->devs) {
    MCUDA(m, cudaSetDevice(d.device));
    MCUDA(m, cudaEventSynchronize(d.gathered[slot]));
  }
  ++m->waited;
  if (d_frame) *d_frame = m->frame[slot];
  if (h_rgb) {
    MCUDA(m, cudaSetDevice(m->devs[0].device));
    MCUDA(m, cudaMemcpy(h_rgb, m->frame[slot], size_t(m->W[slot]) * m->H[slot] * 3 * sizeof(float), cudaMemcpyDeviceToHost));
  }
  return ADN_OK;
}

adn_status adn_multi_last_threshold(adn_multi* m, float* thr_out) {
  if (!m || !thr_out || m->issued == 0) return fail(m, ADN_ERR_INVALID, "multi_last_threshold: no frame enqueued");
  Dev& d = m->devs[0];   // every band of a budgeted frame rendered at the same t*; the first band is never empty
  MADN(m, d, adn_last_threshold(d.ctx, thr_out));
  return ADN_OK;
}

adn_status adn_multi_last_samples(adn_multi* m, int64_t* band_samples) {
  if (!m || !band_samples || m->issued == 0) return fail(m, ADN_ERR_INVALID, "multi_last_samples: no frame enqueued");
  const int slot = int((m->issued - 1) & 1), G = int(m->devs.size());
  std::vector<int32_t> ns;
  for (int r = 0; r < G; ++r) {
    Dev& d = m->devs[size_t(r)];
    int row0, rows;
    band_of(G, m->H[slot], r, &row0, &rows);
    ns.resize(size_t(rows) * m->W[slot]);
    MCUDA(m, cudaSetDevice(d.device));
    MCUDA(m, cudaEventSynchronize(d.rendered[slot]));
    if (!ns.empty()) MCUDA(m, cudaMemcpy(ns.data(), d.ns[slot], ns.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
    int64_t sum = 0;
    for (int32_t c : ns) sum += c;
    band_samples[r] = sum;
  }
  return ADN_OK;
}

adn_status adn_multi_last_times(adn_multi* m, float* render_ms, float* gather_ms) {
  if (!m || m->waited == 0) return fail(m, ADN_ERR_INVALID, "multi_last_times: no completed frame");
  const int slot = int((m->waited - 1) & 1);
  for (size_t r = 0; r < m->devs.size(); ++r) {
    Dev& d = m->devs[r];
    MCUDA(m, cudaSetDevice(d.device));
    float a = 0.f, b = 0.f;
    if (m->issued - m->waited >= 2)   // that slot's events have been re-recorded by the newest frame in flight
      return fail(m, ADN_ERR_INVALID, "multi_last_times: call it before enqueuing the second next frame");
    MCUDA(m, cudaEventElapsedTime(&a, d.start[slot], d.rendered[slot]));
    MCUDA(m, cudaEventElapsedTime(&b, d.rendered[slot], d.gathered[slot]));
    if (render_ms) render_ms[r] = a;
    if (gather_ms) gather_ms[r] = b;
  }
  return ADN_OK;
}

}  // extern "C"
