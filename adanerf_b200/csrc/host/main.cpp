// Headless counterpart of the viewer's main (adanerf_real_time_viewer/src/main.cpp:15-98): same positional
// model-path argument and -s / -bs options, renders `-f` frames along a small orbit inside the view cell,
// prints the per-frame time the way ImageGenerator::inference logs its 100-frame averages
// (imagegenerator.cpp:370-393) and optionally writes the last frame as a binary PPM (-w).  --views V renders V cameras per
// frame in one call (ImageGenerator::inference_views), spread evenly along the orbit, e.g. the two eyes of a stereo pair.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include <cuda_runtime_api.h>

#include "../../../include/adanerf_b200_multi.h"
#include "image_generator.h"

class FeatureSet {};   // stand-ins for the viewer's classes: only their names appear in ImageGenerator::inference
class Encoding {};

int main(int argc, char** argv) {
  std::string model = "sample/";
  int W = 800, H = 800, batch = -1, frames = 20, device = 0, gpus = 1, views = 0;
  long long budget = 0;   // --budget: samples per frame (0 = fixed threshold)
  bool write = false, surface = false, oracle = false;
  for (int i = 1; i < argc; ++i) {
    const std::string a = argv[i];
    if ((a == "-s" || a == "--size") && i + 2 < argc) { W = std::atoi(argv[++i]); H = std::atoi(argv[++i]); }
    else if ((a == "-bs" || a == "--batchSize") && i + 1 < argc) batch = std::atoi(argv[++i]);
    else if ((a == "-f" || a == "--frames") && i + 1 < argc) frames = std::atoi(argv[++i]);
    else if ((a == "-dev" || a == "--device") && i + 1 < argc) device = std::atoi(argv[++i]);
    else if (a == "-w" || a == "--writeImages") write = true;
    else if (a == "--surface") surface = true;   // one frame through ImageGenerator::inference(camera, cudaSurfaceObject_t, ...)
    else if ((a == "-g" || a == "--gpus") && i + 1 < argc) gpus = std::atoi(argv[++i]);
    else if (a == "--budget" && i + 1 < argc) budget = std::atoll(argv[++i]);
    else if (a == "--views" && i + 1 < argc) views = std::atoi(argv[++i]);   // V cameras per frame, one call
    else if (a == "--oracle") oracle = true;   // the sampling network's view (ImageGenerator::switchRenderOracle, the viewer's O key)
    else if (a[0] != '-') model = a;
    else { std::fprintf(stderr, "usage: %s modelPath [-s W H] [-bs raysPerBatch] [-f frames] [-dev id] [-g gpus] [--budget samplesPerFrame] [--views V] [--oracle] [--surface] [-w]\n", argv[0]); return 2; }
  }
  if (views != 0 && (views < 1 || gpus > 1 || surface)) {
    std::fprintf(stderr, "--views needs 1 <= V <= 64 on one GPU, without -g and --surface (row bands and the surface path are single-view)\n");
    return 2;
  }
  adn_host::Config config;
  if (!config.load(model)) { std::fprintf(stderr, "couldn't read export directory %s\n", model.c_str()); return 1; }
  std::printf("model %s: K = %d, adaptiveSamplingThreshold = %g\n", model.c_str(), config.numRaymarchSamples, config.adaptiveSamplingThreshold);
  if (config.one_network && (oracle || budget > 0)) {
    std::fprintf(stderr, "%s is a one-network export (LinearlySpacedZNearZFar): it has no sampling network to view (--oracle) "
                 "and places K samples on every ray (--budget)\n", model.c_str());
    return 2;
  }
  // -w: the last frame as a binary PPM in the model directory, saturate(x) * 255 truncated (the viewer's pixels)
  // (--views: adn_frame_view<v>.ppm, one per view)
  auto write_ppm = [&](const std::vector<float>& rgb, int view = -1) {
    const std::string out = model + (view < 0 ? std::string("/adn_frame.ppm") : "/adn_frame_view" + std::to_string(view) + ".ppm");
    FILE* fp = std::fopen(out.c_str(), "wb");
    if (!fp) { std::fprintf(stderr, "cannot write %s\n", out.c_str()); return false; }
    std::fprintf(fp, "P6\n%d %d\n255\n", W, H);
    const size_t px = size_t(W) * H * 3, first = view < 0 ? 0 : size_t(view) * px;
    for (size_t i = first; i < first + px; ++i) {
      const float v = rgb[i] > 0.f ? std::fmin(rgb[i], 1.f) : 0.f;
      std::fputc(int(v * 255.0f), fp);
    }
    std::fclose(fp);
    std::printf("wrote %s\n", out.c_str());
    return true;
  };
  if (gpus > 1) {
    // Row bands over `gpus` devices of this node + one NCCL gather per frame (include/adanerf_b200_multi.h); two frames
    // in flight, so the gather of a frame overlaps the next frame's sampling MLP.  --budget: one frame budget, every band at
    // the frame's threshold; frames are then rendered one at a time so that each one's threshold and M can be printed.
    adn_multi* m = nullptr;
    float thr = 0.f;
    int K = 0;
    if (adn_multi_create_from_export_dir(&m, model.c_str(), nullptr, gpus, &thr, &K) != ADN_OK) { std::fprintf(stderr, "multi-GPU load failed\n"); return 1; }
    if (budget > 0 && adn_multi_set_option(m, "sample_budget", budget) != ADN_OK) { std::fprintf(stderr, "sample budget: %s\n", adn_multi_last_error(m)); return 1; }
    if (oracle && adn_multi_set_option(m, "sampling_view", 1) != ADN_OK) { std::fprintf(stderr, "sampling view: %s\n", adn_multi_last_error(m)); return 1; }
    std::vector<int64_t> band_m(size_t(gpus), 0);
    adn_host::Camera cam;
    cam.width = W;
    cam.height = H;
    std::vector<float> rgb(size_t(W) * H * 3);
    float rot[9];
    auto pose_at = [&](int f) {
      const float t = 6.2831853f * float(f) / float(frames > 0 ? frames : 1);
      for (int a = 0; a < 3; ++a) cam.pos[a] = config.scene.view_cell_center[a];
      cam.pos[0] += 0.3f * config.scene.view_cell_size[0] * std::cos(t);
      cam.pos[1] += 0.3f * config.scene.view_cell_size[1] * std::sin(t);
      cam.yaw = t;
      cam.rotation(rot);
    };
    std::chrono::steady_clock::time_point t0;
    for (int f = 0; f < frames + 2; ++f) {
      if (f == 2) {   // two warm-up frames (allocation, NCCL channel setup): drain, then time a full pipeline
        if (budget == 0 && adn_multi_wait_frame(m, nullptr, nullptr) != ADN_OK) { std::fprintf(stderr, "%s\n", adn_multi_last_error(m)); return 1; }
        t0 = std::chrono::steady_clock::now();
      }
      pose_at(f);
      if (adn_multi_render_camera(m, cam.pos, rot, W, H, thr, K) != ADN_OK) { std::fprintf(stderr, "%s\n", adn_multi_last_error(m)); return 1; }
      if (budget > 0) {
        if (adn_multi_wait_frame(m, nullptr, f == frames + 1 ? rgb.data() : nullptr) != ADN_OK) { std::fprintf(stderr, "%s\n", adn_multi_last_error(m)); return 1; }
        if (f < 2) continue;
        float t = 0.f;
        if (adn_multi_last_threshold(m, &t) != ADN_OK || adn_multi_last_samples(m, band_m.data()) != ADN_OK) { std::fprintf(stderr, "%s\n", adn_multi_last_error(m)); return 1; }
        long long total = 0;
        for (int64_t b : band_m) total += b;
        std::printf("frame %d: threshold %.7g, %lld samples (budget %lld)\n", f - 2, double(t), total, budget);
        continue;
      }
      if (f >= 1 && f != 2 && adn_multi_wait_frame(m, nullptr, nullptr) != ADN_OK) { std::fprintf(stderr, "%s\n", adn_multi_last_error(m)); return 1; }
    }
    if (budget == 0 && adn_multi_wait_frame(m, nullptr, rgb.data()) != ADN_OK) { std::fprintf(stderr, "%s\n", adn_multi_last_error(m)); return 1; }
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    const size_t ng = size_t(gpus);
    std::vector<float> r_ms(ng, 0.f), g_ms(ng, 0.f);
    adn_multi_last_times(m, r_ms.data(), g_ms.data());
    float r_max = 0.f, g_max = 0.f;
    for (int i = 0; i < gpus; ++i) { r_max = std::max(r_max, r_ms[size_t(i)]); g_max = std::max(g_max, g_ms[size_t(i)]); }
    std::printf("%d frames %dx%d on %d GPUs: %.3f ms/frame (%.1f fps); last frame: slowest band %.3f ms, gather %.3f ms\n", frames, W, H, gpus,
                ms / frames, 1000.0 * frames / ms, r_max, g_max);
    double sum = 0;
    for (float v : rgb) sum += v;
    std::printf("checksum %.6f\n", sum);
    adn_multi_destroy(m);
    return write && !write_ppm(rgb) ? 1 : 0;
  }
  adn_host::ImageGenerator gen;
  if (!gen.load(config, device)) { std::fprintf(stderr, "load failed: %s\n", gen.last_error()); return 1; }
  adn_scene sc{};
  const bool probed = adn_probe_export_dir(model.c_str(), &sc, nullptr, nullptr, nullptr) == ADN_OK;
  for (int id = 0; id < 2; ++id) {
    int d = 0, w = 0, sk = -1;
    if (!gen.net_shape(id, &d, &w, &sk)) continue;
    // the encoding as adn_create reads the scene: a negative band count is posEnc none; the sampling net's 0 = the shading net's
    const int p = id == 0 && sc.n_freq_pos0 ? sc.n_freq_pos0 : sc.n_freq_pos, q = id == 0 && sc.n_freq_dir0 ? sc.n_freq_dir0 : sc.n_freq_dir;
    char enc[32] = "?";
    if (probed) std::snprintf(enc, sizeof(enc), p < 0 && q < 0 ? "none" : "%d-%d", p < 0 ? 0 : p, q < 0 ? 0 : q);
    std::printf("net %d: %s %d x %d, skip %d, posEnc %s", id, id == 0 ? "sampling" : "shading", d, w, sk, enc);
    if (id == 0) std::printf(", %d depth cells", gen.depth_cells());
    std::printf("\n");
  }
  if (budget > 0 && !gen.set_sample_budget(budget)) { std::fprintf(stderr, "sample budget: %s\n", gen.last_error()); return 1; }
  if (oracle) gen.switchRenderOracle();
  const int nv = std::max(views, 1);
  std::vector<int32_t> ns(budget > 0 ? size_t(W) * H * nv : 0);   // per-ray sample counts, for M under a budget
  adn_host::Camera cam;
  cam.width = W;
  cam.height = H;
  std::vector<adn_host::Camera> cams(size_t(nv), cam);
  std::vector<float> rgb(size_t(W) * H * 3 * nv);
  float* d_rgb = nullptr;   // --views: the frame's views on the device, copied back after each call
  int32_t* d_ns = nullptr;
  if (views > 0 && (cudaMalloc(reinterpret_cast<void**>(&d_rgb), rgb.size() * 4) != cudaSuccess || (budget > 0 && cudaMalloc(reinterpret_cast<void**>(&d_ns), ns.size() * 4) != cudaSuccess))) {
    std::fprintf(stderr, "cudaMalloc failed\n");
    return 1;
  }
  double total_ms = 0;
  for (int f = 0; f < frames + 2; ++f) {
    const float t = 6.2831853f * float(f) / float(frames > 0 ? frames : 1);
    for (int v = 0; v < nv; ++v) {   // view v a 1 / V turn further along the orbit
      const float tv = t + 6.2831853f * float(v) / float(nv);
      adn_host::Camera& c = cams[size_t(v)];
      for (int a = 0; a < 3; ++a) c.pos[a] = config.scene.view_cell_center[a];
      c.pos[0] += 0.3f * config.scene.view_cell_size[0] * std::cos(tv);
      c.pos[1] += 0.3f * config.scene.view_cell_size[1] * std::sin(tv);
      c.yaw = tv;
    }
    cam = cams[0];
    const auto t0 = std::chrono::steady_clock::now();
    const bool ok = views > 0 ? gen.inference_views(cams.data(), nv, d_rgb, batch, config.numRaymarchSamples, d_ns) &&
                                    cudaMemcpy(rgb.data(), d_rgb, rgb.size() * 4, cudaMemcpyDeviceToHost) == cudaSuccess &&
                                    (!d_ns || cudaMemcpy(ns.data(), d_ns, ns.size() * 4, cudaMemcpyDeviceToHost) == cudaSuccess)
                              : gen.inference_host(cam, rgb.data(), batch, config.numRaymarchSamples, budget > 0 ? ns.data() : nullptr);
    if (!ok) {
      std::fprintf(stderr, "inference failed: %s\n", gen.last_error());
      return 1;
    }
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (f >= 2) total_ms += ms;   // two warm-up frames (allocation)
    if (budget > 0 && f >= 2) {
      float thr = 0.f;
      long long m = 0;
      for (int32_t c : ns) m += c;
      if (!gen.last_threshold(&thr)) { std::fprintf(stderr, "%s\n", gen.last_error()); return 1; }
      std::printf("frame %d: threshold %.7g, %lld samples (budget %lld)\n", f - 2, double(thr), m, budget);
    }
  }
  if (surface) {
    // The viewer's frame path: a cudaArray with surface load / store (what cudaGraphicsGLRegisterImage hands out,
    // interoprenderbuffer.cpp:53-83), a surface object on it, ImageGenerator::inference with the reference's signature.
    cudaArray_t arr = nullptr;
    const cudaChannelFormatDesc fmt = cudaCreateChannelDesc(8, 8, 8, 8, cudaChannelFormatKindUnsigned);   // uchar4
    cudaResourceDesc res{};
    cudaSurfaceObject_t surf = 0;
    if (cudaMallocArray(&arr, &fmt, size_t(W), size_t(H), cudaArraySurfaceLoadStore) != cudaSuccess) { std::fprintf(stderr, "cudaMallocArray failed\n"); return 1; }
    res.resType = cudaResourceTypeArray;
    res.res.array.array = arr;
    if (cudaCreateSurfaceObject(&surf, &res) != cudaSuccess) { std::fprintf(stderr, "cudaCreateSurfaceObject failed\n"); return 1; }
    std::vector<FeatureSet*> fs;
    std::vector<Encoding> enc;
    if (!gen.inference(cam, (unsigned long long)surf, batch, config.numRaymarchSamples, fs, enc)) { std::fprintf(stderr, "inference failed: %s\n", gen.last_error()); return 1; }
    cudaDeviceSynchronize();
    std::vector<unsigned char> px(size_t(W) * H * 4);
    if (cudaMemcpy2DFromArray(px.data(), size_t(W) * 4, arr, 0, 0, size_t(W) * 4, size_t(H), cudaMemcpyDeviceToHost) != cudaSuccess) { std::fprintf(stderr, "readback failed\n"); return 1; }
    // rgb holds the same camera's fp32 frame (last loop iteration): saturate(x) * 255 truncated, alpha 255 -- the
    // viewer's clamp as nvcc compiles it (FADD.SAT: NaN -> 0)
    size_t bad = 0;
    for (size_t i = 0; i < size_t(W) * H; ++i) {
      for (int c = 0; c < 3; ++c) {
        const float v = rgb[3 * i + c] > 0.f ? std::fmin(rgb[3 * i + c], 1.f) : 0.f;
        if (px[4 * i + c] != (unsigned char)(v * 255.0f)) ++bad;
      }
      if (px[4 * i + 3] != 255) ++bad;
    }
    std::printf("surface frame %dx%d%s: %zu mismatching bytes against the fp32 frame\n", W, H, oracle ? " (sampling view)" : "", bad);
    cudaDestroySurfaceObject(surf);
    cudaFreeArray(arr);
    if (bad) return 1;
  }
  adn_stats st{};
  gen.stats(&st);
  std::printf("%d frames %dx%d%s: %.3f ms/frame (%.1f fps), last frame %lld samples (%.2f per ray), %lld kernel launches\n", frames, W, H,
              views > 0 ? (" x " + std::to_string(nv) + " views").c_str() : "", total_ms / frames, 1000.0 * frames / total_ms,
              (long long)st.n_samples, double(st.n_samples) / (double(W) * H * nv), (long long)st.kernel_launches);
  for (int v = 0; views > 0 && v < nv; ++v) {   // the last frame's cameras, with every float exact (%.9g)
    const adn_host::Camera& c = cams[size_t(v)];
    float rot[9];
    c.rotation(rot);
    std::printf("view %d: pos %.9g %.9g %.9g rot", v, double(c.pos[0]), double(c.pos[1]), double(c.pos[2]));
    for (float r : rot) std::printf(" %.9g", double(r));
    std::printf("\n");
  }
  double sum = 0;   // the same checksum as the multi-GPU path prints, of the last frame
  for (float v : rgb) sum += v;
  std::printf("checksum %.6f\n", sum);
  cudaFree(d_rgb);
  cudaFree(d_ns);
  if (write && views > 0) {
    for (int v = 0; v < nv; ++v)
      if (!write_ppm(rgb, v)) return 1;
    return 0;
  }
  return write && !write_ppm(rgb) ? 1 : 0;
}
