#include "image_generator.h"

#include <cmath>

namespace adn_host {

bool Config::load(const std::string& dir) {
  model_dir = dir;
  int n[2] = {0, 0};
  // a one-network export (LinearlySpacedZNearZFar) has its net in the shading slot and none in the sampling slot
  if (adn_probe_export_dir(dir.c_str(), &scene, &adaptiveSamplingThreshold, &numRaymarchSamples, n) != ADN_OK || n[1] <= 0)
    return false;
  one_network = n[0] == 0;
  return true;
}

void Camera::rotation(float rot[9]) const {
  // forward = (cos pitch * sin yaw, cos pitch * cos yaw, sin pitch) in the z-up world of the DONeRF scenes;
  // the pinhole rays look down -z in camera space (src/util/raygeneration.py:24-25).
  const float cp = std::cos(pitch), sp = std::sin(pitch), cy = std::cos(yaw), sy = std::sin(yaw);
  const float f[3] = {cp * sy, cp * cy, sp};
  const float r[3] = {cy, -sy, 0.f};                                    // right = forward x world-up, normalised
  const float u[3] = {r[1] * f[2] - r[2] * f[1], r[2] * f[0] - r[0] * f[2], r[0] * f[1] - r[1] * f[0]};   // up = right x forward
  for (int i = 0; i < 3; ++i) {
    rot[3 * i + 0] = r[i];
    rot[3 * i + 1] = u[i];
    rot[3 * i + 2] = -f[i];
  }
}

ImageGenerator::~ImageGenerator() {
  if (ctx_) adn_destroy(ctx_);
}

bool ImageGenerator::load(const Config& config, int device) {
  if (ctx_) {
    adn_destroy(ctx_);
    ctx_ = nullptr;
  }
  int k = 0;
  const adn_status s = adn_create_from_export_dir(&ctx_, config.model_dir.c_str(), device, &thr_, &k);
  if (s != ADN_OK) {
    err_ = std::string("adn_create_from_export_dir: ") + adn_strerror(s);
    return false;
  }
  return true;
}

bool ImageGenerator::apply_options(int batch_size) {
  if (batch_size > 0) adn_set_option(ctx_, "chunk_rays", batch_size);
  if (adn_set_option(ctx_, "sampling_view", render_oracle_ ? 1 : 0) != ADN_OK) {
    err_ = adn_last_error(ctx_);
    return false;
  }
  return true;
}

bool ImageGenerator::inference(const Camera& camera, uint8_t* d_rgba8, int batch_size, int num_samples, void* stream) {
  if (!ctx_) return false;
  float rot[9];
  camera.rotation(rot);
  if (!apply_options(batch_size)) return false;
  const adn_status s =
      adn_render_camera_rgba8(ctx_, camera.pos, rot, camera.width, camera.height, 0, camera.height, thr_, num_samples, d_rgba8, stream);
  if (s != ADN_OK) err_ = adn_last_error(ctx_);
  return s == ADN_OK;
}

bool ImageGenerator::inference(Camera& camera, unsigned long long output_surf, int batch_size, int num_samples,
                               std::vector<::FeatureSet*>& /*feature_sets*/, std::vector<::Encoding>& /*encodings*/) {
  if (!ctx_) return false;
  float rot[9];
  camera.rotation(rot);
  if (!apply_options(batch_size)) return false;
  const adn_status s = adn_render_camera_surface(ctx_, camera.pos, rot, camera.width, camera.height, 0, camera.height, thr_, num_samples,
                                                 output_surf, nullptr);
  if (s != ADN_OK) err_ = adn_last_error(ctx_);
  return s == ADN_OK;
}

bool ImageGenerator::inference_host(const Camera& camera, float* h_rgb, int batch_size, int num_samples, int32_t* h_nsamples) {
  if (!ctx_) return false;
  float rot[9];
  camera.rotation(rot);
  if (!apply_options(batch_size)) return false;
  const adn_status s =
      adn_render_camera_host(ctx_, camera.pos, rot, camera.width, camera.height, 0, camera.height, thr_, num_samples, h_rgb, h_nsamples);
  if (s != ADN_OK) err_ = adn_last_error(ctx_);
  return s == ADN_OK;
}

bool ImageGenerator::inference_views(const Camera* cameras, int n_views, float* d_rgb, int batch_size, int num_samples,
                                     int32_t* d_nsamples, void* stream) {
  if (!ctx_) return false;
  if (!cameras || n_views < 1) {
    err_ = "inference_views: need at least one camera";
    return false;
  }
  std::vector<float> poses(size_t(n_views) * 3), rots(size_t(n_views) * 9);
  for (int v = 0; v < n_views; ++v) {
    const Camera& c = cameras[v];
    if (c.width != cameras[0].width || c.height != cameras[0].height) {
      err_ = "inference_views: every camera must have the same size";
      return false;
    }
    for (int a = 0; a < 3; ++a) poses[size_t(v) * 3 + a] = c.pos[a];
    c.rotation(rots.data() + size_t(v) * 9);
  }
  if (!apply_options(batch_size)) return false;
  const adn_status s = adn_render_views_camera(ctx_, n_views, poses.data(), rots.data(), cameras[0].width, cameras[0].height, thr_,
                                               num_samples, d_rgb, d_nsamples, stream);
  if (s != ADN_OK) err_ = adn_last_error(ctx_);
  return s == ADN_OK;
}

bool ImageGenerator::set_sample_budget(int64_t max_samples) {
  if (!ctx_) return false;
  const adn_status s = adn_set_option(ctx_, "sample_budget", max_samples);
  if (s != ADN_OK) err_ = adn_last_error(ctx_);
  return s == ADN_OK;
}

bool ImageGenerator::last_threshold(float* thr) {
  if (!ctx_) return false;
  const adn_status s = adn_last_threshold(ctx_, thr);
  if (s != ADN_OK) err_ = adn_last_error(ctx_);
  return s == ADN_OK;
}

const char* ImageGenerator::last_error() const { return err_.c_str(); }

bool ImageGenerator::stats(adn_stats* out) { return ctx_ && adn_get_stats(ctx_, out) == ADN_OK; }

bool ImageGenerator::net_shape(int net_id, int* depth, int* width, int* skip) {
  return ctx_ && adn_net_shape(ctx_, net_id, depth, width, skip) == ADN_OK;
}

int ImageGenerator::depth_cells() {
  int n_out = 0;
  return ctx_ && adn_net_dims(ctx_, 0, nullptr, &n_out) == ADN_OK ? n_out : 0;
}

}  // namespace adn_host
