// C++ host side for the viewer: the public surface of the reference's `ImageGenerator`
// (adanerf_real_time_viewer/include/imagegenerator.h:61-62 `inference(...)`, :58 `load(...)`) and the pieces
// of `Config` / `Camera` it needs (config.h:31-59, camera.h), re-implemented over the C ABI
// (include/adanerf_b200.h).  No TensorRT, no OpenGL: the frame is produced into a linear RGBA8 / fp32 buffer
// that the caller maps to its display resource (the reference writes the same uchar4 through surf2Dwrite,
// adaptive_cuda_kernels.cu:846-851).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../../include/adanerf_b200.h"
#include "../../../include/adanerf_b200_views.h"

// The viewer's own types that appear in ImageGenerator::inference's parameter list (include/featureset.h:25,
// include/encoding.h:10).  The replacement never looks inside them -- the features and encodings of the hot path live in
// the CUDA kernels behind the C ABI -- so forward declarations are all it needs; in the viewer build they resolve to the
// viewer's classes and NeuralRenderer::render (neuralrenderer.cpp:158-160) compiles unchanged.
class FeatureSet;
class Encoding;

namespace adn_host {

// Counterpart of Config (config.cpp:270-344): what the export directory says.
struct Config {
  adn_scene scene{};
  float adaptiveSamplingThreshold = 0.f;
  int numRaymarchSamples = 0;
  std::string model_dir;
  bool one_network = false;            // a NeRF export with no sampling net (rayMarchSampler = [LinearlySpacedZNearZFar])
  bool load(const std::string& dir);   // parses config.ini + dataset_info.txt + model{0,1}.onnx headers
};

// Counterpart of Camera (camera.cpp:26-94): position + yaw/pitch fly camera producing the 3x3 rotation
// the feature kernels consume (row-major, columns = right / up / -forward in world space).
struct Camera {
  float pos[3] = {0, 0, 0};
  float yaw = 0.f, pitch = 0.f;
  int width = 800, height = 800;
  void rotation(float rot[9]) const;
};

class ImageGenerator {
 public:
  ImageGenerator() = default;
  ~ImageGenerator();
  ImageGenerator(const ImageGenerator&) = delete;
  ImageGenerator& operator=(const ImageGenerator&) = delete;

  // ImageGenerator::load (imagegenerator.cpp:203-245): builds the device context and packs both networks.
  bool load(const Config& config, int device = 0);

  // ImageGenerator::inference (imagegenerator.cpp:247-478): renders the camera's frame.  `batch_size` is
  // the rays-per-batch knob of the viewer (-bs); `num_samples` = K.  d_rgba8: device buffer [W*H] uchar4.
  bool inference(const Camera& camera, uint8_t* d_rgba8, int batch_size, int num_samples, void* stream = nullptr);
  // The reference's parameter list, verbatim (include/imagegenerator.h:61-62; called from neuralrenderer.cpp:158-160):
  // `output_surf` is the cudaSurfaceObject_t of the GL-registered render buffer (buffermanager.h:34) and receives uchar4
  // pixels through surf2Dwrite (adaptive_cuda_kernels.cu:846-851); the feature-set / encoding vectors are accepted and
  // ignored.
  bool inference(Camera& camera, unsigned long long /*cudaSurfaceObject_t*/ output_surf, int batch_size, int num_samples,
                 std::vector<::FeatureSet*>& feature_sets, std::vector<::Encoding>& encodings);
  // Same into a host fp32 buffer [W*H*3] (copies inside).
  bool inference_host(const Camera& camera, float* h_rgb, int batch_size, int num_samples, int32_t* h_nsamples = nullptr);
  // Several cameras in one call (adn_render_views_camera): n_views frames of the cameras' common size (1-64 views, e.g. the
  // two eyes of a head-mounted display) under one sample budget.  d_rgb: device buffer [n_views*H*W*3] fp32, view-major;
  // d_nsamples (may be null): [n_views*H*W].
  bool inference_views(const Camera* cameras, int n_views, float* d_rgb, int batch_size, int num_samples,
                       int32_t* d_nsamples = nullptr, void* stream = nullptr);

  // Frame-cost control (adn_set_option "sample_budget"): at most `max_samples` samples per inference call, the config's
  // adaptiveSamplingThreshold being the floor; 0 = off.  last_threshold(): the threshold the last frame used (synchronises).
  bool set_sample_budget(int64_t max_samples);
  bool last_threshold(float* thr);

  // ImageGenerator::switchRenderOracle (include/imagegenerator.h:69, the viewer's `O` key): toggles the render-oracle view.
  // While it is on, every inference overload draws the sampling network's view (adn_set_option "sampling_view") instead
  // of the rendered frame.
  void switchRenderOracle() { render_oracle_ = !render_oracle_; }
  bool renderOracle() const { return render_oracle_; }

  const char* last_error() const;
  bool stats(adn_stats* out);
  // The loaded network's shape (adn_net_shape): depth, width and skip layer (-1 = none).
  bool net_shape(int net_id, int* depth, int* width, int* skip);
  // The sampling net's depth cells D (multiDepthFeatures, adn_net_dims' outputs of net 0); 0 when there is none.
  int depth_cells();

 private:
  // the per-frame options every inference overload applies before it renders: rays per batch and the render-oracle view
  bool apply_options(int batch_size);

  adn_ctx* ctx_ = nullptr;
  float thr_ = 0.f;
  bool render_oracle_ = false;
  std::string err_;
};

}  // namespace adn_host
