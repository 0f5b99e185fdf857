// Loader for the reference's export directory {config.ini, dataset_info.txt, model0.onnx, model1.onnx}
// (writer: src/export.py:28-93, src/train_data.py:180-195; reader in the viewer: config.cpp:200-344,
// imagegenerator.cpp:92-147).  Pure C++: a key=value parser and a protobuf wire-format walker that
// pulls the fp32 initialisers out of the ONNX files by name (no TensorRT / onnx libraries needed).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/adanerf_b200.h"

namespace adn {

struct NamedTensor {
  std::string name;
  std::vector<float> data;
  int64_t rows = 0, cols = 0;
};

struct ExportDir {
  adn_scene scene{};
  float threshold = 0.0f;  // adaptiveSamplingThreshold
  int num_samples = 0;     // numRaymarchSamples[1]
  int sampler = 0;         // rayMarchSampler[1]: 0 = FromClassifiedDepthAdaptive(NoDepthRange), 1 = FromClassifiedDepth;
                           // 2 = a one-network export, rayMarchSampler = [LinearlySpacedZNearZFar(NoDepthRange)]
  int pdf_transform = 0;   // sampler 1: 1 = sigmoid, 2 = softmax (from losses[0])
  int depth_cells = 128;   // multiDepthFeatures: the sampling net's output width D (32, 64, 128 or 256)
  std::vector<NamedTensor> nets[2];   // sampler 2: nets[0] empty, model0.onnx in nets[1]
};

bool read_onnx_initializers(const std::string& path, std::vector<NamedTensor>& out, std::string& err);
bool load_export_dir(const std::string& dir, ExportDir& out, std::string& err);

// The sampling net of model0.onnx has ex.depth_cells outputs (multiDepthFeatures); a loader that builds the networks
// checks this after load_export_dir.  False: err says why.
bool check_depth_cells(const ExportDir& ex, std::string& err);

}  // namespace adn
