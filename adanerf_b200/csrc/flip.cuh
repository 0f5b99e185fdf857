// FLIP (Andersson et al., HPG 2020) of two sRGB images on the device: the metric src/evaluate.py:119-161 reports through
// src/util/flip_loss.py, as a per-pixel map and its mean (adn_image_flip).
#pragma once
#include <cuda_runtime.h>

#include <cstddef>

namespace adn {

// Largest filter radius the kernels stage: the CSF radius ceil(3 sqrt(0.04 / (2 pi^2)) ppd) is 28 at ppd 200, the cap.
// (The feature radius ceil(3 * 0.041 ppd) is always the smaller of the two.)
constexpr int kFlipMaxRadius = 28;
constexpr double kFlipMaxPpd = 200.0;
constexpr int kFlipTaps = 2 * kFlipMaxRadius + 1;

// The 1-D filters every 2-D filter of the metric factors into (each in exact arithmetic):
//   A, RG:  the CSF Gaussians of the achromatic and red-green channels, normalised to sum 1, in x and in y;
//   BY1/2:  the two Gaussian terms of the blue-yellow CSF, each normalised to sum 1; the 2-D filter is
//           by_w1 BY1(x)BY1(y) + by_w2 BY2(x)BY2(y);
//   FG:     the feature Gaussian exp(-t^2 / 2 sd^2), normalised to sum 1;
//   EDGE:   -t exp(-t^2 / 2 sd^2), positive taps scaled to sum 1 and negative ones to sum -1 (the sign depends on t only,
//           so the 2-D normalisation of t exp(..) exp(..) factors into this times FG);
//   POINT:  (t^2 / sd^2 - 1) exp(-t^2 / 2 sd^2), normalised like EDGE.
// Tap k of a filter of radius R weighs the pixel at offset k - R (cross-correlation, as conv2d).
enum FlipFilter { kFlipA, kFlipRG, kFlipBY1, kFlipBY2, kFlipFG, kFlipEdge, kFlipPoint, kFlipNumFilters };

struct FlipConsts {
  int r;                  // CSF radius (filters A, RG, BY1, BY2)
  int rf;                 // feature radius (FG, EDGE, POINT)
  float by_w1, by_w2;     // weights of the two blue-yellow terms
  float cmax;             // HyAB^0.7 of Hunt-adjusted pure green against pure blue
  float rgb2xyz[9];       // linear RGB -> XYZ divided by the D65 white (row-major)
  float xyz2rgb[9];       // XYZ divided by the white -> linear RGB
  float w[kFlipNumFilters * kFlipTaps];   // filter f, tap k at w[f * kFlipTaps + k]
};

// Builds the constants in double from pixels_per_degree and rounds each to fp32 once.  Needs 0 < ppd <= kFlipMaxPpd.
void flip_consts(double pixels_per_degree, FlipConsts* out);

// Device scratch launch_flip needs for a W x H pair (the sum, the partial sums and the horizontal-pass planes of both images).
size_t flip_scratch_bytes(int W, int H);

// FLIP of d_a against d_b ([H*W, 3] fp32 each, row-major sRGB): d_map [H*W] (may be NULL) and the sum of the map in double
// at static_cast<double*>(d_scratch)[0] (deterministic).  Three launches: the horizontal passes, the vertical passes with
// everything per pixel, and the final reduction.  Needs W, H >= 1 and W * H < 2^31.
cudaError_t launch_flip(const float* d_a, const float* d_b, int W, int H, const FlipConsts& c, void* d_scratch, float* d_map,
                        cudaStream_t s);

}  // namespace adn
