// Information-weighted multi-scale SSIM (IW-SSIM, Wang & Li 2011) of two images on the device: the metric src/evaluate.py:81-88
// reports as "ssim" through src/util/IW_SSIM_PyTorch.py with its default parameters (adn_image_iwssim).
#pragma once
#include <cuda_runtime.h>

#include <cstddef>

namespace adn {

constexpr int kIwNsc = 5;            // scales: a Laplacian pyramid of height 5
constexpr int kIwMinSize = 161;      // the coarsest band, ceil(n / 16), must hold one 11 x 11 window
constexpr int kIwMaxN = 10;          // neighbourhood vector: 3 x 3 neighbours plus the parent (scales 1-3)

// Input layouts of adn_image_iwssim (ADN_IWSSIM_GRAY / ADN_IWSSIM_EVALUATE_RGB).
enum IwLayout { kIwGray = 0, kIwEvaluateRgb = 1 };

// Everything a call's launches need, derived on the host from the metric image's rows x cols: level sizes, offsets into
// the scratch buffer and the blocks of each batched launch.
struct IwPlan {
  int rows[kIwNsc], cols[kIwNsc];    // level l is ceil(rows / 2^l) x ceil(cols / 2^l)
  size_t lvl_off[kIwNsc];            // element offset of level l within one image's levels (all levels of one image, then the other)
  size_t lvl_total;                  // elements of one image's levels
  int band_blk[kIwNsc + 1];          // band launch: first block of each level
  int cov_blk[kIwNsc];               // covariance launch: first block of scales 1-4 (and the end)
  int main_blk[kIwNsc + 1];          // quality / weight launch: first tile of each scale (and the end)
  int main_tx[kIwNsc];               // tiles per row of each scale's cs map
  double gauss[11];                  // the 11-tap Gaussian (sigma 1.5), normalised: the 2-D window is its outer product
  // scratch offsets in bytes
  size_t off_g, off_b, off_cov, off_eig, off_part, off_out, bytes;
};

// The plan for a metric image of rows x cols (both >= kIwMinSize, rows * cols < 2^31).
IwPlan iwssim_plan(int rows, int cols);

// IW-SSIM of d_image (distorted) against d_reference (original), both W x H in `layout`, with the plan for the metric's
// image (rows x cols: H x W for kIwGray, W x H for kIwEvaluateRgb, whose [H*W, 3] buffer the metric views as [W, H]).
// Writes 6 doubles at d_scratch + p.off_out: the score, then wmcs of scales 1..5.  Ten launches; deterministic.
cudaError_t launch_iwssim(const float* d_image, const float* d_reference, int layout, const IwPlan& p, void* d_scratch,
                          cudaStream_t s);

}  // namespace adn
