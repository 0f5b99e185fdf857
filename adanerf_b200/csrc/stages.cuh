// SIMT stages of the AdaNeRF hot path (HBM-bound byte/index work): ray generation, SpherePosDir
// features (stage 0), threshold / top-K / scan compaction (stage 2), positional encoding (stage 3),
// per-ray transmittance scan + composite (stage 5).  Launchers only; kernels in stages.cu.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace adn {

struct SceneDev {
  float c[3];          // view_cell_center (fp32, features.py:759 / :345)
  float r2;            // float(view_cell_radius**2) (features.py:761,786)
  float sqrt_max_depth;  // float(math.sqrt(max_depth)) (nerf_raymarch_common.py:229)
  int n_freq_pos, n_freq_dir;
  int n_freq_pos0, n_freq_dir0;   // sampling-net encoding (10/4 or 2/2)
  int ndc;                        // NDC variant: ndc_rays + no position normalisation (features.py:429-431)
  float ndc_cw, ndc_ch;           // float(-1 / (W / (2 focal))), float(-1 / (H / (2 focal)))
};

struct CameraRays {  // src/util/raygeneration.py:10-26 in double precision
  double start_x, start_y, focal, x_pp, y_pp;
  int W, H, row0;
};

struct PoseDev {
  float pose[3];
  float rot[9];
};

// The cameras of a call over several views, passed to the kernels as a kernel parameter: every launch carries its own copy,
// so nothing is uploaded that a later call could overwrite before the kernel reads it, and no host synchronisation is
// needed.  Rays are view-major: ray g of the call is ray g - v N of view v = g / N.  kMaxViews x 48 B = 3 KB keeps every
// launch's parameters under the 4 KB of the classic kernel-parameter limit.
constexpr int kMaxViews = 64;
struct ViewTable {
  long long ray0;         // the launch's first ray in the call's view-major order (a chunk's offset)
  long long n_per_view;   // N
  PoseDev v[kMaxViews];
};

cudaError_t launch_gen_dirs(const CameraRays& cam, long long n_rays, float* d_dirs, cudaStream_t s);
// Stage 0.  Any of d_x0 (fp32 features), d_ray_o / d_ray_d and d_tiles0 may be null (not written).  d_tiles0: the sampling
// net's packed input tiles (sampling_tiles in tiles.cuh) with tile_terms terms (1 or 2).
// views (may be null): ray i of the launch takes the camera of its view instead of pd; with cam its pixel is its index inside
// the view (cam.row0 must then be 0).
cudaError_t launch_stage0(const SceneDev& sc, const PoseDev& pd, const float* d_dirs, const CameraRays* cam,
                          long long n_rays, float* d_x0, float* d_ray_o, float* d_ray_d, uint8_t* d_tiles0, int tile_terms,
                          cudaStream_t s, const ViewTable* views = nullptr);
// The rays of a render without a sampling net (option "sampler" 2): d_ray_o [N,3] = pose, d_ray_d [N,3] = R d (the FMA
// chain of stage 0), from d_dirs or, when cam is given, the pixels' directions.  d_ray_dirs (may be null): the directions
// whose norm nerf_raw2outputs scales its distances by, R d or on NDC scenes (sc.ndc) ndc_rays' un-normalised direction.
// views: as for launch_stage0.
cudaError_t launch_camera_rays(const SceneDev& sc, const PoseDev& pd, const float* d_dirs, const CameraRays* cam,
                               long long n_rays, float* d_ray_o, float* d_ray_d, float* d_ray_dirs, cudaStream_t s,
                               const ViewTable* views = nullptr);

// Stage 2.  tile_state: [n_ctas + 2] uint64 scratch zeroed by the launcher (memsetAsync).
size_t stage2_scratch_bytes(long long n_rays);
// Host-side bookkeeping of a stage-2 scratch buffer (owned by whoever owns the buffer): launch epoch and ticket base, so
// the tile states / ticket counter need no per-launch memset.
struct Stage2Sync {
  void* scratch = nullptr;
  size_t cleared_bytes = 0;
  uint32_t epoch = 0, ticket_base = 0;
};
// d_thr: when non-null the kernel reads the threshold from this device float (a sample-budget threshold) instead of `thr`.
// D: the depth cells of a raw0 row (multiDepthFeatures: 32, 64, 128 or 256), raw0 [n_rays, D] and d_zlut [D]; 1 <= K <= min(D, 128).
cudaError_t launch_stage2(const float* d_raw0, long long n_rays, float thr, int K, const float* d_zlut, int32_t* d_count,
                          int32_t* d_offset, int32_t* d_cell, int32_t* d_ray, float* d_z, float* d_zp, long long* d_total,
                          void* d_scratch, Stage2Sync* sync, cudaStream_t s, const float* d_thr = nullptr, int D = 128);

// Sample budget: writes to *d_thr the smallest threshold t >= thr_min (> 0) at which stage 2 over raw0 [n_rays, D] with K
// samples per ray yields at most max_samples (>= n_rays) samples in all.  At D = 128 d_raw0 must be 16-byte aligned.
// d_keys: [n_rays * (K - 1)] uint32 scratch; d_work: budget_work_bytes() of scratch.  Stream ordered, no host synchronisation; adds its kernel count to *launches.
//
// group (may be null, or have a null fn): the call is one member of a budget group.  fn is called on the host once per select
// round, after the kernel that filled that round's histogram (2049 uint64 words in round 0: 2048 bins and the ray count,
// 2048 in rounds 1 and 2), and must sum the words in place across all members, ordered on the stream it is given.  Every
// member then selects the t* of all members' rays together (max_samples is the group's budget), and runs all three rounds
// even with no rays or no candidates.  When fn returns non-zero the launcher stops enqueueing and records the status and
// the round; *d_thr is then not written.
struct BudgetGroup {
  int (*fn)(void* user, uint64_t* d_words, int64_t n_words, void* stream) = nullptr;
  void* user = nullptr;
  int status = 0;          // fn's last return value
  int failed_round = -1;   // the round whose reduction failed, -1 = none
};
size_t budget_work_bytes();
cudaError_t launch_budget_threshold(const float* d_raw0, long long n_rays, float thr_min, int K, long long max_samples,
                                    uint32_t* d_keys, void* d_work, float* d_thr, int num_sms, cudaStream_t s, int* launches,
                                    BudgetGroup* group = nullptr, int D = 128);
// Dense (thr == 0): count = K, offset = ray*K, total = N*K; no index arrays are materialised.
cudaError_t launch_stage2_dense(long long n_rays, int K, int32_t* d_count, int32_t* d_offset, long long* d_total,
                                cudaStream_t s);
// Linear placement (option "sampler" 2, LinearlySpacedZNearZFar): every ray takes the K depths d_zt [K].  Writes the layout
// of launch_pdf_sample: count = K, offset = r K, ray [N K] = r, z [N K] and *d_total = N K; d_count, d_offset, d_ray and
// d_total may be null (not written).  N K < 2^31.
cudaError_t launch_linear_sample(long long n_rays, int K, const float* d_zt, int32_t* d_count, int32_t* d_offset, int32_t* d_ray,
                                 float* d_z, long long* d_total, cudaStream_t s);

// Fixed-K sampler (rayMarchSampler FromClassifiedDepth, the DONeRF baseline): per ray the inverse CDF of the transformed
// raw0 [n_rays, 128] at K + 2 evenly spaced u, the first and last dropped, warped to world depth.  transform: 1 = sigmoid,
// 2 = softmax.  Writes count = K, offset = r K, ray [N K] = r, z [N K] (ascending per ray) and *d_total = N K; any of
// d_count, d_offset, d_ray, d_total may be null (not written).  wbase = depth_range[1] - depth_range[0] + 1 (double),
// dr_min = depth_range[0]: LogTransform.to_world as the z table of the adaptive path computes it.
constexpr int kPdfSigmoid = 1, kPdfSoftmax = 2;
cudaError_t launch_pdf_sample(const float* d_raw0, long long n_rays, int K, int transform, double wbase, float dr_min,
                              int32_t* d_count, int32_t* d_offset, int32_t* d_ray, float* d_z, long long* d_total, cudaStream_t s);

// The sampling network's view (the viewer's render-oracle mode): raw0 [n_rays, 128] (16-byte aligned) -> per ray the three
// cells that lead raw0's stable descending radix order, as (c + 0.5) / 128 into d_rgb [n_rays, 3] and as uchar4 pixels
// (value * 255 truncated, alpha 255) into d_rgba8 [n_rays]; either output may be null.
cudaError_t launch_sampling_view(const float* d_raw0, long long n_rays, float* d_rgb, uint8_t* d_rgba8, cudaStream_t s);

// Stage 3.  Adaptive: sample s -> (d_ray[s], d_z[s]).  Dense (d_ray == nullptr): ray = s / K,
// z = d_zlut_dense[s % K].  n_samples read from d_total when non-null.  d_x1 (fp32 features) and d_tiles1 (the shading
// net's packed input tiles, shading_tiles in tiles.cuh) may be null (not written).
cudaError_t launch_stage3(const SceneDev& sc, const float* d_ray_o, const float* d_ray_d, const int32_t* d_ray,
                          const float* d_z, const float* d_zlut_dense, int K, long long n_samples, const long long* d_total,
                          float* d_x1, uint8_t* d_tiles1, int num_sms, cudaStream_t s);

// Optional per-ray / per-slot outputs of the composite (adaptive_raw2outputs' other return values and the tensors
// RayMarchFromPoses.postprocess puts into the inference dict, src/features.py:536-577).  Any pointer may be null.
struct Stage5Aux {
  float* weights = nullptr;     // [N,K] zero padded (NeRFWeightsOutput)
  float* alpha = nullptr;       // [N,K] zero padded, sigmoid(a) * zp (NeRFAlphaOutput)
  float* z_vals = nullptr;      // [N,K] world depth, NaN padded and NaN at z == +-0 unless dense (NeRFInputFeatureZVals)
  float* depth_map = nullptr;   // [N] sum w z
  float* acc_map = nullptr;     // [N] sum w
  float* disp_map = nullptr;    // [N] 1 / torch.max(1e-10, depth_map / acc_map), NaN when the quotient is
  float* depth_est = nullptr;   // [N] LogTransform.from_world(depth_map, depth_range) (NeRFOutputDepth)
  int linear_depth = 0;         // NDC: depth_est = depth_map (features.py:573-574)
  float dr_min = 0.0f;          // depth_range[0]
  float log_range = 1.0f;       // float(log(depth_range[1] - depth_range[0] + 1))
  bool any() const { return weights || alpha || z_vals || depth_map || acc_map || disp_map || depth_est; }
};

// Stage 5.  zp: adaptive -> packed [M]; dense -> raw0 [N, K] (K = D, one sample per depth cell).
// d_ray_d non-null: the density composite of the fixed-K sampler (nerf_raw2outputs, src/nerf_raymarch_common.py:19-68)
// over K samples per ray at offset r K: alpha = 1 - exp(-relu(a) dist), dist = (z[k+1] - z[k], last 1e10) * |ray_d [N,3]|;
// d_zp, d_offset, d_count and dense are not read, and z_vals is z unchanged.
cudaError_t launch_stage5(const float* d_raw1, const float* d_zp, const float* d_z, const float* d_zlut_dense,
                          const int32_t* d_offset, const int32_t* d_count, long long n_rays, int K, int dense,
                          float* d_rgb, uint8_t* d_rgba8, const Stage5Aux& aux, cudaStream_t s, const float* d_ray_d = nullptr);

// Linear RGBA8 pixels [rows * W] -> surf2Dwrite(uchar4, surface, 4 x, row0 + y) (adaptive_cuda_kernels.cu:846-851).
cudaError_t launch_rgba_to_surface(const uint8_t* d_rgba8, int W, int row0, int rows, unsigned long long surface, cudaStream_t s);

// Image metric (src/evaluate.py:49-54): sum over all values of (a - b)^2 in double, deterministic two-stage
// reduction.  d_partials: kMetricBlocks doubles of scratch; d_sum receives the total.  clamp01: clip `a` to [0,1] first
// (what the reference does to an image before it is written / compared as 8-bit, src/evaluate.py:257-258).
constexpr int kMetricBlocks = 592;
cudaError_t launch_image_sqdiff(const float* d_a, const float* d_b, long long n_values, int clamp01, double* d_partials,
                                double* d_sum, cudaStream_t s);

}  // namespace adn
