/*
 * adanerf_b200 -- C ABI of the H100-native AdaNeRF inference renderer (libadanerf_b200.so).
 *
 * One data-parallel hot path, hand-written for sm_90a:
 *   rays -> SpherePosDir features -> sampling MLP (wgmma, bf16x3 split precision)
 *        -> threshold / top-K / scan compaction -> positional encoding
 *        -> shading MLP (wgmma, bf16) -> per-ray transmittance scan + alpha composite.
 *
 * Each entry point cites the reference interface (relative to thomasneff/AdaNeRF) it replaces.
 * Conventions: plain pointers and sizes only; integer status codes (0 = ok), never exceptions;
 * "d_" pointers are device memory owned by the caller, "h_" pointers are host memory; the context
 * owns packed weights and scratch; work is stream ordered (`stream` is a cudaStream_t passed as
 * void*, NULL = legacy default stream); no host synchronisation inside unless stated; one context
 * per device; a context is not thread safe.  There is NO CPU fallback: every call fails with
 * ADN_ERR_CUDA / ADN_ERR_NO_DEVICE when no sm_90 device is usable.
 * Order across streams: the calls on one context execute in the order they were issued, whatever
 * stream each names (the *_host entries run on a stream of the context's own): every call that
 * enqueues work waits for the previous call's work and records an event after its own, since all
 * calls share the context's scratch.  The caller still orders its own kernels against a call's
 * outputs (on the call's stream, or with an event recorded there).  A call on a stream that is
 * capturing a CUDA graph fails with ADN_ERR_INVALID before it enqueues anything: stage 2's launch
 * epoch and ticket base are host state that a replayed graph would not update.
 */
#ifndef ADANERF_B200_H
#define ADANERF_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct adn_ctx adn_ctx;
typedef int adn_status;

enum {
  ADN_OK = 0,
  ADN_ERR_INVALID = 1,      /* bad argument / unsupported shape */
  ADN_ERR_CUDA = 2,         /* CUDA runtime error (see adn_last_error) */
  ADN_ERR_NO_DEVICE = 3,    /* no CUDA device / not compute capability 9.x (Hopper) */
  ADN_ERR_NO_WEIGHTS = 4,   /* render called before both nets were set */
  ADN_ERR_IO = 5,           /* export directory / file problems */
  ADN_ERR_KERNEL = 6        /* device-side watchdog tripped (mbarrier timeout) */
};

/* Scene constants.  Source: the export's dataset_info.txt written by src/export.py:47-54
 * (view_cell_center, view_cell_size, depth_range = WARPED range, fov, max_depth) and the feature
 * set constructors src/features.py:286-287 (zNear/zFar), :326-339 (posEnc / posEncArgs). */
typedef struct adn_scene {
  float view_cell_center[3];
  float view_cell_size[3];
  float depth_range[2];
  float max_depth;
  float fov;            /* radians; focal = 0.5*W/tan(fov/2)  (src/datasets.py:181-182) */
  float z_near, z_far;  /* 0.001, 1.0 */
  /* Shading-net encoding, posEnc[1] / posEncArgs[1] (default "10-4"): position and direction band counts P <= 20, D <= 10;
   * the net reads 3 + 6 P position and 3 + 6 D direction columns.  Negative: posEnc none, the 3-column identity (the
   * reference's -1, src/features.py:326-328), the same as 0 bands. */
  int32_t n_freq_pos;
  int32_t n_freq_dir;
  /* Sampling-net encoding, posEnc[0] / posEncArgs[0], 6 + 6 (P0 + D0) input columns, P0 + D0 <= 20: 0 = the shading
   * net's field above (e.g. "10-4", 90 features), negative = 0 bands or posEnc none, positive = that count (e.g. 2/2,
   * "2-2", 30 features, configs/fine_training_ndc.ini:8).  Outside these limits adn_create returns ADN_ERR_INVALID. */
  int32_t n_freq_pos0, n_freq_dir0;
  /* NDC / LLFF variant (configs/fine_training_ndc.ini: useNDC, FromClassifiedDepthAdaptiveNoDepthRange,
   * rayMarchNormalization[1] = None): rays go through ndc_rays(H, W, focal, near = 1)
   * (src/nerf_raymarch_common.py:71-88, src/features.py:429-431), sample depths are the cell centres in [0,1]
   * (no depth-range warp), positions are not normalised, NeRFOutputDepth is the depth map itself.
   * ndc_w / ndc_h: the dataset's image size (features.py:350-351); ndc_focal <= 0 -> 0.5 * ndc_w / tan(fov / 2). */
  int32_t use_ndc;
  int32_t ndc_w, ndc_h;
  float ndc_focal;
} adn_scene;

/* One named parameter tensor, fp32, row-major [rows, cols] ([out, in] for weights, [out, 1] or
 * [1, out] for biases), with the reference's state_dict names: `layers.{i}.weight|bias` for the
 * sampling net (src/models.py:71-76), `pts_linears.{i}`, `views_linears.0`, `feature_linear`,
 * `alpha_linear`, `rgb_linear` for the shading net (src/models.py:226-244). */
typedef struct adn_tensor_desc {
  const char* name;
  const float* data;    /* host pointer */
  int64_t rows, cols;
} adn_tensor_desc;

typedef struct adn_stats {
  int64_t n_rays;          /* rays of the last render call */
  int64_t n_samples;       /* M = surviving samples of the last render call (valid after a sync) */
  float ms_stage[6];       /* device ms of stages 0..5 of the last *profiled* render (adn_set_option "profile"=1) */
  int64_t kernel_launches; /* kernels launched by this context so far */
} adn_stats;

/* ---- lifetime --------------------------------------------------------------------------- */
/* Replaces ImageGenerator::ImageGenerator + FeatureSet::create (imagegenerator.cpp:84-201,
 * featureset.cpp:67-137) and TrainConfig.initialize's feature setup (src/train_data.py:63-239). */
adn_status adn_create(adn_ctx** out, const adn_scene* scene, int device);
void adn_destroy(adn_ctx* ctx);
const char* adn_strerror(adn_status s);
const char* adn_last_error(const adn_ctx* ctx);
const char* adn_version(void);

/* net_id 0 = sampling net (BaseNet, src/models.py:18-195), 1 = shading net (NeRF, :199-277).
 * Packs the fp32 parameters into the kernels' layout (bf16 hi/lo split, swizzled K-major tiles).
 * Replaces load_state_dict / ImageGenerator::initEngine's ONNX->TensorRT build.
 * The network's shape (the reference's `layers`, `layerWidth`, `skips`) is read from the tensor shapes:
 *   sampling net: layers.0 .. layers.{D-1}, D = 1-12, at most 128 inputs, hidden width W = 128 or 256 in every hidden
 *     layer, D = 32, 64, 128 or 256 outputs: the depth cells the net classifies (multiDepthFeatures); no skips.  32 and
 *     64 outputs are padded to the kernel's 128 rows with zero weights; every raw0 the ABI exposes is [N, D].
 *   shading net: the scene's encoding, P = 3 + 6 n_freq_pos and V = 3 + 6 n_freq_dir columns (63 and 27 for posEnc
 *     10-4): pts_linears.0 reads P columns, views_linears.0 reads W + V; D = 1-10 pts_linears, W = 128 or 256, view
 *     branch W/2; no skip, or one skip after layer i in [0, D-2], which shows as pts_linears.{i+1} reading W + P columns
 *     (the reference's skips = auto is a skip at 4 for D >= 6 and none for D <= 4).
 *   The sampling net must read the 6 + 6 (n_freq_pos0 + n_freq_dir0) columns of the scene's encoding to render.
 * Any other shape fails with ADN_ERR_INVALID and adn_last_error names the offending tensor and, for the shading net, the
 * column count the scene's encoding expects. */
adn_status adn_set_weights(adn_ctx* ctx, int net_id, const adn_tensor_desc* tensors, int n_tensors);

/* The shape adn_set_weights inferred: depth D, width W (of a one-layer sampling net: its output width) and the skip layer
 * (-1 = none; always -1 for the sampling net). */
adn_status adn_net_shape(adn_ctx* ctx, int net_id, int* depth, int* width, int* skip);

/* Loads {config.ini, dataset_info.txt, model0.onnx, model1.onnx} as written by src/export.py:28-93
 * (the directory the C++ viewer takes with -mp, adanerf_real_time_viewer/README.md:38-43).
 * Creates the context with the scene from dataset_info.txt; threshold / K from config.ini are
 * returned through thr_out / k_out (may be NULL).  A config.ini with rayMarchSampler = [.., FromClassifiedDepth] (the
 * DONeRF sampler; with InverseSqrtDistCentered and log, not NDC) sets options "sampler" = 1 and "pdf_transform" from
 * losses[0]: BCEWithLogitsLoss -> 1, CrossEntropyLoss / CrossEntropyLossWeighted -> 2; any other loss is refused.
 * multiDepthFeatures = [D, D] (missing: 128) must hold two equal entries from {32, 64, 128, 256}, and model0.onnx's last
 * layer must have D rows; otherwise ADN_ERR_IO. */
adn_status adn_create_from_export_dir(adn_ctx** out, const char* dir, int device, float* thr_out, int* k_out);

/* Host-only (no GPU needed): parses the export directory like adn_create_from_export_dir and returns the
 * scene, threshold, K and the number of fp32 tensors found in model0.onnx / model1.onnx.  It does not report the
 * sampler: callers that need it read rayMarchSampler / losses from config.ini themselves.  It checks multiDepthFeatures
 * itself (two equal entries from {32, 64, 128, 256}) but not against model0.onnx's output rows: it builds no network, and
 * reads directories whose initialisers are cut down (e.g. to one row each) to save space.  The loaders that build the
 * networks check that too.  Replaces Config::load + Config::loadDatasetInfo
 * (adanerf_real_time_viewer/src/config.cpp:270-344). */
adn_status adn_probe_export_dir(const char* dir, adn_scene* scene_out, float* thr_out, int* k_out, int* n_tensors_out /*[2]*/);

/* name: "chunk_rays" (rays per internal batch, 0 = auto), "profile" (0/1 per-stage event timing),
 * "mlp0_terms" (3 = bf16x3 split precision [default], 1 = plain bf16; parity experiments only),
 * "fuse_encoder" (1 = positional encoding of the samples inside the shading kernel, a tile ahead of its MLP: no
 *   [M, P + V]-sized tile buffer and no separate stage-3 launch [default]; NDC scenes always take the separate kernel;
 *   0 = separate kernel; both render the same bits),
 * "sample_budget" (B > 0 = every adaptive render -- rays, aux, camera, rgba8, surface, *_host -- takes its `thr` as a floor
 *   and renders with the smallest threshold t* >= thr whose total sample count M over the whole call is <= B, chosen on
 *   the device with no host synchronisation; the picture is exactly that of a fixed-threshold call at t*.  Fails with
 *   ADN_ERR_INVALID in dense mode (thr == 0) and when B < n_rays.  The stage-2 slot of ms_stage includes the selection.
 *   Calls of more than one chunk keep raw0 and the ray origins / directions of the whole call (536 B per ray: the caller's
 *   d_oracle_weights when given, else context scratch).  0 = off [default]).
 *   The frame cost follows M, so B is a frame-time knob.  Row bands of one frame share one t* and one B through a budget
 *   group (adn_set_budget_group below); without one each call chooses its own.
 * "sampling_view" (1 = every render -- rays, aux, camera, rgba8, surface, *_host -- draws the sampling network's view, the
 *   C++ viewer's render-oracle mode behind ImageGenerator::switchRenderOracle (imagegenerator.cpp:316-326): stage 0 and the
 *   sampling MLP run, then per ray the three depth cells c0, c1, c2 that lead the sampling net's output in descending order
 *   are drawn as (c + 0.5) / 128 into rgb, and as uchar4 (value * 255 truncated, alpha 255) into the RGBA8 / surface
 *   pixels (samplesToImage, base_cuda_kernels.cu:487-528; see adn_sampling_view for the order); stages 2-5 do not run.
 *   In this mode `thr` / `K` are validated as before but not used; d_oracle_weights still receives raw0 (its rows must be
 *   16-byte aligned); d_nsamples receives 0 for every ray; non-NULL auxiliary outputs fail with ADN_ERR_INVALID;
 *   "sample_budget" is not applied (no selection runs, a budget group makes no reductions, adn_last_threshold returns
 *   `thr`); adn_get_stats reports n_samples = 0 and, profiled, stages 0-1 in ms_stage[0..1], the view in ms_stage[5] and 0
 *   in ms_stage[2..4].  0 = off [default]: renders are exactly as without the option),
 * "sampler" (0 = FromClassifiedDepthAdaptive, the threshold / top-K sampler and sigmoid(a) * zp composite [default];
 *   1 = FromClassifiedDepth, the DONeRF sampler (src/nerf_raymarch_common.py:606-660): every render -- rays, aux, camera,
 *   rgba8, surface, *_host, chunked or not -- places exactly K samples per ray by the inverse CDF of
 *   pdf_transform(raw0) (nerf_sample_pdf, det = True, :160-192) and composites them with nerf_raw2outputs (:19-68):
 *   alpha = 1 - exp(-relu(a) dist), dist = (z[k+1] - z[k], last 1e10) * |rays_d|.  `thr` is ignored; 1 <= K <= 128;
 *   d_nsamples receives K for every ray; z_vals is never NaN; "sample_budget" > 0 and NDC scenes fail with
 *   ADN_ERR_INVALID; "sampling_view" works as in the adaptive mode (it reads raw0 only);
 *   2 = LinearlySpacedZNearZFar, NeRF with no sampling network (src/features.py:417-479,564-577): only the shading slot
 *   (adn_set_weights net 1, pts_linears.*) is used.  It is a one-network context: setting sampler 2 fails with
 *   ADN_ERR_INVALID while the sampling slot holds a network (the shading net of a two-network run is not a NeRF of its
 *   own), and adn_set_weights(ctx, 0, ...) fails while sampler is 2.  Every render entry -- rays, aux, camera, rgba8, surface, *_host,
 *   chunked or not -- starts the rays at the camera, rays_o = pose and rays_d = R dir (not renormalised; on NDC scenes
 *   ndc_rays follows), places the same K depths on every ray, z = z_near (1 - t) + z_far t with t = linspace(0, 1, K + 1)[k] +
 *   0.5 / K, warped by LogTransform.to_world with the scene's depth_range (NDC scenes: not warped; adn_linear_depths), and
 *   composites them with nerf_raw2outputs as sampler 1 does (on NDC scenes |rays_d| is that of ndc_rays' direction).
 *   `thr` is ignored; 1 <= K <= 128 and N K < 2^31 per chunk; d_nsamples receives K for every ray; z_vals is never NaN;
 *   d_oracle_weights must be NULL; "sample_budget" > 0 and "sampling_view" fail with ADN_ERR_INVALID.  Profiled,
 *   adn_get_stats reports the rays in ms_stage[0], 0 in ms_stage[1], the placement in ms_stage[2], the encoding (when not
 *   fused) in ms_stage[3], the shading MLP in ms_stage[4] and the composite in ms_stage[5]),
 * "pdf_transform" (what sampler 1 applies to raw0 before the inverse CDF, chosen by losses[0] of the training config:
 *   1 = sigmoid (BCEWithLogitsLoss) [default], 2 = softmax (CrossEntropyLoss, CrossEntropyLossWeighted).  0, the
 *   reference's "no transform", fails with ADN_ERR_INVALID: raw0 then gives a non-monotone cdf, whose sample placement
 *   would depend on the internals of ATen's binary search). */
adn_status adn_set_option(adn_ctx* ctx, const char* name, int64_t value);

/* Budget group: several contexts (one per row band, on one device or several) whose budgeted calls choose ONE threshold, the
 * t* a single context would choose over all their rays together, under ONE budget B.  The threshold selection is an exact
 * radix select over integer histograms, so it is enough that every member sums its histograms with the others' before each
 * of its three select rounds.  The context calls `fn` on the host, from the thread that makes the call, while it enqueues:
 * once per round (after the candidate extraction, then after each histogram kernel).  `fn` must add d_words[0 .. n_words)
 * (uint64 device memory; 2049 words in round 0 -- 2048 bins and the member's ray count --, 2048 in rounds 1 and 2) in place
 * across all members, ordered on `stream` (the call's stream, a cudaStream_t; NULL = legacy default stream), and return 0,
 * e.g. ncclAllReduce(d_words, d_words, n_words, ncclUint64, ncclSum, comm, stream).  Counts stay below 2^63, so a signed
 * 64-bit sum gives the same words.  Q = B - sum N is formed on the device, 0 when sum N > B.
 * Every budgeted call honours the group -- rays, aux, camera, rgba8, surface, *_host -- and so does adn_budget_threshold.
 * A budgeted call with no rays still runs the selection and every reduction (it renders nothing and may pass NULL outputs).
 * Contract between the members:
 *   - every member makes the same sequence of budgeted calls, with the same `thr`, `K` and sample budget B, and the same
 *     value of option "sampling_view" (a member drawing the view makes no reductions);
 *   - checks that can differ between members (B >= the rays of all members, the 2^32 - 1 candidate limit over all
 *     members, dense mode) are made by the caller before any member enqueues: a member refuses a call before its first
 *     reduction only for what it can see itself;
 *   - a member whose call fails before its first reduction leaves the others waiting in theirs.
 * A non-zero return from `fn` fails the call with ADN_ERR_CUDA (adn_last_error names the round) and nothing more of it is
 * enqueued; the context stays usable.  fn = NULL leaves the group: calls choose their own threshold again. */
typedef int (*adn_budget_reduce_fn)(void* user, uint64_t* d_words, int64_t n_words, void* stream);
adn_status adn_set_budget_group(adn_ctx* ctx, adn_budget_reduce_fn fn, void* user);
adn_status adn_get_stats(adn_ctx* ctx, adn_stats* out);   /* synchronises the context's stream */
/* The threshold the last render call used: t* under "sample_budget", else its `thr` argument.  Synchronises like
 * adn_get_stats. */
adn_status adn_last_threshold(adn_ctx* ctx, float* thr_out);

/* ---- the hot path ----------------------------------------------------------------------- */
/* render(rays, sampling_net, shading_net, adaptiveSamplingThreshold): one call = what
 * TrainConfig.inference(batch, gradient=False, is_inference=True) computes (src/train_data.py:278-299):
 *   d_dirs  [N,3] camera-space pixel directions (DatasetKeyConstants.ray_directions_samples)
 *   pose[3], rot[9] (row-major 3x3) HOST pointers (ImagePose / ImageRotation)
 *   thr = adaptiveSamplingThreshold (0 = dense K samples, K must then be D), K = numRaymarchSamples[1], 1 <= K <= min(D, 128)
 *   (D = the sampling net's depth cells; D != 128 renders only with option "sampler" 0 and without "sampling_view")
 *   d_rgb [N,3] fp32 (outs[-1][:, :3]); d_nsamples [N] int32 or NULL (AdaptiveSamplePositions * K);
 *   d_oracle_weights [N,D] fp32 or NULL (dicts[1]["OracleWeights"], i.e. raw sampling-net output). */
adn_status adn_render_rays(adn_ctx* ctx, const float* pose, const float* rot, const float* d_dirs, int64_t n_rays,
                           float thr, int K, float* d_rgb, int32_t* d_nsamples, float* d_oracle_weights,
                           void* stream);

/* Auxiliary outputs of the same call: the other return values of adaptive_raw2outputs
 * (src/nerf_raymarch_common.py:137-144) and the tensors RayMarchFromPoses.postprocess stores in the inference dict
 * (src/features.py:536-577), read by plots.render_all_imgs / the depth export (src/plots.py:272-306).
 * Every pointer is a device pointer and may be NULL; [N,K] tensors are padded like the reference's. */
typedef struct adn_aux_outputs {
  float* d_weights;    /* [N,K] "NeRFWeightsOutput": alpha * transmittance, 0 in unused slots */
  float* d_alpha;      /* [N,K] "NeRFAlphaOutput": sigmoid(raw alpha) * sampling-net value, 0 in unused slots */
  float* d_z_vals;     /* [N,K] "NeRFInputFeatureZVals": world depth of the samples, NaN in unused slots and, as in the
                          reference's adaptive path, at samples with z == +-0 (dense mode keeps 0) */
  float* d_depth_map;  /* [N] sum_k w z (world depth) */
  float* d_acc_map;    /* [N] sum_k w */
  float* d_disp_map;   /* [N] 1 / torch.max(1e-10, depth_map / acc_map): NaN when the quotient is (0 / 0 at acc == 0) */
  float* d_depth_est;  /* [N] "NeRFOutputDepth": LogTransform.from_world(depth_map, depth_range) */
} adn_aux_outputs;
adn_status adn_render_rays_aux(adn_ctx* ctx, const float* pose, const float* rot, const float* d_dirs, int64_t n_rays,
                               float thr, int K, float* d_rgb, int32_t* d_nsamples, float* d_oracle_weights,
                               const adn_aux_outputs* aux, void* stream);

/* Same, generating the pinhole rays of image rows [row0, row0+rows) of a WxH frame on the device
 * (src/util/raygeneration.py:10-26; ray id = y*W + x).  Replaces Camera::UpdateFeaturesBatch +
 * ImageGenerator::inference's batch loop (camera.cpp:160-201, imagegenerator.cpp:247-478).
 * d_rgb [rows*W,3].  This is the multi-GPU tile entry: each rank renders its row band. */
adn_status adn_render_camera(adn_ctx* ctx, const float* pose, const float* rot, int W, int H, int row0, int rows,
                             float thr, int K, float* d_rgb, int32_t* d_nsamples, void* stream);

/* Viewer output format: RGBA8 (adaptive_cuda_kernels.cu:846-851 writes uchar4 through surf2Dwrite);
 * d_rgba8 is a linear [rows*W] uchar4 buffer the caller copies/maps to its GL resource. */
adn_status adn_render_camera_rgba8(adn_ctx* ctx, const float* pose, const float* rot, int W, int H, int row0, int rows,
                                   float thr, int K, uint8_t* d_rgba8, void* stream);

/* The viewer's own output target: a cudaSurfaceObject_t bound to the GL-registered cudaArray of the current render buffer
 * (adanerf_real_time_viewer/src/interoprenderbuffer.cpp:53-83); uchar4 pixels written with surf2Dwrite at (x, row0 + y)
 * exactly like adaptive_cuda_kernels.cu:846-851.  `surface` is the cudaSurfaceObject_t value (an unsigned 64-bit handle;
 * the header stays free of CUDA types). */
adn_status adn_render_camera_surface(adn_ctx* ctx, const float* pose, const float* rot, int W, int H, int row0, int rows,
                                     float thr, int K, unsigned long long surface, void* stream);

/* End-to-end variants with HOST buffers: H2D of the inputs and D2H of the results happen inside the
 * call and the call returns after the results are on the host.  Buffers the caller registered (below) or allocated
 * page-locked itself are the source / target of the DMA; anything else goes through pinned staging owned by the
 * context (one extra host copy each way). */
adn_status adn_render_rays_host(adn_ctx* ctx, const float* pose, const float* rot, const float* h_dirs, int64_t n_rays,
                                float thr, int K, float* h_rgb, int32_t* h_nsamples);
adn_status adn_render_camera_host(adn_ctx* ctx, const float* pose, const float* rot, int W, int H, int row0, int rows,
                                  float thr, int K, float* h_rgb, int32_t* h_nsamples);

/* Page-locks [p, p + bytes) in place (cudaHostRegister) for the *_host entry points.  The caller owns the memory and must
 * keep it allocated until adn_unregister_host_buffer / adn_destroy: the library never registers memory on its own (a
 * buffer freed and re-allocated at the same address would keep a stale registration).  The viewer's equivalent is the
 * GL-registered cudaArray of InteropRenderbuffer (adanerf_real_time_viewer/src/interoprenderbuffer.cpp:53-83). */
adn_status adn_register_host_buffer(adn_ctx* ctx, const void* p, size_t bytes);
adn_status adn_unregister_host_buffer(adn_ctx* ctx, const void* p);

/* Input / output width of a network set with adn_set_weights (sampling net: n_out is D, its depth cells, the width of
 * every raw0 the ABI reads or writes while it is set; 128 applies while none is). */
adn_status adn_net_dims(adn_ctx* ctx, int net_id, int* n_in, int* n_out);

/* ---- stage-level entry points (parity tests drive each kernel in isolation) ------------- */
/* stage 0: SpherePosDir.batch (src/features.py:845-899). d_x0 [N, 6 + 6 (P0 + D0)] fp32 (dir block first), d_ray_o/d [N,3]. */
adn_status adn_stage0_features(adn_ctx* ctx, const float* pose, const float* rot, const float* d_dirs, int64_t n_rays,
                               float* d_x0, float* d_ray_o, float* d_ray_d, void* stream);
/* stage 0a: generate_ray_directions (src/util/raygeneration.py:10-26). d_dirs [rows*W,3]. */
adn_status adn_generate_ray_directions(adn_ctx* ctx, int W, int H, int row0, int rows, float* d_dirs, void* stream);
/* stage 1: BaseNet.forward (src/models.py:183-195). d_x0 [N,n_in] fp32 -> d_raw0 [N,D] fp32 (D = n_out). */
adn_status adn_mlp0_forward(adn_ctx* ctx, const float* d_x0, int64_t n_rays, float* d_raw0, void* stream);
/* stage 2: FromClassifiedDepthAdaptive.generate (src/nerf_raymarch_common.py:699-757) + the mask
 * compaction of RayMarchFromPoses.batch (src/features.py:445-446,481-484).  Packed order is ray-major,
 * depth-ascending (= torch boolean-mask order).  d_raw0 [N,D], D = the sampling net's depth cells (128 while none is
 * set); 1 <= K <= min(D, 128).  Outputs: d_count/d_offset [N] int32 (exclusive scan),
 * d_cell/d_ray [cap] int32, d_z (world depth) / d_zp [cap] fp32, d_total (int64, device). cap >= N*K. */
adn_status adn_stage2_sample(adn_ctx* ctx, const float* d_raw0, int64_t n_rays, float thr, int K,
                             int32_t* d_count, int32_t* d_offset, int32_t* d_cell, int32_t* d_ray,
                             float* d_z, float* d_zp, int64_t* d_total, void* stream);
/* stage 2 threshold under a sample budget: *d_thr (device float) = the smallest t >= thr_min (> 0) with
 * sum_r clamp(#{cells of ray r >= t}, 1, K) <= max_samples (>= n_rays) -- the sample count stage 2 gives at t
 * (src/nerf_raymarch_common.py:726-749) -- from d_raw0 [N,D] (D as for adn_stage2_sample; 16-byte aligned at D = 128).
 * Exact: a radix select over the rays'
 * rank-2..K values. */
adn_status adn_budget_threshold(adn_ctx* ctx, const float* d_raw0, int64_t n_rays, float thr_min, int K, int64_t max_samples,
                                float* d_thr, void* stream);
/* FromClassifiedDepth's sample placement (the stage 2 of option "sampler" = 1): nerf_sample_pdf(linspace(0, 1, 129),
 * transform(raw0), K + 2, det = True) (src/nerf_raymarch_common.py:160-192, 606-660), samples 1 .. K, warped to world depth
 * with the scene's LogTransform.  d_raw0 [N,128] fp32; transform 1 = sigmoid, 2 = softmax.  Outputs (d_count, d_offset,
 * d_ray may be NULL): d_count [N] = K, d_offset [N] = r K, d_ray [N K] = r, d_z [N K] world depth, ascending per ray.
 * N K < 2^31.  Like adn_sampling_view it is an inspection entry and takes no stream: it runs on the context's own stream,
 * after the context's earlier calls, and returns once its outputs are written; d_raw0 must be complete when it is called
 * (the stream-ordered path is option "sampler" on the render entries). */
/* The rays of option "sampler" = 2 (RayMarchFromPoses.batch without a sampling net, src/features.py:417-431): d_dirs [N,3]
 * camera-space directions -> d_ray_o [N,3] = pose and d_ray_d [N,3] = R d, as nerf_get_ray_dirs' bmm forms it (the FMA chain
 * of stage 0), which adn_stage3_encode reads (it applies ndc_rays itself on NDC scenes).  d_ray_dirs [N,3] (may be NULL):
 * the directions whose norm nerf_raw2outputs scales its distances by, which adn_stage5_density_composite reads: R d, or on
 * NDC scenes ndc_rays' un-normalised direction (:430, as RayMarchFromPoses.postprocess passes it; needs the scene's ndc_w /
 * ndc_h).  Like adn_pdf_sample it is an inspection entry and takes no stream: it runs on the context's own stream, after
 * the context's earlier calls, and returns once its outputs are written (the stream-ordered path is option "sampler" = 2
 * on the render entries). */
adn_status adn_camera_rays(adn_ctx* ctx, const float* pose, const float* rot, const float* d_dirs, int64_t n_rays, float* d_ray_o,
                           float* d_ray_d, float* d_ray_dirs);
/* The K depths (1 <= K <= 128) option "sampler" = 2 places on every ray: LinearlySpacedZNearZFar.generate with det = True
 * (src/nerf_raymarch_common.py:310-326) in torch's fp32 steps, the to_world pow in double; on NDC scenes
 * LinearlySpacedZNearZFarNoDepthRange (:276-289), no warp.  d_z [K] fp32.  Like adn_pdf_sample it runs on the context's
 * own stream and returns once d_z is written. */
adn_status adn_linear_depths(adn_ctx* ctx, int K, float* d_z);
adn_status adn_pdf_sample(adn_ctx* ctx, const float* d_raw0, int64_t n_rays, int K, int transform, int32_t* d_count,
                          int32_t* d_offset, int32_t* d_ray, float* d_z);
/* The sampling network's view of raw0 alone (what option "sampling_view" draws after the sampling MLP), the viewer's
 * samplesToImage (adanerf_real_time_viewer/src/cuda/base_cuda_kernels.cu:487-528): d_raw0 [N,128] fp32, 16-byte aligned ->
 * d_rgb [N,3] fp32 (c0, c1, c2 as (c + 0.5) / 128) and d_rgba8 [N] uchar4 (each value * 255 truncated, alpha 255); either
 * output may be NULL.  c0, c1, c2 are the first three cells of the stable descending order that cub::BlockRadixSort gives
 * (CUDA 12.x CUB): keys compare as the twiddled bit patterns, with -0 equal to +0, so a positive NaN ranks above +inf and
 * a negative NaN below -inf, and equal keys keep the lower cell first.
 * Unlike the other stage entries it takes no stream: it is an inspection entry for a raw0 the caller already has (the
 * stream-ordered path is option "sampling_view" on the render entries).  It runs on the context's own stream, after the
 * context's earlier calls, like the *_host entries, and returns once its outputs are written (it synchronises that
 * stream); d_raw0 must be complete when the call is made. */
adn_status adn_sampling_view(adn_ctx* ctx, const float* d_raw0, int64_t n_rays, float* d_rgb, uint8_t* d_rgba8);
/* stage 3: RayMarchFromPoses.batch encode (src/features.py:458-479). d_x1 [M, P + V] fp32 (pos block first; adn_net_dims). */
adn_status adn_stage3_encode(adn_ctx* ctx, const float* d_ray_o, const float* d_ray_d, const int32_t* d_ray,
                             const float* d_z, int64_t n_samples, float* d_x1, void* stream);
/* stage 4: NeRF.forward (src/models.py:254-277). d_x1 [M, P + V] fp32 -> d_raw1 [M,4] fp32 = [rgb, alpha]. */
adn_status adn_mlp1_forward(adn_ctx* ctx, const float* d_x1, int64_t n_samples, float* d_raw1, void* stream);
/* stage 5: adaptive_raw2outputs (src/nerf_raymarch_common.py:91-144, accumulation_mult "alpha").
 * d_weights / d_depth_map may be NULL; d_weights is [N,K] zero padded like the reference's. */
adn_status adn_stage5_composite(adn_ctx* ctx, const float* d_raw1, const float* d_zp, const float* d_z,
                                const int32_t* d_offset, const int32_t* d_count, int64_t n_rays, int K,
                                float* d_rgb, float* d_weights, float* d_depth_map, void* stream);
/* stage 5 with every output a render can ask for: d_rgb [N,3] and d_rgba8 [N] uchar4 (the viewer's pixels) may each be
 * NULL, and so may every pointer of *aux (aux itself may be NULL).  depth_est uses the context's scene (depth_range, NDC)
 * exactly as a render does.  dense = 0: the packed layout of adn_stage2_sample (d_zp, d_z [M], d_offset / d_count [N]).
 * dense = 1: RayMarchFromPoses without remapping -- K must be 128 or D, d_zp is the sampling net's raw0 [N,K], z comes from
 * the context's dense depth table (what a thr == 0 render uses), and d_z / d_offset / d_count are ignored. */
adn_status adn_stage5_composite_aux(adn_ctx* ctx, const float* d_raw1, const float* d_zp, const float* d_z,
                                    const int32_t* d_offset, const int32_t* d_count, int64_t n_rays, int K, int dense,
                                    float* d_rgb, uint8_t* d_rgba8, const adn_aux_outputs* aux, void* stream);

/* stage 5 of option "sampler" = 1: nerf_raw2outputs (src/nerf_raymarch_common.py:19-68) over K samples per ray,
 * d_raw1 [N K, 4] and d_z [N K] in adn_pdf_sample's layout, d_ray_d [N,3] the ray directions of stage 0.  Outputs as
 * adn_stage5_composite_aux (each may be NULL); z_vals is d_z unchanged, alpha the density alpha.  K = 1: the reference's
 * dists are empty ([N, 0], :35-37), so every ray composites to nothing (rgb, weights, alpha, acc and depth 0; disp NaN).
 * No stream: it runs and synchronises like adn_pdf_sample. */
adn_status adn_stage5_density_composite(adn_ctx* ctx, const float* d_raw1, const float* d_z, const float* d_ray_d, int64_t n_rays,
                                        int K, float* d_rgb, uint8_t* d_rgba8, const adn_aux_outputs* aux);

/* ---- evaluation metric on the device ------------------------------------------------------ */
/* calculate_mse / calculate_psnr (src/evaluate.py:49-54) of two device images of n_values floats each:
 * mse = sum((a - b)^2) / n_values (double accumulation, deterministic), psnr = 10 log10(1 / mse).
 * clamp01 != 0 clips d_image to [0,1] first (src/evaluate.py:257-258).  Synchronises the stream; results on the host. */
adn_status adn_image_metrics(adn_ctx* ctx, const float* d_image, const float* d_reference, int64_t n_values, int clamp01,
                             double* mse_out, double* psnr_out, void* stream);
/* FLIP (Andersson et al., HPG 2020) of two device images, as src/evaluate.py:119-161 computes it through
 * src/util/flip_loss.py: d_image and d_reference are W x H sRGB pixels, [H*W, 3] fp32 row-major (no alignment needed);
 * d_flip_map [H*W] receives the per-pixel FLIP and *mean_out its mean (double accumulation, deterministic).  Either output
 * may be NULL, not both.  pixels_per_degree is the observer's (evaluate.py uses 0.7 * 3840 / 0.7 * pi / 180 = 67.02...);
 * it must be finite with 0 < ppd <= 200, the largest the kernels' filter radius (28 px) covers.  W, H >= 1, W * H < 2^31.
 * Inputs are clamped to [0,1] by the metric itself; a NaN input pixel makes the map NaN within the filter radius (10 px at
 * the default ppd) and the mean NaN, as the reference does.  The map is symmetric in the two images, bit for bit.
 * Like adn_sampling_view it takes no stream: it runs on the context's own stream after the context's earlier calls and
 * returns once the map is written and the mean is on the host (the inputs must be complete when the call is made).
 * Scratch: 56 B per pixel, kept by the context. */
adn_status adn_image_flip(adn_ctx* ctx, const float* d_image, const float* d_reference, int W, int H, double pixels_per_degree,
                          float* d_flip_map, double* mean_out);
/* Information-weighted multi-scale SSIM (IW-SSIM, Wang & Li 2011) of two device images, as src/evaluate.py:81-88 computes
 * it through src/util/IW_SSIM_PyTorch.py with its defaults (5 scales, 3 x 3 neighbourhoods with the parent band,
 * sigma_nsq 0.4, K = (0.01, 0.03), L = 255, an 11 x 11 Gaussian of sigma 1.5).  d_reference is the metric's original: its
 * bands weight the scales and supply the parent band, so the metric is not symmetric.  Layouts:
 *   ADN_IWSSIM_GRAY          [H*W] fp32 planes, H rows of W, used as given (the metric's constants assume values 0..255);
 *   ADN_IWSSIM_EVALUATE_RGB  [H*W, 3] fp32 as evaluate.py holds its images: each becomes rgb2gray(x.view(W, H, -1)), that is
 *                            round-half-even(0.2989 r + 0.5870 g + 0.1140 b) in fp32, an image of W rows of H pixels (for
 *                            W != H a reshuffle of the frame, not its transpose).  Images in [0, 1] become 0s and 1s, as
 *                            in evaluate.py, so scores stay close to 1.
 * *score_out receives the score and scale_out[5] (may be NULL) wmcs of scales 1..5; the score is the product of |wmcs_s|
 * raised to (0.0448, 0.2856, 0.3001, 0.2363, 0.1333).  Pyramid in fp64, bands rounded to fp32 once, everything after them
 * in fp64; deterministic (a repeated call returns the same bits).
 * W, H >= 161 (the coarsest band must hold one 11 x 11 window) and W * H < 2^31; NULL inputs or score_out, or an unknown
 * layout, fail with ADN_ERR_INVALID before any launch.  A scale whose rebuilt covariance cannot be inverted (all its
 * adjusted eigenvalues 0, or a zero pivot) is NaN and so is the score, with ADN_OK: an all-zero reference (every band 0,
 * where the reference's torch.linalg.inv raises) and a NaN input pixel do this.
 * Like adn_image_flip it takes no stream: it runs on the context's own stream after the context's earlier calls and returns
 * with the results on the host (the inputs must be complete when the call is made).  Scratch, kept by the context: about
 * 16 B per pixel of the metric's image for both pyramids. */
#define ADN_IWSSIM_GRAY          0
#define ADN_IWSSIM_EVALUATE_RGB  1
adn_status adn_image_iwssim(adn_ctx* ctx, const float* d_image, const float* d_reference, int W, int H, int layout,
                            double* score_out, double* scale_out);

#ifdef __cplusplus
}
#endif
#endif /* ADANERF_B200_H */
