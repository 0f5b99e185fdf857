/* adanerf_b200 -- several cameras in one render call (libadanerf_b200.so, the same library and context as
 * include/adanerf_b200.h, whose conventions hold here: device "d_" pointers, `stream` a cudaStream_t passed as void*, stream
 * ordered with no host synchronisation, calls on one context executed in the order they were issued whatever stream each
 * names, and a call on a stream that is capturing a CUDA graph refused with ADN_ERR_INVALID before anything is enqueued).
 *
 * The [n_images, n_samples] batches TrainConfig.inference takes (src/train_data.py:278-299, SpherePosDir.batch /
 * RayMarchFromPoses.batch, src/features.py:392-427,845-864), stereo pairs and view sets:
 *   poses [V,3] and rots [V,9] (row-major 3x3 each) are HOST pointers, read before the call returns; 1 <= V <= 64 (each
 *   launch carries the camera table in its kernel parameters: 48 B a view).
 *   Rays are view-major: ray v N + i is ray i of view v (the order tile(poses, n_samples) gives), and every output is
 *   laid out [V N, ...] like the single-view entries' [N, ...].  Rays never interact: without a sample budget a call is
 *   bit for bit the V single-view calls concatenated.  Every option applies to the whole call as to one camera: the
 *   samplers, NDC scenes (one image size for all views), dense mode, fuse_encoder, chunk_rays (a chunk may split a view),
 *   sampling_view and budget groups; "sample_budget" chooses ONE t* under ONE B over all V N rays, so every view renders at
 *   the same threshold (a call is then bit for bit the V single-view calls at thr = t*); adn_last_threshold reports that
 *   t*, and adn_get_stats reports the call as it does a single-view call of V N rays.  V = 1 gives exactly the bits of the
 *   single-view entry.
 *   Refused with ADN_ERR_INVALID before anything is enqueued: V < 1 or V > 64, NULL tables, N < 1 (W, H < 1), V N that
 *   overflows int64, and a capturing stream; then every check of the single-view entries applies to the V N rays.
 * Row bands (row0 / rows) and the multi-GPU entries (include/adanerf_b200_multi.h) stay single-view.
 */
#ifndef ADANERF_B200_VIEWS_H
#define ADANERF_B200_VIEWS_H

#include "adanerf_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* d_dirs [V N,3] camera-space directions, n_per_view = N; d_rgb [V N,3], d_nsamples [V N], d_oracle_weights [V N,D] and
 * aux ([V N,K] / [V N]; aux may be NULL) as adn_render_rays_aux. */
adn_status adn_render_views_rays(adn_ctx* ctx, int n_views, const float* poses, const float* rots, const float* d_dirs,
                                 int64_t n_per_view, float thr, int K, float* d_rgb, int32_t* d_nsamples,
                                 float* d_oracle_weights, const adn_aux_outputs* aux, void* stream);
/* V whole W x H frames generated on the device (ray v W H + y W + x): d_rgb [V,H,W,3], d_nsamples [V,H,W] or NULL. */
adn_status adn_render_views_camera(adn_ctx* ctx, int n_views, const float* poses, const float* rots, int W, int H, float thr,
                                   int K, float* d_rgb, int32_t* d_nsamples, void* stream);
/* The same as the viewer's pixels: d_rgba8 [V,H,W] uchar4. */
adn_status adn_render_views_camera_rgba8(adn_ctx* ctx, int n_views, const float* poses, const float* rots, int W, int H,
                                         float thr, int K, uint8_t* d_rgba8, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ADANERF_B200_VIEWS_H */
