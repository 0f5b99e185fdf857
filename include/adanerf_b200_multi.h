/* adanerf_b200 -- multi-GPU frame renderer (libadanerf_b200_multi.so, links NCCL).
 *
 * One host thread drives G devices of one node (each frame's bands are enqueued from one short-lived thread per device
 * when G > 1): one adn_ctx per device (weights replicated), contiguous row bands of the
 * image per device (ray id = y * W + x, images are rgb.reshape(h, w, 3) with no flip -- src/util/saveimage.py:46 of
 * thomasneff/AdaNeRF), each device generates its own rays from (pose, rot, row0, rows), and ONE NCCL gather per frame
 * (grouped ncclSend / ncclRecv over NVLink) collects the RGB tiles on the first device.  ncclCommInitAll over the
 * devices, a render stream and a communication stream per device; two frames may be in flight, so the gather of frame
 * f overlaps the sampling MLP of frame f + 1 (SURVEY.md 8e).
 *
 * The reference has no multi-GPU path (src/train_data.py:73 selects a single device; the viewer renders on the GL
 * device): this is the BASELINE.json north_star's "rays shard embarrassingly across the 8 GPUs as image tiles with one
 * NCCL gather of RGB tiles".  Invariant (tests/test_multi.py): the gathered frame equals the single-GPU frame bit for bit.
 */
#ifndef ADANERF_B200_MULTI_H
#define ADANERF_B200_MULTI_H

#include "adanerf_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct adn_multi adn_multi;

/* devices: CUDA ordinals (NULL: 0 .. n_devices-1).  The first one receives the gathered frame. */
adn_status adn_multi_create(adn_multi** out, const adn_scene* scene, const int* devices, int n_devices);
/* Export directory {config.ini, dataset_info.txt, model0.onnx, model1.onnx} (src/export.py:28-93), read once. */
adn_status adn_multi_create_from_export_dir(adn_multi** out, const char* dir, const int* devices, int n_devices, float* thr_out,
                                            int* k_out);
void adn_multi_destroy(adn_multi* m);
const char* adn_multi_last_error(const adn_multi* m);
int adn_multi_devices(const adn_multi* m);

/* Same tensors to every device (see adn_set_weights). */
adn_status adn_multi_set_weights(adn_multi* m, int net_id, const adn_tensor_desc* tensors, int n_tensors);
/* The same option on every device (see adn_set_option), except "sample_budget": B > 0 is the budget of the whole frame.
 * Every device's context joins a budget group (adn_set_budget_group) whose reducer is ncclAllReduce(ncclUint64, ncclSum)
 * on that device's communicator and the band's stream, so all bands render at the one threshold t* a single device would
 * choose for the frame (M <= B over all bands; the frame equals the single-GPU budgeted frame bit for bit).  The bands of a
 * frame are then enqueued from one host thread per device, and a device with no rows still makes its (empty) budgeted
 * call.  B < W * H, dense mode (thr == 0) and more than 2^32 - 1 candidates (W * H * (K - 1)) are refused for the whole
 * frame before any device enqueues.  0 = off.  With "sampling_view" = 1 the frame is the sampling net's view on every band
 * and no budget is applied (nor its checks made), as on one device. */
adn_status adn_multi_set_option(adn_multi* m, const char* name, int64_t value);

/* Row band of device `rank` for an image of H rows: rows [row0, row0 + rows), whole rows, sizes differ by at most one. */
void adn_multi_band(const adn_multi* m, int H, int rank, int* row0, int* rows);

/* Enqueues one W x H frame: every device renders its band, then the bands are gathered on the first device.  Returns
 * without waiting; at most two frames may be in flight (ADN_ERR_INVALID otherwise). */
adn_status adn_multi_render_camera(adn_multi* m, const float* pose, const float* rot, int W, int H, float thr, int K);

/* Waits for the oldest frame in flight.  *d_frame (may be NULL) receives the [H*W, 3] fp32 frame on the first device;
 * it stays valid until the second next adn_multi_render_camera.  h_rgb (may be NULL) receives a host copy. */
adn_status adn_multi_wait_frame(adn_multi* m, const float** d_frame, float* h_rgb);

/* Device time of the last completed frame on each device: render (band) and gather, in ms; arrays of n_devices. */
adn_status adn_multi_last_times(adn_multi* m, float* render_ms, float* gather_ms);

/* The threshold the newest frame enqueued rendered at: t* under "sample_budget" (the same on every band), else its `thr`.
 * Synchronises the first device. */
adn_status adn_multi_last_threshold(adn_multi* m, float* thr_out);
/* Samples M of each band of the newest frame enqueued (band_samples: array of n_devices; their sum is the frame's M).
 * Waits for that frame's bands. */
adn_status adn_multi_last_samples(adn_multi* m, int64_t* band_samples);

#ifdef __cplusplus
}
#endif
#endif /* ADANERF_B200_MULTI_H */
