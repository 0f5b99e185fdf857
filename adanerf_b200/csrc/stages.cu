// SIMT stages (see stages.cuh).  All position math uses explicit round-to-nearest intrinsics in the
// reference's operation order so results track the PyTorch fp32 path (no FMA contraction where torch
// has separate mul/add; an FMA chain where ATen's K=3 bmm uses one).
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <algorithm>

#include "mlp.cuh"
#include "posenc.cuh"
#include "ptx.cuh"
#include "stages.cuh"
#include "tiles.cuh"

namespace adn {

// posEnc 10-4, the encoding with compile-time kernels (and 2-2 for the sampling net)
constexpr int kNFreqPos = 10;
constexpr int kNFreqDir = 4;
constexpr int kFeat = 90;

// ------------------------------------------------------------------------------------ stage 0a
__device__ __forceinline__ void pixel_dir(const CameraRays& cam, long long ray, float (&d)[3]) {
  const int y = cam.row0 + int(ray / cam.W);
  const int x = int(ray % cam.W);
  const double rx = __dadd_rn(cam.start_x, __dmul_rn(cam.x_pp, double(x)));
  const double ry = __dadd_rn(cam.start_y, __dmul_rn(cam.y_pp, double(y)));
  const double rz = cam.focal;
  const double n = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(rx, rx), __dmul_rn(ry, ry)), __dmul_rn(rz, rz)));
  d[0] = float(__ddiv_rn(rx, n));
  d[1] = float(-__ddiv_rn(ry, n));
  d[2] = float(-__ddiv_rn(rz, n));
}

__global__ void gen_dirs_kernel(const __grid_constant__ CameraRays cam, long long n_rays, float* __restrict__ dirs) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n_rays) return;
  float d[3];
  pixel_dir(cam, i, d);
  dirs[3 * i + 0] = d[0];
  dirs[3 * i + 1] = d[1];
  dirs[3 * i + 2] = d[2];
}

cudaError_t launch_gen_dirs(const CameraRays& cam, long long n_rays, float* d_dirs, cudaStream_t s) {
  if (n_rays <= 0) return cudaSuccess;
  gen_dirs_kernel<<<unsigned((n_rays + 255) / 256), 256, 0, s>>>(cam, n_rays, d_dirs);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------ stage 0b
// nds = R * d : ATen bmm with K = 3 accumulates as an FMA chain over k = 0,1,2 (src/features.py:858-859, and
// nerf_get_ray_dirs, src/nerf_raymarch_common.py:147-152)
__device__ __forceinline__ void rotate_dir(const PoseDev& pd, const float (&d)[3], float (&nds)[3]) {
#pragma unroll
  for (int r = 0; r < 3; ++r)
    nds[r] = __fmaf_rn(pd.rot[3 * r + 2], d[2], __fmaf_rn(pd.rot[3 * r + 1], d[1], __fmul_rn(pd.rot[3 * r + 0], d[0])));
}

// Where ray i of a launch takes its camera from, and its index inside its view (pix: its pixel when the rays are generated
// from a camera).  OnePose: one camera for the launch, pix = i.  PerView: the row of its view in a ViewTable (view-major
// rays, the launch starting at ray t.ray0 of the call).
struct OnePose {
  const PoseDev& pd;
  __device__ __forceinline__ const PoseDev& of(long long i, long long& pix) const {
    pix = i;
    return pd;
  }
};
struct PerView {
  const ViewTable& t;
  __device__ __forceinline__ const PoseDev& of(long long i, long long& pix) const {
    const long long g = t.ray0 + i;
    const long long v = g / t.n_per_view;
    pix = g - v * t.n_per_view;
    return t.v[v];
  }
};

// SpherePosDir.batch (src/features.py:845-899) up to the encodings: the pixel direction d of ray i (pixel pix), the ray
// origin p on the view-cell sphere, the rotated direction nds and its unit copy dn.
template <bool FROM_CAMERA>
__device__ __forceinline__ void sphere_pos_dir(const SceneDev& sc, const PoseDev& pd, const float* __restrict__ dirs,
                                               const CameraRays& cam, long long i, long long pix, float (&p)[3], float (&nds)[3],
                                               float (&dn)[3]) {
  float d[3];
  if (FROM_CAMERA) {
    pixel_dir(cam, pix, d);
  } else {
    d[0] = dirs[3 * i + 0];
    d[1] = dirs[3 * i + 1];
    d[2] = dirs[3 * i + 2];
  }
  rotate_dir(pd, d, nds);
  // compute_ray_offset (:769-791)
  float omc[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) omc[a] = __fsub_rn(pd.pose[a], sc.c[a]);
  const float udot = __fadd_rn(__fadd_rn(__fmul_rn(omc[0], nds[0]), __fmul_rn(omc[1], nds[1])), __fmul_rn(omc[2], nds[2]));
  const float omc2 = __fadd_rn(__fadd_rn(__fmul_rn(omc[0], omc[0]), __fmul_rn(omc[1], omc[1])), __fmul_rn(omc[2], omc[2]));
  const float delta = __fsub_rn(__fmul_rn(udot, udot), __fsub_rn(omc2, sc.r2));
  const float t = __fadd_rn(-udot, __fsqrt_rn(fmaxf(delta, 0.0f)));
#pragma unroll
  for (int a = 0; a < 3; ++a) p[a] = __fadd_rn(pd.pose[a], __fmul_rn(nds[a], t));
  const float nn = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(nds[0], nds[0]), __fmul_rn(nds[1], nds[1])), __fmul_rn(nds[2], nds[2])));
#pragma unroll
  for (int a = 0; a < 3; ++a) dn[a] = __fdiv_rn(nds[a], nn);
}

// One thread per ray, the encodings "10-4" or "2-2" at compile time.
template <bool FROM_CAMERA, int NFD, int NFP, class Poses>
__device__ __forceinline__ void stage0_body(const SceneDev& sc, const Poses& poses, const float* __restrict__ dirs,
                                            const CameraRays& cam, long long n_rays, float* __restrict__ x0,
                                            float* __restrict__ ray_o, float* __restrict__ ray_d, uint8_t* __restrict__ tiles0,
                                            int tile_terms, uint8_t* s_tile) {
  constexpr int F0 = 6 + 6 * (NFD + NFP);       // 90 ("10-4") or 30 ("2-2")
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;   // grid covers whole 128-ray tiles
  float f[F0];
#pragma unroll
  for (int j = 0; j < F0; ++j) f[j] = 0.0f;
  if (i < n_rays) {
    float p[3], nds[3], dn[3];
    long long pix;
    const PoseDev& pd = poses.of(i, pix);
    sphere_pos_dir<FROM_CAMERA>(sc, pd, dirs, cam, i, pix, p, nds, dn);
    posenc3<NFD>(dn, f);                           // 27 / 15: direction block FIRST (:868)
    posenc3<NFP>(p, f + 3 + 6 * NFD);              // 63 / 15
    if (ray_o) {
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        ray_o[3 * i + a] = p[a];
        ray_d[3 * i + a] = nds[a];
      }
    }
    if (x0) {
#pragma unroll
      for (int j = 0; j < F0; ++j) x0[i * F0 + j] = f[j];
    }
  }
  if (tiles0) {   // the CTA's 128 rays are one tile of the sampling net's input
    const TileFormat fmt = sampling_tiles(F0, tile_terms);
    store_tile(fmt, f, s_tile, tiles0 + size_t(i >> 7) * fmt.tile_bytes());
    store_tiles_drain();
  }
}

template <bool FROM_CAMERA, int NFD = kNFreqDir, int NFP = kNFreqPos>
__global__ void __launch_bounds__(128)
stage0_kernel(const __grid_constant__ SceneDev sc, const __grid_constant__ PoseDev pd, const float* __restrict__ dirs,
              const __grid_constant__ CameraRays cam, long long n_rays, float* __restrict__ x0, float* __restrict__ ray_o,
              float* __restrict__ ray_d, uint8_t* __restrict__ tiles0, int tile_terms) {
  extern __shared__ __align__(1024) uint8_t s_tile[];
  stage0_body<FROM_CAMERA, NFD, NFP>(sc, OnePose{pd}, dirs, cam, n_rays, x0, ray_o, ray_d, tiles0, tile_terms, s_tile);
}

// The same over the views of a multi-view call: each ray takes its view's camera.
template <bool FROM_CAMERA, int NFD = kNFreqDir, int NFP = kNFreqPos>
__global__ void __launch_bounds__(128)
stage0_views_kernel(const __grid_constant__ SceneDev sc, const __grid_constant__ ViewTable views, const float* __restrict__ dirs,
                    const __grid_constant__ CameraRays cam, long long n_rays, float* __restrict__ x0, float* __restrict__ ray_o,
                    float* __restrict__ ray_d, uint8_t* __restrict__ tiles0, int tile_terms) {
  extern __shared__ __align__(1024) uint8_t s_tile[];
  stage0_body<FROM_CAMERA, NFD, NFP>(sc, PerView{views}, dirs, cam, n_rays, x0, ray_o, ray_d, tiles0, tile_terms, s_tile);
}

// Any other encoding (sc.n_freq_dir0 + sc.n_freq_pos0 <= 20 bands, 0 = posEnc none): the same features, written one at a
// time into x0 and the tile image, so no thread holds its up to 126 features at once.
template <bool FROM_CAMERA, class Poses>
__device__ __forceinline__ void stage0_rt_body(const SceneDev& sc, const Poses& poses, const float* __restrict__ dirs,
                                               const CameraRays& cam, long long n_rays, float* __restrict__ x0,
                                               float* __restrict__ ray_o, float* __restrict__ ray_d,
                                               uint8_t* __restrict__ tiles0, int tile_terms, uint8_t* s_tile) {
  const int nfd = sc.n_freq_dir0, nfp = sc.n_freq_pos0;
  const int F0 = 6 + 6 * (nfd + nfp);
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;   // grid covers whole 128-ray tiles
  const TileFormat fmt = sampling_tiles(F0, tile_terms);
  if (tiles0) zero_row(fmt, s_tile, threadIdx.x, 0, fmt.n_blk);
  if (i < n_rays) {
    float p[3], nds[3], dn[3];
    long long pix;
    const PoseDev& pd = poses.of(i, pix);
    sphere_pos_dir<FROM_CAMERA>(sc, pd, dirs, cam, i, pix, p, nds, dn);
    auto put = [&](int c, float v) {
      if (x0) x0[i * F0 + c] = v;
      if (tiles0) put_feature(fmt, s_tile, c >> 6, threadIdx.x, c & 63, v);
    };
    posenc3_rt(dn, nfd, put);                                             // direction block FIRST (:868)
    posenc3_rt(p, nfp, [&](int j, float v) { put(3 + 6 * nfd + j, v); });
    if (ray_o) {
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        ray_o[3 * i + a] = p[a];
        ray_d[3 * i + a] = nds[a];
      }
    }
  }
  if (tiles0) {
    flush_tile(fmt, s_tile, tiles0 + size_t(i >> 7) * fmt.tile_bytes());
    store_tiles_drain();
  }
}

template <bool FROM_CAMERA>
__global__ void __launch_bounds__(128)
stage0_rt_kernel(const __grid_constant__ SceneDev sc, const __grid_constant__ PoseDev pd, const float* __restrict__ dirs,
                 const __grid_constant__ CameraRays cam, long long n_rays, float* __restrict__ x0, float* __restrict__ ray_o,
                 float* __restrict__ ray_d, uint8_t* __restrict__ tiles0, int tile_terms) {
  extern __shared__ __align__(1024) uint8_t s_tile[];
  stage0_rt_body<FROM_CAMERA>(sc, OnePose{pd}, dirs, cam, n_rays, x0, ray_o, ray_d, tiles0, tile_terms, s_tile);
}

template <bool FROM_CAMERA>
__global__ void __launch_bounds__(128)
stage0_rt_views_kernel(const __grid_constant__ SceneDev sc, const __grid_constant__ ViewTable views, const float* __restrict__ dirs,
                       const __grid_constant__ CameraRays cam, long long n_rays, float* __restrict__ x0, float* __restrict__ ray_o,
                       float* __restrict__ ray_d, uint8_t* __restrict__ tiles0, int tile_terms) {
  extern __shared__ __align__(1024) uint8_t s_tile[];
  stage0_rt_body<FROM_CAMERA>(sc, PerView{views}, dirs, cam, n_rays, x0, ray_o, ray_d, tiles0, tile_terms, s_tile);
}

cudaError_t launch_stage0(const SceneDev& sc, const PoseDev& pd, const float* d_dirs, const CameraRays* cam,
                          long long n_rays, float* d_x0, float* d_ray_o, float* d_ray_d, uint8_t* d_tiles0, int tile_terms,
                          cudaStream_t s, const ViewTable* views) {
  if (n_rays <= 0) return cudaSuccess;
  const long long n_pad = ((n_rays + kTileM - 1) / kTileM) * kTileM;
  const unsigned grid = unsigned((n_pad + 127) / 128);
  CameraRays c{};
  const int tile_bytes = int(sampling_tiles(0, 2).tile_bytes());   // the largest sampling tile
  const size_t smem = d_tiles0 ? sampling_tiles(0, tile_terms).tile_bytes() : 0;
  if (cam) c = *cam;
  // the compile-time encodings where the scene has them, else the run-time one
  auto run = [&](auto k_cam, auto k_rays, unsigned long long* attr) -> cudaError_t {
    if (set_max_dyn_smem_once(reinterpret_cast<const void*>(k_cam), tile_bytes, &attr[0]) != cudaSuccess ||
        set_max_dyn_smem_once(reinterpret_cast<const void*>(k_rays), tile_bytes, &attr[1]) != cudaSuccess)
      return cudaGetLastError();
    if (cam) k_cam<<<grid, 128, smem, s>>>(sc, pd, d_dirs, c, n_rays, d_x0, d_ray_o, d_ray_d, d_tiles0, tile_terms);
    else k_rays<<<grid, 128, smem, s>>>(sc, pd, d_dirs, c, n_rays, d_x0, d_ray_o, d_ray_d, d_tiles0, tile_terms);
    return cudaGetLastError();
  };
  auto run_views = [&](auto k_cam, auto k_rays, unsigned long long* attr) -> cudaError_t {
    if (set_max_dyn_smem_once(reinterpret_cast<const void*>(k_cam), tile_bytes, &attr[0]) != cudaSuccess ||
        set_max_dyn_smem_once(reinterpret_cast<const void*>(k_rays), tile_bytes, &attr[1]) != cudaSuccess)
      return cudaGetLastError();
    if (cam) k_cam<<<grid, 128, smem, s>>>(sc, *views, d_dirs, c, n_rays, d_x0, d_ray_o, d_ray_d, d_tiles0, tile_terms);
    else k_rays<<<grid, 128, smem, s>>>(sc, *views, d_dirs, c, n_rays, d_x0, d_ray_o, d_ray_d, d_tiles0, tile_terms);
    return cudaGetLastError();
  };
  static unsigned long long attr104[2] = {0, 0}, attr22[2] = {0, 0}, attr_rt[2] = {0, 0};   // per device
  static unsigned long long vattr104[2] = {0, 0}, vattr22[2] = {0, 0}, vattr_rt[2] = {0, 0};
  const bool e104 = sc.n_freq_pos0 == kNFreqPos && sc.n_freq_dir0 == kNFreqDir, e22 = sc.n_freq_pos0 == 2 && sc.n_freq_dir0 == 2;
  if (views) {
    if (e104) return run_views(stage0_views_kernel<true>, stage0_views_kernel<false>, vattr104);
    if (e22) return run_views(stage0_views_kernel<true, 2, 2>, stage0_views_kernel<false, 2, 2>, vattr22);
    return run_views(stage0_rt_views_kernel<true>, stage0_rt_views_kernel<false>, vattr_rt);
  }
  if (e104) return run(stage0_kernel<true>, stage0_kernel<false>, attr104);
  if (e22) return run(stage0_kernel<true, 2, 2>, stage0_kernel<false, 2, 2>, attr22);
  return run(stage0_rt_kernel<true>, stage0_rt_kernel<false>, attr_rt);
}

// ------------------------------------------------------------------------------------ camera rays (sampler 2)
// RayMarchFromPoses.batch's rays when no sampling net runs (src/features.py:417-431): rays_d = R d as nerf_get_ray_dirs'
// bmm forms it (not renormalised) and rays_o = pose.  ray_dirs (may be null) gets the directions whose norm
// nerf_raw2outputs scales its distances by: rays_d itself, or on NDC scenes ndc_rays' un-normalised direction (what
// RayMarchFromPoses.postprocess hands it, not the unit copy that is encoded).  12 B in (or the pixel's direction from cam),
// 24 B out per ray, 36 B with ray_dirs.
template <bool FROM_CAMERA, class Poses>
__device__ __forceinline__ void camera_rays_body(const SceneDev& sc, const Poses& poses, const float* __restrict__ dirs,
                                                 const CameraRays& cam, long long n_rays, float* __restrict__ ray_o,
                                                 float* __restrict__ ray_d, float* __restrict__ ray_dirs) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n_rays) return;
  long long pix;
  const PoseDev& pd = poses.of(i, pix);
  float d[3], nds[3];
  if (FROM_CAMERA) {
    pixel_dir(cam, pix, d);
  } else {
#pragma unroll
    for (int a = 0; a < 3; ++a) d[a] = __ldg(dirs + 3 * i + a);
  }
  rotate_dir(pd, d, nds);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    ray_o[3 * i + a] = pd.pose[a];
    ray_d[3 * i + a] = nds[a];
  }
  if (ray_dirs) {
    float v[3] = {nds[0], nds[1], nds[2]};
    if (sc.ndc) {   // :430
      float oo[3];
      ndc_ray(sc, pd.pose, nds, oo, v);
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) ray_dirs[3 * i + a] = v[a];
  }
}

template <bool FROM_CAMERA>
__global__ void __launch_bounds__(256)
camera_rays_kernel(const __grid_constant__ SceneDev sc, const __grid_constant__ PoseDev pd, const float* __restrict__ dirs,
                   const __grid_constant__ CameraRays cam, long long n_rays, float* __restrict__ ray_o, float* __restrict__ ray_d,
                   float* __restrict__ ray_dirs) {
  camera_rays_body<FROM_CAMERA>(sc, OnePose{pd}, dirs, cam, n_rays, ray_o, ray_d, ray_dirs);
}

// The same over the views of a multi-view call: each ray takes its view's camera.
template <bool FROM_CAMERA>
__global__ void __launch_bounds__(256)
camera_rays_views_kernel(const __grid_constant__ SceneDev sc, const __grid_constant__ ViewTable views, const float* __restrict__ dirs,
                         const __grid_constant__ CameraRays cam, long long n_rays, float* __restrict__ ray_o,
                         float* __restrict__ ray_d, float* __restrict__ ray_dirs) {
  camera_rays_body<FROM_CAMERA>(sc, PerView{views}, dirs, cam, n_rays, ray_o, ray_d, ray_dirs);
}

cudaError_t launch_camera_rays(const SceneDev& sc, const PoseDev& pd, const float* d_dirs, const CameraRays* cam,
                               long long n_rays, float* d_ray_o, float* d_ray_d, float* d_ray_dirs, cudaStream_t s,
                               const ViewTable* views) {
  if (n_rays <= 0) return cudaSuccess;
  const unsigned grid = unsigned((n_rays + 255) / 256);
  const CameraRays c = cam ? *cam : CameraRays{};
  if (views && cam) camera_rays_views_kernel<true><<<grid, 256, 0, s>>>(sc, *views, d_dirs, c, n_rays, d_ray_o, d_ray_d, d_ray_dirs);
  else if (views) camera_rays_views_kernel<false><<<grid, 256, 0, s>>>(sc, *views, d_dirs, c, n_rays, d_ray_o, d_ray_d, d_ray_dirs);
  else if (cam) camera_rays_kernel<true><<<grid, 256, 0, s>>>(sc, pd, d_dirs, c, n_rays, d_ray_o, d_ray_d, d_ray_dirs);
  else camera_rays_kernel<false><<<grid, 256, 0, s>>>(sc, pd, d_dirs, c, n_rays, d_ray_o, d_ray_d, d_ray_dirs);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------- stage 2
// FromClassifiedDepthAdaptive.generate (src/nerf_raymarch_common.py:699-757) + mask compaction
// (src/features.py:445-446,481-484), single pass:
//   * one warp per ray, lane l owns cells 4l..4l+3 (one coalesced 512-byte row load),
//   * survivors = cells >= thr; more than K survivors -> K rounds of warp arg-max (value descending,
//     ties lower cell first); none -> the arg-max cell; order inside a ray = ascending cell = ascending z,
//   * per-CTA exclusive scan of the counts + decoupled look-back across CTAs (dynamic tickets), so the
//     packed order is deterministic ray-major (the torch boolean-mask order) with no host sync.
constexpr int kS2Rays = 64;     // rays per CTA
constexpr int kS2Threads = 256;  // 8 warps x 8 rays

// Order-preserving map float -> uint32 (larger float <-> larger key); -0.0 is folded onto +0.0 so it ties
// with it like a float compare does.  Every real input maps to a key >= 0x007FFFFF, so 0 means "no entry".
__device__ __forceinline__ uint32_t order_key(float v) {
  const uint32_t u = __float_as_uint(v + 0.0f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ void cswap_desc(unsigned long long& a, unsigned long long& b) {
  const unsigned long long hi = a > b ? a : b, lo = a > b ? b : a;
  a = hi;
  b = lo;
}

// Returns the 4 selection masks (bit l of sel[j] <-> cell 4l+j) and the count, warp uniform.
// More than K survivors: K rounds of "pop the best head".  Each lane keeps its (up to 4) candidates as
// 64-bit composites (order_key << 2 | 3 - j), sorted descending, so the head of every lane is its best
// remaining cell; one REDUX.MAX over the heads + a ballot finds the winner (ties: lowest lane = lowest
// cell, and inside a lane the lower j sorts first), and only the winning lane pops.
__device__ __forceinline__ int select_cells(const float4 v4, float thr, int K, int lane, uint32_t (&sel)[4]) {
  const float v[4] = {v4.x, v4.y, v4.z, v4.w};
  uint32_t act[4];
  int cnt = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    act[j] = __ballot_sync(0xffffffffu, v[j] >= thr);
    cnt += __popc(act[j]);
  }
  if (cnt > 0 && cnt <= K) {
#pragma unroll
    for (int j = 0; j < 4; ++j) sel[j] = act[j];
    return cnt;
  }
  const bool fallback = (cnt == 0);          // nothing >= thr: the arg-max cell (:748-749)
  const int need = fallback ? 1 : K;
  unsigned long long h[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const bool cand = fallback || ((act[j] >> lane) & 1u);
    h[j] = cand ? (((unsigned long long)order_key(v[j]) << 2) | (unsigned long long)(3 - j)) : 0ull;
  }
  cswap_desc(h[0], h[1]);
  cswap_desc(h[2], h[3]);
  cswap_desc(h[0], h[2]);
  cswap_desc(h[1], h[3]);
  cswap_desc(h[1], h[2]);
  uint32_t mine = 0;
  for (int round = 0; round < need; ++round) {
    const uint32_t head = uint32_t(h[0] >> 2);
    const uint32_t m = __reduce_max_sync(0xffffffffu, head);
    const uint32_t who = __ballot_sync(0xffffffffu, head == m);
    if (lane == __ffs(who) - 1) {
      mine |= 1u << (3 - int(h[0] & 3ull));
      h[0] = h[1];
      h[1] = h[2];
      h[2] = h[3];
      h[3] = 0ull;
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) sel[j] = __ballot_sync(0xffffffffu, (mine >> j) & 1u);
  return need;
}

// Lane `lane`'s four cells of a 128-cell row: one 16-byte load when the rows are 16-byte aligned, else four 4-byte loads
// (a float4 load from an address that is not a multiple of 16 faults).
__device__ __forceinline__ float4 ld_row_quad(const float* __restrict__ row, int lane, bool aligned16) {
  if (aligned16) return __ldg(reinterpret_cast<const float4*>(row) + lane);
  const float* p = row + 4 * lane;
  return make_float4(__ldg(p), __ldg(p + 1), __ldg(p + 2), __ldg(p + 3));
}

__device__ __forceinline__ unsigned long long ld_volatile_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

// Tile bookkeeping, executed by one full warp.  Tiles are numbered by dynamic tickets, so every predecessor a tile
// spins on has already started.  A tile's state word carries flag and value together (no fence needed).
// State word: [63:62] flag (1 = tile aggregate, 2 = inclusive prefix), [61:40] launch epoch, [39:0] value.  A word whose
// epoch is not the current launch's reads as "not ready", so the state array is never cleared between launches
// (launch_stage2 zeroes it when the buffer is new and when the 22-bit epoch wraps); tickets are consumed relative to a
// per-launch base for the same reason.
constexpr unsigned long long kS2FlagAgg = 1ull << 62, kS2FlagInc = 2ull << 62, kS2ValMask = (1ull << 40) - 1;
constexpr uint32_t kS2EpochMask = (1u << 22) - 1;
__device__ __forceinline__ unsigned long long s2_pack(unsigned long long flag, uint32_t epoch, long long value) {
  return flag | ((unsigned long long)epoch << 40) | ((unsigned long long)value & kS2ValMask);
}
// flag of a state word as seen by launch `epoch` (0 = not ready / stale)
__device__ __forceinline__ uint32_t s2_flag(unsigned long long st, uint32_t epoch) {
  return (uint32_t(st >> 40) & kS2EpochMask) == epoch ? uint32_t(st >> 62) : 0u;
}

// Exclusive scan of the tile's 64 per-ray counts (-> s_off); publishes the tile aggregate right away so that the
// successors' look-backs can pass over this tile while it is still busy.  Returns the tile total.
__device__ __forceinline__ int s2_tile_scan(const int* s_cnt, int* s_off, int tile, int lane,
                                            unsigned long long* __restrict__ tile_state, uint32_t epoch) {
  const int a = s_cnt[2 * lane], b = s_cnt[2 * lane + 1];
  int x = a + b;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  const int excl = x - (a + b);
  s_off[2 * lane] = excl;
  s_off[2 * lane + 1] = excl + a;
  const int tile_total = __shfl_sync(0xffffffffu, x, 31);
  if (tile > 0 && lane == 0) atomicExch(&tile_state[tile], s2_pack(kS2FlagAgg, epoch, tile_total));
  return tile_total;
}

// Decoupled look-back over the preceding tiles (-> *s_prefix), then publishes this tile's inclusive prefix.
// The inclusive prefixes travel along the tile sequence one window per L2 round trip, and with ~10^4 small tiles
// that chain is the kernel's critical path: the window is 128 tiles (4 independent loads per lane in flight) so
// the chain is ~80 hops instead of ~320.
__device__ __forceinline__ void s2_lookback(long long* s_prefix, int tile, int tile_total, int n_tiles, int lane,
                                            unsigned long long* __restrict__ tile_state, long long* __restrict__ total,
                                            uint32_t epoch) {
  long long prefix = 0;
  if (tile > 0) {
    int idx = tile - 1;   // nearest predecessor not yet accounted for
    const long long t0 = clock64();
    bool done = false;
    while (!done) {
      unsigned long long st[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int my = idx - 32 * k - lane;
        st[k] = (my >= 0) ? ld_volatile_u64(&tile_state[my]) : s2_pack(kS2FlagInc, epoch, 0);   // virtual predecessor of tile 0
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (done) break;
        int first_inc;
        while (true) {
          const uint32_t fl = s2_flag(st[k], epoch);
          const uint32_t ready = __ballot_sync(0xffffffffu, fl != 0);
          const uint32_t inc = __ballot_sync(0xffffffffu, fl == 2);
          first_inc = inc ? (__ffs(inc) - 1) : 32;   // lanes [0, first_inc] must all be ready
          const uint32_t need = (first_inc >= 31) ? 0xffffffffu : ((2u << first_inc) - 1u);
          if ((ready & need) == need) break;
          if (clock64() - t0 > ADN_WATCHDOG_CYCLES) asm volatile("trap;");
          const int my = idx - 32 * k - lane;
          if (my >= 0) st[k] = ld_volatile_u64(&tile_state[my]);
        }
        long long contrib = (lane <= first_inc) ? (long long)(st[k] & kS2ValMask) : 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, o);
        prefix += contrib;
        if (first_inc < 32) done = true;
      }
      idx -= 128;
    }
  }
  if (lane == 0) {
    atomicExch(&tile_state[tile], s2_pack(kS2FlagInc, epoch, prefix + tile_total));
    *s_prefix = prefix;
    if (tile == n_tiles - 1) *total = prefix + tile_total;
  }
}

__global__ void __launch_bounds__(kS2Threads)
stage2_kernel(const float* __restrict__ raw0, long long n_rays, float thr, const float* __restrict__ d_thr, int K,
              const float* __restrict__ zlut, int32_t* __restrict__ count, int32_t* __restrict__ offset,
              int32_t* __restrict__ cell_out, int32_t* __restrict__ ray_out, float* __restrict__ z_out,
              float* __restrict__ zp_out, long long* __restrict__ total, unsigned long long* __restrict__ tile_state,
              unsigned int* __restrict__ ticket, int n_tiles, uint32_t epoch, uint32_t ticket_base, bool aligned16) {
  __shared__ uint32_t s_sel[kS2Rays][4];
  __shared__ int s_cnt[kS2Rays];
  __shared__ int s_off[kS2Rays];
  __shared__ long long s_prefix;
  __shared__ int s_tile;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (d_thr) thr = *d_thr;   // threshold chosen on the device (sample budget)
  if (threadIdx.x == 0) s_tile = int(atomicAdd(ticket, 1u) - ticket_base);
  __syncthreads();
  const int tile = s_tile;
  const long long ray0 = (long long)tile * kS2Rays;

  // phase 1: selection (the warp's 8 row loads are issued up front: 8 x 512 B in flight per warp)
  float4 rows8[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const long long r = ray0 + warp * 8 + i;
    rows8[i] = (r < n_rays) ? ld_row_quad(raw0 + r * 128, lane, aligned16) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int rl = warp * 8 + i;
    const long long r = ray0 + rl;
    int cnt = 0;
    uint32_t sel[4] = {0, 0, 0, 0};
    if (r < n_rays) cnt = select_cells(rows8[i], thr, K, lane, sel);
    if (lane == 0) {
      s_cnt[rl] = cnt;
#pragma unroll
      for (int j = 0; j < 4; ++j) s_sel[rl][j] = sel[j];
    }
  }
  __syncthreads();

  // CTA scan + decoupled look-back (warp 0)
  if (warp == 0) {
    const int tile_total = s2_tile_scan(s_cnt, s_off, tile, lane, tile_state, epoch);
    s2_lookback(&s_prefix, tile, tile_total, n_tiles, lane, tile_state, total, epoch);
  }
  __syncthreads();
  const long long prefix = s_prefix;

  // phase 2: write the packed samples (ray-major, ascending cell)
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int rl = warp * 8 + i;
    const long long r = ray0 + rl;
    if (r >= n_rays) break;
    const float4 v4 = rows8[i];
    const float v[4] = {v4.x, v4.y, v4.z, v4.w};
    const long long off = prefix + s_off[rl];
    if (lane == 0) {
      count[r] = s_cnt[rl];
      offset[r] = int32_t(off);
    }
    const uint32_t below = (1u << lane) - 1u;
    int rank = 0;
    uint32_t sel[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      sel[j] = s_sel[rl][j];
      rank += __popc(sel[j] & below);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if ((sel[j] >> lane) & 1u) {
        const int cell = 4 * lane + j;
        const long long o = off + rank;
        z_out[o] = zlut[cell];
        zp_out[o] = v[j];
        if (cell_out) cell_out[o] = cell;
        ray_out[o] = int32_t(r);
        ++rank;
      }
    }
  }
}

// ---- thread-per-ray variant (K <= 16): the default path.
// The warp-per-ray kernel above spends ~480 warp instructions per ray once most rays overflow K (cross-lane pop rounds),
// which makes it issue bound at ~15 % of HBM.  Here every THREAD owns a ray, so each instruction advances 32 rays:
//   * the tile's 64 rows land in shared memory through cp.async (each warp fetches its own 32 rows, 512 B per
//     instruction); rows are padded to 33 x 16 B so that "thread t reads chunk c of row t" is bank-conflict free,
//   * a ray is 16 groups of 8 cells; the thread keeps the 16 group maxima (shared memory, 5 x 16 B per thread) and
//     runs up to K rounds of: max group (first on ties) -> first cell of that group holding the max -> record it,
//     overwrite it with -inf, refresh the group's maximum.  Round 0 is always taken (the arg-max fallback of
//     :748-749), later rounds only while the popped value is >= thr, so one loop covers "none", "<= K" and "> K"
//     survivors with the reference's order (value descending, ties lower cell first) and no per-case branches,
//   * picks are emitted in ascending cell order (rank = popcount of the selection mask below the cell) into a
//     shared staging area that aliases the dead rows, then copied out coalesced after the tile's look-back scan.
constexpr int kS2tRowBytes = 528;
constexpr int kS2tGmBytes = 0;    // group maxima live in registers
constexpr size_t kS2tSmemBytes = size_t(kS2Rays) * (kS2tRowBytes + kS2tGmBytes) + 128 * sizeof(float);

// Issues the copies of one tile's 64 rows into `rows` (stride kS2tRowBytes) and commits them; the caller waits
// (cp.async.wait_group 0 + __syncwarp) before it reads its row.  Each warp fetches the 32 rows its own threads own: one
// 512-byte row per cp.async instruction (16 B per lane, coalesced), nothing staged in registers, and only a __syncwarp
// between the copies and their consumers.  (A bulk copy per thread serialises into a 32-iteration uniform-register
// waterfall.)
__device__ __forceinline__ void s2t_fetch_rows(const float* __restrict__ raw0, long long n_rays, long long ray0, uint8_t* rows,
                                               int warp, int lane) {
  const float* src = raw0 + (ray0 + warp * 32) * 128 + lane * 4;
  const uint32_t dst = smem_u32(rows + (warp * 32) * kS2tRowBytes + lane * 16);
  const long long left = n_rays - (ray0 + warp * 32);
#pragma unroll 8
  for (int i = 0; i < 32; ++i) {
    if (i < left)
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + i * kS2tRowBytes), "l"(src + i * 128) : "memory");
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}

// The 16 group maxima (groups of 8 cells) of a staged row.
__device__ __forceinline__ void s2t_group_maxima(const uint8_t* row, float (&g)[16]) {
  const float4* row4 = reinterpret_cast<const float4*>(row);
  auto max8 = [](const float4 a, const float4 b) {
    return fmaxf(fmaxf(fmaxf(a.x, a.y), fmaxf(a.z, a.w)), fmaxf(fmaxf(b.x, b.y), fmaxf(b.z, b.w)));
  };
#pragma unroll
  for (int q = 0; q < 16; ++q) g[q] = max8(row4[2 * q], row4[2 * q + 1]);
}

// One pop round: returns the row's largest remaining value (ties: lowest cell) and its cell, and removes it (-inf in the
// row, refreshed group maximum).
__device__ __forceinline__ float s2t_pop(uint8_t* row, float (&g)[16], int& cell) {
  const float NEG = __int_as_float(0xff800000);
  const float m = fmaxf(fmaxf(fmaxf(fmaxf(g[0], g[1]), fmaxf(g[2], g[3])), fmaxf(fmaxf(g[4], g[5]), fmaxf(g[6], g[7]))),
                        fmaxf(fmaxf(fmaxf(g[8], g[9]), fmaxf(g[10], g[11])), fmaxf(fmaxf(g[12], g[13]), fmaxf(g[14], g[15]))));
  int gi = 0;
#pragma unroll
  for (int i = 15; i >= 0; --i) gi = (g[i] == m) ? i : gi;   // first group holding the maximum
  float* grp = reinterpret_cast<float*>(row) + 8 * gi;
  const float4 a = reinterpret_cast<const float4*>(grp)[0], b = reinterpret_cast<const float4*>(grp)[1];
  const float x[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  bool found = false;
  int idx = 0;
  float nm = NEG;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const bool e = (x[i] == m) && !found;    // first cell of the group holding the maximum
    found = found || e;
    idx = e ? i : idx;
    nm = fmaxf(nm, e ? NEG : x[i]);          // the group's maximum once that cell is gone
  }
  grp[idx] = NEG;
#pragma unroll
  for (int i = 0; i < 16; ++i) g[i] = (i == gi) ? nm : g[i];
  cell = 8 * gi + idx;
  return m;
}

template <int KMAX>
__global__ void __launch_bounds__(kS2Rays)
stage2_thread_kernel(const float* __restrict__ raw0, long long n_rays, float thr, const float* __restrict__ d_thr, int K,
                     const float* __restrict__ zlut, int32_t* __restrict__ count, int32_t* __restrict__ offset,
                     int32_t* __restrict__ cell_out, int32_t* __restrict__ ray_out, float* __restrict__ z_out,
                     float* __restrict__ zp_out, long long* __restrict__ total, unsigned long long* __restrict__ tile_state,
                     unsigned int* __restrict__ ticket, int n_tiles, uint32_t epoch, uint32_t ticket_base) {
  extern __shared__ __align__(16) uint8_t s2t_smem[];
  uint8_t* rows = s2t_smem;
  uint8_t* gms = rows + kS2Rays * kS2tRowBytes;
  float* zl = reinterpret_cast<float*>(gms + kS2Rays * kS2tGmBytes);
  __shared__ int s_cnt[kS2Rays];
  __shared__ int s_off[kS2Rays];
  __shared__ long long s_prefix;
  __shared__ int s_tile;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) s_tile = int(atomicAdd(ticket, 1u) - ticket_base);
  if (d_thr) thr = *d_thr;   // threshold chosen on the device (sample budget)
  __syncthreads();
  const int tile = s_tile;
  const long long ray0 = (long long)tile * kS2Rays;
  const long long r = ray0 + tid;
  const bool valid = r < n_rays;
  uint8_t* row = rows + tid * kS2tRowBytes;
  s2t_fetch_rows(raw0, n_rays, ray0, rows, warp, lane);
  zl[tid] = zlut[tid];
  zl[tid + 64] = zlut[tid + 64];
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncwarp();

  float g[16];   // group maxima, registers
  s2t_group_maxima(row, g);

  uint32_t mk0 = 0, mk1 = 0, mk2 = 0, mk3 = 0;   // selection mask over the 128 cells
  float mv[KMAX];                                 // popped values, pick order
  uint32_t cp[KMAX / 4];                          // popped cells, 8 bits each
#pragma unroll
  for (int j = 0; j < KMAX / 4; ++j) cp[j] = 0;
  int cnt = 0;
  bool active = valid;
#pragma unroll
  for (int j = 0; j < KMAX; ++j) {
    mv[j] = 0.0f;
    if (j >= K) break;                                        // warp uniform
    if (!__any_sync(0xffffffffu, active)) break;              // warp uniform
    int cell;
    const float m = s2t_pop(row, g, cell);
    const bool sel = active && (j == 0 || m >= thr);
    active = sel;
    const uint32_t bit = sel ? (1u << (cell & 31)) : 0u;
    const int w = cell >> 5;
    mk0 |= (w == 0) ? bit : 0u;
    mk1 |= (w == 1) ? bit : 0u;
    mk2 |= (w == 2) ? bit : 0u;
    mk3 |= (w == 3) ? bit : 0u;
    mv[j] = m;
    cp[j >> 2] |= uint32_t(cell) << (8 * (j & 3));
    cnt += sel ? 1 : 0;
  }

  s_cnt[tid] = cnt;
  __syncthreads();   // every thread is done with its row: the row area becomes the staging area
  int tile_total_w0 = 0;
  if (warp == 0) tile_total_w0 = s2_tile_scan(s_cnt, s_off, tile, lane, tile_state, epoch);
  __syncthreads();
  const int off = s_off[tid];

  float* st_z = reinterpret_cast<float*>(rows);
  float* st_zp = st_z + kS2Rays * KMAX;
  int32_t* st_ray = reinterpret_cast<int32_t*>(st_zp + kS2Rays * KMAX);
  int32_t* st_cell = st_ray + kS2Rays * KMAX;
  const int c0 = __popc(mk0), c1 = c0 + __popc(mk1), c2 = c1 + __popc(mk2);
#pragma unroll
  for (int j = 0; j < KMAX; ++j) {
    if (j < cnt) {
      const int cell = int((cp[j >> 2] >> (8 * (j & 3))) & 127u);
      const int w = cell >> 5;
      const uint32_t mk = (w == 0) ? mk0 : (w == 1) ? mk1 : (w == 2) ? mk2 : mk3;
      const int base = (w == 0) ? 0 : (w == 1) ? c0 : (w == 2) ? c1 : c2;
      const int p = off + base + __popc(mk & ((1u << (cell & 31)) - 1u));
      st_z[p] = zl[cell];
      st_zp[p] = mv[j];
      st_ray[p] = int32_t(r);
      st_cell[p] = cell;
    }
  }
  // the look-back (a chain of L2 round trips) starts only after this warp's own staging work is out of the way
  if (warp == 0) s2_lookback(&s_prefix, tile, tile_total_w0, n_tiles, lane, tile_state, total, epoch);
  __syncthreads();
  const long long prefix = s_prefix;
  if (valid) {
    count[r] = cnt;
    offset[r] = int32_t(prefix + off);
  }
  const int tile_total = s_off[kS2Rays - 1] + s_cnt[kS2Rays - 1];
  for (int i = tid; i < tile_total; i += kS2Rays) {
    const long long o = prefix + i;
    z_out[o] = st_z[i];
    zp_out[o] = st_zp[i];
    ray_out[o] = st_ray[i];
    if (cell_out) cell_out[o] = st_cell[i];
  }
}

// ---- D != 128 depth cells (multiDepthFeatures 32, 64 or 256): raw0 rows of D cells, D / 32 = C cells per lane.
// select_cells for C cells per lane (bit l of sel[j] <-> cell C l + j), same contract: >= thr, top K by value with ties to
// the lower cell, the arg-max cell when nothing passes.  Each pop round takes every lane's best remaining candidate (the
// lowest j on ties), one REDUX.MAX over those heads and a ballot (ties: the lowest lane).
template <int C>
__device__ __forceinline__ int select_cells_c(const float (&v)[C], float thr, int K, int lane, uint32_t (&sel)[C]) {
  uint32_t act[C];
  int cnt = 0;
#pragma unroll
  for (int j = 0; j < C; ++j) {
    act[j] = __ballot_sync(0xffffffffu, v[j] >= thr);
    cnt += __popc(act[j]);
  }
  if (cnt > 0 && cnt <= K) {
#pragma unroll
    for (int j = 0; j < C; ++j) sel[j] = act[j];
    return cnt;
  }
  const bool fallback = (cnt == 0);
  const int need = fallback ? 1 : K;
  uint32_t key[C];   // 0 = not a candidate (every real input has a key >= 0x007FFFFF)
#pragma unroll
  for (int j = 0; j < C; ++j) key[j] = (fallback || ((act[j] >> lane) & 1u)) ? order_key(v[j]) : 0u;
  uint32_t mine = 0;
  for (int round = 0; round < need; ++round) {
    uint32_t head = 0u;
    int hj = 0;
#pragma unroll
    for (int j = 0; j < C; ++j) {
      hj = key[j] > head ? j : hj;
      head = key[j] > head ? key[j] : head;
    }
    const uint32_t m = __reduce_max_sync(0xffffffffu, head);
    const uint32_t who = __ballot_sync(0xffffffffu, head == m);
    if (lane == __ffs(who) - 1) {
      mine |= 1u << hj;
#pragma unroll
      for (int j = 0; j < C; ++j) key[j] = j == hj ? 0u : key[j];
    }
  }
#pragma unroll
  for (int j = 0; j < C; ++j) sel[j] = __ballot_sync(0xffffffffu, (mine >> j) & 1u);
  return need;
}

// Lane `lane`'s C cells of a D = 32 C row (4-byte loads: any row alignment).
template <int C>
__device__ __forceinline__ void ld_row_cells(const float* __restrict__ row, int lane, float (&v)[C]) {
#pragma unroll
  for (int j = 0; j < C; ++j) v[j] = __ldg(row + C * lane + j);
}

// Stage 2 over raw0 [n_rays, 32 C]: stage2_kernel's warp-per-ray layout, scan and look-back, with C cells per lane.
template <int C>
__global__ void __launch_bounds__(kS2Threads)
stage2_cells_kernel(const float* __restrict__ raw0, long long n_rays, float thr, const float* __restrict__ d_thr, int K,
                    const float* __restrict__ zlut, int32_t* __restrict__ count, int32_t* __restrict__ offset,
                    int32_t* __restrict__ cell_out, int32_t* __restrict__ ray_out, float* __restrict__ z_out,
                    float* __restrict__ zp_out, long long* __restrict__ total, unsigned long long* __restrict__ tile_state,
                    unsigned int* __restrict__ ticket, int n_tiles, uint32_t epoch, uint32_t ticket_base) {
  constexpr int D = 32 * C;
  __shared__ uint32_t s_sel[kS2Rays][C];
  __shared__ int s_cnt[kS2Rays];
  __shared__ int s_off[kS2Rays];
  __shared__ long long s_prefix;
  __shared__ int s_tile;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (d_thr) thr = *d_thr;
  if (threadIdx.x == 0) s_tile = int(atomicAdd(ticket, 1u) - ticket_base);
  __syncthreads();
  const int tile = s_tile;
  const long long ray0 = (long long)tile * kS2Rays;

  float rows8[8][C];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const long long r = ray0 + warp * 8 + i;
#pragma unroll
    for (int j = 0; j < C; ++j) rows8[i][j] = 0.0f;
    if (r < n_rays) ld_row_cells<C>(raw0 + r * D, lane, rows8[i]);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int rl = warp * 8 + i;
    const long long r = ray0 + rl;
    int cnt = 0;
    uint32_t sel[C];
#pragma unroll
    for (int j = 0; j < C; ++j) sel[j] = 0u;
    if (r < n_rays) cnt = select_cells_c<C>(rows8[i], thr, K, lane, sel);
    if (lane == 0) {
      s_cnt[rl] = cnt;
#pragma unroll
      for (int j = 0; j < C; ++j) s_sel[rl][j] = sel[j];
    }
  }
  __syncthreads();

  if (warp == 0) {
    const int tile_total = s2_tile_scan(s_cnt, s_off, tile, lane, tile_state, epoch);
    s2_lookback(&s_prefix, tile, tile_total, n_tiles, lane, tile_state, total, epoch);
  }
  __syncthreads();
  const long long prefix = s_prefix;

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int rl = warp * 8 + i;
    const long long r = ray0 + rl;
    if (r >= n_rays) break;
    const long long off = prefix + s_off[rl];
    if (lane == 0) {
      count[r] = s_cnt[rl];
      offset[r] = int32_t(off);
    }
    const uint32_t below = (1u << lane) - 1u;
    int rank = 0;
    uint32_t sel[C];
#pragma unroll
    for (int j = 0; j < C; ++j) {
      sel[j] = s_sel[rl][j];
      rank += __popc(sel[j] & below);
    }
#pragma unroll
    for (int j = 0; j < C; ++j) {
      if ((sel[j] >> lane) & 1u) {
        const int cell = C * lane + j;
        const long long o = off + rank;
        z_out[o] = __ldg(zlut + cell);
        zp_out[o] = rows8[i][j];
        if (cell_out) cell_out[o] = cell;
        ray_out[o] = int32_t(r);
        ++rank;
      }
    }
  }
}

size_t stage2_scratch_bytes(long long n_rays) {
  const long long n_tiles = (n_rays + kS2Rays - 1) / kS2Rays;
  return size_t(n_tiles + 2) * 8;
}

cudaError_t launch_stage2(const float* d_raw0, long long n_rays, float thr, int K, const float* d_zlut, int32_t* d_count,
                          int32_t* d_offset, int32_t* d_cell, int32_t* d_ray, float* d_z, float* d_zp, long long* d_total,
                          void* d_scratch, Stage2Sync* sync, cudaStream_t s, const float* d_thr, int D) {
  if (n_rays <= 0) return cudaMemsetAsync(d_total, 0, sizeof(long long), s);
  if (D != 32 && D != 64 && D != 128 && D != 256) return cudaErrorInvalidValue;
  const int n_tiles = int((n_rays + kS2Rays - 1) / kS2Rays);
  const size_t bytes = stage2_scratch_bytes(n_rays);
  // [ticket | states]: cleared only when the buffer is new / has grown or the epoch wraps (see the state-word comment)
  sync->epoch = (sync->epoch + 1) & kS2EpochMask;
  if (sync->scratch != d_scratch || sync->cleared_bytes < bytes || sync->epoch == 0) {
    cudaError_t e = cudaMemsetAsync(d_scratch, 0, bytes, s);
    if (e != cudaSuccess) return e;
    sync->scratch = d_scratch;
    sync->cleared_bytes = bytes;
    sync->epoch = 1;
    sync->ticket_base = 0;
  }
  unsigned int* ticket = reinterpret_cast<unsigned int*>(d_scratch);
  unsigned long long* state = reinterpret_cast<unsigned long long*>(d_scratch) + 1;
  const uint32_t epoch = sync->epoch, base = sync->ticket_base;
  sync->ticket_base += uint32_t(n_tiles);   // the launch consumes exactly n_tiles tickets (unsigned wrap-around is fine)
  // thread-per-ray kernel whenever its assumptions hold (K <= 16, 16-byte aligned rows for the cp.async fetch)
  const bool aligned = (reinterpret_cast<uintptr_t>(d_raw0) & 15u) == 0;
#define ADN_S2_CELLS(C)                                                                                                       \
  stage2_cells_kernel<C><<<n_tiles, kS2Threads, 0, s>>>(d_raw0, n_rays, thr, d_thr, K, d_zlut, d_count, d_offset, d_cell, d_ray, \
                                                        d_z, d_zp, d_total, state, ticket, n_tiles, epoch, base)
  if (D == 32) ADN_S2_CELLS(1);
  else if (D == 64) ADN_S2_CELLS(2);
  else if (D == 256) ADN_S2_CELLS(8);
#undef ADN_S2_CELLS
  else if (K <= 8 && aligned)
    stage2_thread_kernel<8><<<n_tiles, kS2Rays, kS2tSmemBytes, s>>>(d_raw0, n_rays, thr, d_thr, K, d_zlut, d_count, d_offset, d_cell,
                                                                   d_ray, d_z, d_zp, d_total, state, ticket, n_tiles, epoch, base);
  else if (K <= 16 && aligned)
    stage2_thread_kernel<16><<<n_tiles, kS2Rays, kS2tSmemBytes, s>>>(d_raw0, n_rays, thr, d_thr, K, d_zlut, d_count, d_offset, d_cell,
                                                                    d_ray, d_z, d_zp, d_total, state, ticket, n_tiles, epoch, base);
  else
    stage2_kernel<<<n_tiles, kS2Threads, 0, s>>>(d_raw0, n_rays, thr, d_thr, K, d_zlut, d_count, d_offset, d_cell, d_ray, d_z, d_zp,
                                                 d_total, state, ticket, n_tiles, epoch, base, aligned);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------- sample budget
// The smallest threshold t* >= thr_min whose sample count M(t*) is at most B = max_samples, with no host round trip.
// For t > 0 stage 2 gives ray r  n_r(t) = clamp(#{cells >= t}, 1, K)  samples (src/nerf_raymarch_common.py:726-749), so
//   M(t) = N + #{(r, j) : 2 <= j <= K, v_r^(j) >= t},   v_r^(j) = the j-th largest raw0 value of ray r (ties counted),
// and with S = the multiset of those rank-2..K values that are >= thr_min and Q = B - N:
//   |S| <= Q -> t* = thr_min,   else t* = nextafterf(s_(Q+1), +inf), s_(Q+1) = the (Q+1)-th largest element of S.
// S is positive, so float order is uint32 bit order: S is written as keys (0 = no entry) and the (Q+1)-th largest key is
// found by a radix select over bits [31:21], [20:10], [9:0]; the first histogram is folded into the extraction pass.
// Histograms use integer atomics (order independent), so t* is deterministic.
//
// The global histograms are uint64 words, and round 0 carries one more word, the call's ray count N (q = B - N is formed
// on the device from it).  Integer sums do not depend on order, so members of a budget group (BudgetGroup) that add each
// round's words across all members before its select all narrow to the same prefix: the t* of one call over every
// member's rays.  Work layout: round 0 [kBudgetBins bins | N], round 1 [kBudgetBins], round 2 [kBudgetBins], BudgetState.
constexpr int kBudgetBins = 2048;
constexpr int kBudgetWords0 = kBudgetBins + 1;
struct BudgetState {
  unsigned long long k;   // rank still sought inside the current prefix (1 = largest)
  uint32_t prefix;        // key bits fixed so far
  uint32_t done;          // 1: |S| <= Q, t* = thr_min
};
__host__ __device__ constexpr int budget_round_offset(int round) { return round == 0 ? 0 : kBudgetWords0 + (round - 1) * kBudgetBins; }
size_t budget_work_bytes() { return size_t(budget_round_offset(3)) * 8 + sizeof(BudgetState); }

// Adds the CTA's histogram into the global one; CTA 0 also stores the call's ray count (the round-0 histogram's last word).
__device__ __forceinline__ void budget_flush_hist(const uint32_t* s_hist, unsigned long long* __restrict__ hist, long long n_rays = -1) {
  for (int b = threadIdx.x; b < kBudgetBins; b += blockDim.x)
    if (s_hist[b]) atomicAdd(hist + b, (unsigned long long)s_hist[b]);
  if (n_rays >= 0 && blockIdx.x == 0 && threadIdx.x == 0) hist[kBudgetBins] = (unsigned long long)n_rays;
}

// K <= 16: thread per ray, the group-maximum pop rounds of stage2_thread_kernel; pops 1..K-1 that are >= thr_min are the
// ray's keys.  Keys are staged in the dead row area and written out coalesced; CTAs loop over tiles so the histogram is
// flushed once per CTA.
__global__ void __launch_bounds__(kS2Rays)
budget_keys_thread_kernel(const float* __restrict__ raw0, long long n_rays, float thr_min, int K, uint32_t* __restrict__ keys,
                          unsigned long long* __restrict__ hist) {
  __shared__ __align__(16) uint8_t rows[kS2Rays * kS2tRowBytes];
  __shared__ uint32_t s_hist[kBudgetBins];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int KM1 = K - 1;
  for (int b = tid; b < kBudgetBins; b += kS2Rays) s_hist[b] = 0;
  const long long n_tiles = (n_rays + kS2Rays - 1) / kS2Rays;
  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long ray0 = tile * kS2Rays;
    __syncthreads();   // the previous tile's staged keys have been written out
    s2t_fetch_rows(raw0, n_rays, ray0, rows, warp, lane);
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncwarp();
    uint8_t* row = rows + tid * kS2tRowBytes;
    float g[16];
    s2t_group_maxima(row, g);
    uint32_t key[15];
    bool active = ray0 + tid < n_rays;
    int cell;
    s2t_pop(row, g, cell);   // rank 1: every ray keeps one sample whatever the threshold
#pragma unroll
    for (int j = 0; j < 15; ++j) {
      key[j] = 0u;
      if (j >= KM1) continue;                                   // uniform
      if (!__any_sync(0xffffffffu, active)) continue;          // warp uniform
      const float m = s2t_pop(row, g, cell);
      active = active && m >= thr_min;
      key[j] = active ? __float_as_uint(m) : 0u;
    }
    __syncthreads();   // every row is consumed: the row area becomes the staging area
    uint32_t* st = reinterpret_cast<uint32_t*>(rows);
#pragma unroll
    for (int j = 0; j < 15; ++j) {
      if (j < KM1) st[tid * KM1 + j] = key[j];
      if (key[j]) atomicAdd(&s_hist[key[j] >> 21], 1u);
    }
    __syncthreads();
    const long long n_out = min((long long)kS2Rays, n_rays - ray0) * KM1;
    for (int i = tid; i < n_out; i += kS2Rays) keys[ray0 * KM1 + i] = st[i];
  }
  __syncthreads();
  budget_flush_hist(s_hist, hist, n_rays);
}

// 16 < K <= 128: warp per ray with stage 2's select_cells; the selected cells minus one instance of
// the largest value are the ray's keys (none when no cell reaches thr_min).
__global__ void __launch_bounds__(kS2Threads)
budget_keys_warp_kernel(const float* __restrict__ raw0, long long n_rays, float thr_min, int K, uint32_t* __restrict__ keys,
                        unsigned long long* __restrict__ hist) {
  __shared__ uint32_t s_hist[kBudgetBins];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int b = threadIdx.x; b < kBudgetBins; b += kS2Threads) s_hist[b] = 0;
  __syncthreads();
  const int KM1 = K - 1;
  const long long step = (long long)gridDim.x * (kS2Threads / 32);
  for (long long r = blockIdx.x * (long long)(kS2Threads / 32) + warp; r < n_rays; r += step) {
    const float4 v4 = __ldg(reinterpret_cast<const float4*>(raw0 + r * 128) + lane);
    const float v[4] = {v4.x, v4.y, v4.z, v4.w};
    uint32_t sel[4];
    const int cnt = select_cells(v4, thr_min, K, lane, sel);
    int n_keys = 0;
    if (__any_sync(0xffffffffu, v[0] >= thr_min || v[1] >= thr_min || v[2] >= thr_min || v[3] >= thr_min)) {
      // drop one instance of the largest selected value (lowest lane, then lowest j)
      uint32_t best = 0u;
      int bj = 0;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t k = ((sel[j] >> lane) & 1u) ? __float_as_uint(v[j]) : 0u;
        bj = k > best ? j : bj;
        best = k > best ? k : best;
      }
      const uint32_t m = __reduce_max_sync(0xffffffffu, best);
      const int who = __ffs(__ballot_sync(0xffffffffu, best == m)) - 1;
      if (lane == who) sel[bj] &= ~(1u << lane);
#pragma unroll
      for (int j = 0; j < 4; ++j) sel[j] = __shfl_sync(0xffffffffu, sel[j], who);
      const uint32_t below = (1u << lane) - 1u;
      int base = 0;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if ((sel[j] >> lane) & 1u) {
          const uint32_t k = __float_as_uint(v[j]);
          keys[r * KM1 + base + __popc(sel[j] & below)] = k;
          atomicAdd(&s_hist[k >> 21], 1u);
        }
        base += __popc(sel[j]);
      }
      n_keys = cnt - 1;
    }
    for (int p = n_keys + lane; p < KM1; p += 32) keys[r * KM1 + p] = 0u;
  }
  __syncthreads();
  budget_flush_hist(s_hist, hist, n_rays);
}

// budget_keys_warp_kernel over raw0 [n_rays, 32 C] (D != 128), every K: select_cells_c at thr_min, one instance of the
// largest selected value dropped, the rest the ray's keys.
template <int C>
__global__ void __launch_bounds__(kS2Threads)
budget_keys_cells_kernel(const float* __restrict__ raw0, long long n_rays, float thr_min, int K, uint32_t* __restrict__ keys,
                         unsigned long long* __restrict__ hist) {
  constexpr int D = 32 * C;
  __shared__ uint32_t s_hist[kBudgetBins];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int b = threadIdx.x; b < kBudgetBins; b += kS2Threads) s_hist[b] = 0;
  __syncthreads();
  const int KM1 = K - 1;
  const long long step = (long long)gridDim.x * (kS2Threads / 32);
  for (long long r = blockIdx.x * (long long)(kS2Threads / 32) + warp; r < n_rays; r += step) {
    float v[C];
    ld_row_cells<C>(raw0 + r * D, lane, v);
    uint32_t sel[C];
    const int cnt = select_cells_c<C>(v, thr_min, K, lane, sel);
    bool any = false;
#pragma unroll
    for (int j = 0; j < C; ++j) any = any || v[j] >= thr_min;
    int n_keys = 0;
    if (__any_sync(0xffffffffu, any)) {
      uint32_t best = 0u;
      int bj = 0;
#pragma unroll
      for (int j = 0; j < C; ++j) {
        const uint32_t k = ((sel[j] >> lane) & 1u) ? __float_as_uint(v[j]) : 0u;
        bj = k > best ? j : bj;
        best = k > best ? k : best;
      }
      const uint32_t m = __reduce_max_sync(0xffffffffu, best);
      const int who = __ffs(__ballot_sync(0xffffffffu, best == m)) - 1;
#pragma unroll
      for (int j = 0; j < C; ++j) {
        if (lane == who && j == bj) sel[j] &= ~(1u << lane);
        sel[j] = __shfl_sync(0xffffffffu, sel[j], who);
      }
      const uint32_t below = (1u << lane) - 1u;
      int base = 0;
#pragma unroll
      for (int j = 0; j < C; ++j) base += __popc(sel[j] & below);
#pragma unroll
      for (int j = 0; j < C; ++j) {
        if ((sel[j] >> lane) & 1u) {
          const uint32_t k = __float_as_uint(v[j]);
          keys[r * KM1 + base] = k;
          atomicAdd(&s_hist[k >> 21], 1u);
          ++base;
        }
      }
      n_keys = cnt - 1;
    }
    for (int p = n_keys + lane; p < KM1; p += 32) keys[r * KM1 + p] = 0u;
  }
  __syncthreads();
  budget_flush_hist(s_hist, hist, n_rays);
}

// Rounds 1 and 2 of the select: histogram of the next key bits over the keys that carry the current prefix.
__global__ void __launch_bounds__(256)
budget_hist_kernel(const uint32_t* __restrict__ keys, long long n_keys, const BudgetState* __restrict__ st, int round,
                   unsigned long long* __restrict__ hist) {
  __shared__ uint32_t s_hist[kBudgetBins];
  if (st->done) return;   // uniform
  const uint32_t prefix = st->prefix;
  const int match_shift = round == 1 ? 21 : 10, bin_shift = round == 1 ? 10 : 0;
  const uint32_t mask = round == 1 ? 2047u : 1023u;
  for (int b = threadIdx.x; b < kBudgetBins; b += 256) s_hist[b] = 0;
  __syncthreads();
  auto add = [&](uint32_t k) {
    if (k && (k >> match_shift) == prefix) atomicAdd(&s_hist[(k >> bin_shift) & mask], 1u);
  };
  const long long n4 = n_keys >> 2;
  const uint4* k4 = reinterpret_cast<const uint4*>(keys);
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n4; i += 256ll * gridDim.x) {
    const uint4 v = __ldg(k4 + i);
    add(v.x);
    add(v.y);
    add(v.z);
    add(v.w);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n_keys & 3)) add(keys[4 * n4 + threadIdx.x]);
  __syncthreads();
  budget_flush_hist(s_hist, hist);
}

// One CTA: finds the bin of the k-th largest key (descending scan over the bins) and narrows the prefix.  Round 0 also
// decides |S| <= Q, Q = max(B - N, 0) with N the ray count word; round 2 fixes the last bits and writes t*.
__global__ void __launch_bounds__(1024)
budget_select_kernel(const unsigned long long* __restrict__ hist_all, BudgetState* __restrict__ st, int round,
                     unsigned long long max_samples, float thr_min, float* __restrict__ d_thr) {
  __shared__ unsigned long long s_warp[32];
  if (round > 0 && st->done) return;   // uniform
  const unsigned long long* hist = hist_all + budget_round_offset(round);
  const int nb = round == 2 ? 1024 : 2048, per = nb / 1024;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned long long n = hist_all[kBudgetBins], q = max_samples > n ? max_samples - n : 0ull;
  const unsigned long long k = round == 0 ? q + 1 : st->k;
  unsigned long long s = 0;
  for (int u = 0; u < per; ++u) s += hist[nb - 1 - (tid * per + u)];   // thread 0 owns the highest bins
  unsigned long long x = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) s_warp[warp] = x;
  __syncthreads();
  if (warp == 0) {
    unsigned long long w = s_warp[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    s_warp[lane] = w;   // inclusive over warps
  }
  __syncthreads();
  const unsigned long long incl = x + (warp > 0 ? s_warp[warp - 1] : 0ull), total = s_warp[31];
  if (round == 0 && total < k) {   // every candidate fits: the floor threshold itself
    if (tid == 0) {
      st->done = 1u;
      *d_thr = thr_min;
    }
    return;
  }
  unsigned long long excl = incl - s;
  if (excl < k && k <= incl) {     // exactly one thread
    for (int u = 0; u < per; ++u) {
      const uint32_t b = uint32_t(nb - 1 - (tid * per + u));
      const unsigned long long c = hist[b];
      if (k <= excl + c) {
        const uint32_t prefix = (st->prefix << (round == 2 ? 10 : 11)) | b;
        st->prefix = prefix;
        st->k = k - excl;
        // nextafterf(s_(Q+1), +inf) of a positive float (+inf stays +inf)
        if (round == 2) *d_thr = __uint_as_float(prefix >= 0x7f800000u ? 0x7f800000u : prefix + 1u);
        break;
      }
      excl += c;
    }
  }
}

cudaError_t launch_budget_threshold(const float* d_raw0, long long n_rays, float thr_min, int K, long long max_samples,
                                    uint32_t* d_keys, void* d_work, float* d_thr, int num_sms, cudaStream_t s, int* launches,
                                    BudgetGroup* group, int D) {
  if (D != 32 && D != 64 && D != 128 && D != 256) return cudaErrorInvalidValue;
  unsigned long long* hist = static_cast<unsigned long long*>(d_work);
  BudgetState* st = reinterpret_cast<BudgetState*>(hist + budget_round_offset(3));
  const bool grouped = group && group->fn;
  if (group) group->failed_round = -1;
  cudaError_t e = cudaMemsetAsync(d_work, 0, budget_work_bytes(), s);
  if (e != cudaSuccess) return e;
  // every round's words summed across the group, in place, ordered on s
  auto reduce = [&](int round) {
    if (!grouped) return true;
    if ((e = cudaGetLastError()) != cudaSuccess) return false;
    group->status = group->fn(group->user, reinterpret_cast<uint64_t*>(hist + budget_round_offset(round)), round == 0 ? kBudgetWords0 : kBudgetBins, s);
    if (group->status != 0) group->failed_round = round;
    return group->status == 0;
  };
  const long long n_keys = n_rays * (K - 1);
  // a group member runs every kernel and every reduction even without candidates: the others wait for its words
  const bool select_all = n_keys > 0 || grouped;
  int n = 0;
  if (select_all) {
    const unsigned warp_grid = unsigned(std::max(1ll, std::min<long long>((n_rays + kS2Threads / 32 - 1) / (kS2Threads / 32), 8ll * num_sms)));
    if (D == 32) {
      budget_keys_cells_kernel<1><<<warp_grid, kS2Threads, 0, s>>>(d_raw0, n_rays, thr_min, K, d_keys, hist);
    } else if (D == 64) {
      budget_keys_cells_kernel<2><<<warp_grid, kS2Threads, 0, s>>>(d_raw0, n_rays, thr_min, K, d_keys, hist);
    } else if (D == 256) {
      budget_keys_cells_kernel<8><<<warp_grid, kS2Threads, 0, s>>>(d_raw0, n_rays, thr_min, K, d_keys, hist);
    } else if (K <= 16) {
      const long long n_tiles = (n_rays + kS2Rays - 1) / kS2Rays;
      budget_keys_thread_kernel<<<unsigned(std::max(1ll, std::min<long long>(n_tiles, 5ll * num_sms))), kS2Rays, 0, s>>>(
          d_raw0, n_rays, thr_min, K, d_keys, hist);
    } else {
      const long long blocks = (n_rays + kS2Threads / 32 - 1) / (kS2Threads / 32);
      budget_keys_warp_kernel<<<unsigned(std::max(1ll, std::min<long long>(blocks, 8ll * num_sms))), kS2Threads, 0, s>>>(
          d_raw0, n_rays, thr_min, K, d_keys, hist);
    }
    ++n;
  }
  if (!reduce(0)) {
    if (launches) *launches += n;
    return e;
  }
  budget_select_kernel<<<1, 1024, 0, s>>>(hist, st, 0, (unsigned long long)max_samples, thr_min, d_thr);
  ++n;
  if (select_all) {
    const unsigned grid = unsigned(std::max<long long>(1, std::min<long long>((n_keys / 4 + 255) / 256, 4ll * num_sms)));
    for (int round = 1; round <= 2; ++round) {
      budget_hist_kernel<<<grid, 256, 0, s>>>(d_keys, n_keys, st, round, hist + budget_round_offset(round));
      if (!reduce(round)) {
        if (launches) *launches += n + 1;
        return e;
      }
      budget_select_kernel<<<1, 1024, 0, s>>>(hist, st, round, (unsigned long long)max_samples, thr_min, d_thr);
      n += 2;
    }
  }
  if (launches) *launches += n;
  return cudaGetLastError();
}

__global__ void stage2_dense_kernel(long long n_rays, int K, int32_t* __restrict__ count, int32_t* __restrict__ offset,
                                    long long* __restrict__ total) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i == 0) *total = n_rays * K;
  if (i >= n_rays) return;
  if (count) count[i] = K;
  if (offset) offset[i] = int32_t(i * K);
}

cudaError_t launch_stage2_dense(long long n_rays, int K, int32_t* d_count, int32_t* d_offset, long long* d_total,
                                cudaStream_t s) {
  const long long n = n_rays > 0 ? n_rays : 1;
  stage2_dense_kernel<<<unsigned((n + 255) / 256), 256, 0, s>>>(n_rays, K, d_count, d_offset, d_total);
  return cudaGetLastError();
}

// LinearlySpacedZNearZFar(NoDepthRange).generate with det = True (src/nerf_raymarch_common.py:276-326): every ray takes
// the same K depths zt [K].  One thread per sample (N K < 2^31), in pdf_sample_kernel's packed layout.
__global__ void __launch_bounds__(256)
linear_sample_kernel(int n_rays, int K, const float* __restrict__ zt, int32_t* __restrict__ count, int32_t* __restrict__ offset,
                     int32_t* __restrict__ ray, float* __restrict__ z, long long* __restrict__ total) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0 && total) *total = (long long)n_rays * K;
  if (i >= n_rays * K) return;
  const int r = i / K, k = i - r * K;
  z[i] = __ldg(zt + k);
  if (ray) ray[i] = r;
  if (k == 0) {
    if (count) count[r] = K;
    if (offset) offset[r] = i;
  }
}

cudaError_t launch_linear_sample(long long n_rays, int K, const float* d_zt, int32_t* d_count, int32_t* d_offset, int32_t* d_ray,
                                 float* d_z, long long* d_total, cudaStream_t s) {
  const long long n = n_rays * K > 0 ? n_rays * K : 1;   // an empty call still writes *d_total = 0
  linear_sample_kernel<<<unsigned((n + 255) / 256), 256, 0, s>>>(int(n_rays), K, d_zt, d_count, d_offset, d_ray, d_z, d_total);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------- sampling-network view
// The viewer's render-oracle picture (samplesToImage, adanerf_real_time_viewer/src/cuda/base_cuda_kernels.cu:487-528): per
// ray the three cells c0, c1, c2 that come first when the 128 raw0 values are sorted in descending order by
// cub::BlockRadixSort (stable), drawn as (c + 0.5) / 128.  Radix order is the order of the twiddled uint32 keys; the CUB of
// CUDA 12.x ranks -0 as +0 (cub/block/radix_rank_sort_operations.cuh, ProcessFloatMinusZero), so a positive NaN ranks above
// +inf, a negative NaN below -inf, and equal keys keep the lower cell first.  Nothing is sorted here: one thread per ray
// (rows staged like stage2_thread_kernel's) runs three pop rounds over the 16 group maxima of its keys.
__device__ __forceinline__ uint32_t view_key(float v) {
  const uint32_t b = __float_as_uint(v);
  const uint32_t k = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
  return k == 0x7fffffffu ? 0x80000000u : k;   // -0 -> +0
}

__device__ __forceinline__ void view_group_keys(const uint8_t* row, int q, uint32_t (&x)[8]) {
  const float4 a = reinterpret_cast<const float4*>(row)[2 * q], b = reinterpret_cast<const float4*>(row)[2 * q + 1];
  x[0] = view_key(a.x), x[1] = view_key(a.y), x[2] = view_key(a.z), x[3] = view_key(a.w);
  x[4] = view_key(b.x), x[5] = view_key(b.y), x[6] = view_key(b.z), x[7] = view_key(b.w);
}

__global__ void __launch_bounds__(kS2Rays)
sampling_view_kernel(const float* __restrict__ raw0, long long n_rays, float* __restrict__ rgb, uchar4* __restrict__ rgba8) {
  extern __shared__ __align__(16) uint8_t sv_smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long long ray0 = (long long)blockIdx.x * kS2Rays;
  const long long r = ray0 + tid;
  s2t_fetch_rows(raw0, n_rays, ray0, sv_smem, warp, lane);
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncwarp();
  if (r >= n_rays) return;
  const uint8_t* row = sv_smem + tid * kS2tRowBytes;

  uint32_t g[16];   // group maxima of the keys (groups of 8 cells)
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    uint32_t x[8];
    view_group_keys(row, q, x);
    g[q] = max(max(max(x[0], x[1]), max(x[2], x[3])), max(max(x[4], x[5]), max(x[6], x[7])));
  }
  int cell[3] = {-1, -1, -1};
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    uint32_t m = g[0];
#pragma unroll
    for (int q = 1; q < 16; ++q) m = max(m, g[q]);
    int gi = 0;
#pragma unroll
    for (int q = 15; q >= 0; --q) gi = (g[q] == m) ? q : gi;   // first group holding the maximum
    uint32_t x[8];
    view_group_keys(row, gi, x);
    // the first cell of that group holding the maximum that is not taken yet, and the group's maximum without it (at most
    // two of its eight cells are taken, so it keeps one)
    bool found = false;
    int idx = 0;
    uint32_t nm = 0u;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = 8 * gi + i;
      const bool taken = (c == cell[0]) || (c == cell[1]);
      const bool e = !taken && !found && x[i] == m;
      found = found || e;
      idx = e ? i : idx;
      nm = (taken || e) ? nm : max(nm, x[i]);
    }
#pragma unroll
    for (int q = 0; q < 16; ++q) g[q] = (q == gi) ? nm : g[q];
    cell[j] = 8 * gi + idx;
  }
  float v[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) v[j] = (0.5f + float(cell[j])) / 128.0f;
  if (rgb) {
    rgb[3 * r] = v[0];
    rgb[3 * r + 1] = v[1];
    rgb[3 * r + 2] = v[2];
  }
  // clamp(v, 0, 1) * 255 converted to unsigned char (truncation), alpha 255: base_cuda_kernels.cu:522-526
  if (rgba8)
    rgba8[r] = make_uchar4((unsigned char)(__saturatef(v[0]) * 255.0f), (unsigned char)(__saturatef(v[1]) * 255.0f),
                           (unsigned char)(__saturatef(v[2]) * 255.0f), 255);
}

cudaError_t launch_sampling_view(const float* d_raw0, long long n_rays, float* d_rgb, uint8_t* d_rgba8, cudaStream_t s) {
  if (n_rays <= 0) return cudaSuccess;
  const long long n_tiles = (n_rays + kS2Rays - 1) / kS2Rays;
  sampling_view_kernel<<<unsigned(n_tiles), kS2Rays, size_t(kS2Rays) * kS2tRowBytes, s>>>(d_raw0, n_rays, d_rgb,
                                                                                        reinterpret_cast<uchar4*>(d_rgba8));
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------- stage 3
// RayMarchFromPoses.batch (src/features.py:458-479): one thread per packed sample.  RT == false: posEnc 10-4 at compile
// time.  RT == true: sc.n_freq_pos (<= 20) and sc.n_freq_dir (<= 10) bands, the features written one at a time into x1
// and the tile image, so no thread holds its up to 123 + 63 features at once.
template <bool RT>
__global__ void __launch_bounds__(128)
stage3_kernel(const __grid_constant__ SceneDev sc, const float* __restrict__ ray_o, const float* __restrict__ ray_d,
              const int32_t* __restrict__ ray_idx, const float* __restrict__ z, const float* __restrict__ zlut_dense, int K,
              long long n_samples_host, const long long* __restrict__ n_samples_dev, float* __restrict__ x1,
              uint8_t* __restrict__ tiles1) {
  const long long n_samples = n_samples_dev ? *n_samples_dev : n_samples_host;
  const long long n_pad = ((n_samples + kTileM - 1) / kTileM) * kTileM;
  const int n_p = RT ? 3 + 6 * sc.n_freq_pos : 3 + 6 * kNFreqPos;
  const int n_v = RT ? 3 + 6 * sc.n_freq_dir : 3 + 6 * kNFreqDir;
  const TileFormat fmt = shading_tiles(n_p, n_v);
  extern __shared__ __align__(1024) uint8_t s_tile[];
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_pad; i += (long long)gridDim.x * blockDim.x) {
    float f[RT ? 1 : kFeat];
    if (!RT) {
#pragma unroll
      for (int j = 0; j < kFeat; ++j) f[j] = 0.0f;
    }
    if (RT && tiles1) {
      if (threadIdx.x == 0) bulk_wait_read_all();   // the previous tile's copy has finished reading s_tile
      __syncthreads();
      zero_row(fmt, s_tile, threadIdx.x, 0, fmt.n_blk);
    }
    if (i < n_samples) {
      long long r;
      float zw;
      if (ray_idx) {
        r = ray_idx[i];
        zw = z[i];
      } else {
        r = i / K;
        zw = zlut_dense[i - r * K];
      }
      float pos[3], d[3];
      sample_inputs(sc, sc.ndc != 0, ray_o, ray_d, r, zw, pos, d);
      if (RT) {
        const int vb = fmt.n_blk - 1;   // the view block
        posenc3_rt(pos, sc.n_freq_pos, [&](int j, float v) {   // position block FIRST (:473-479)
          if (x1) x1[i * (n_p + n_v) + j] = v;
          if (tiles1) put_feature(fmt, s_tile, j >> 6, threadIdx.x, j & 63, v);
        });
        posenc3_rt(d, sc.n_freq_dir, [&](int j, float v) {
          if (x1) x1[i * (n_p + n_v) + n_p + j] = v;
          if (tiles1) put_feature(fmt, s_tile, vb, threadIdx.x, j, v);
        });
      } else {
        posenc3<kNFreqPos>(pos, f);                      // 63: position block FIRST (:473-479)
        posenc3<kNFreqDir>(d, f + 63);                   // 27
        if (x1) {
#pragma unroll
          for (int j = 0; j < kFeat; ++j) x1[i * kFeat + j] = f[j];
        }
      }
    }
    if (tiles1) {   // the CTA's 128 samples are one tile of the shading net's input
      uint8_t* dst = tiles1 + size_t(i >> 7) * fmt.tile_bytes();
      if (RT) {
        flush_tile(fmt, s_tile, dst);
      } else {
        if (threadIdx.x == 0) bulk_wait_read_all();   // the previous tile's copy has finished reading s_tile
        __syncthreads();
        store_tile(fmt, f, s_tile, dst);
      }
    }
  }
  if (tiles1) store_tiles_drain();
}

cudaError_t launch_stage3(const SceneDev& sc, const float* d_ray_o, const float* d_ray_d, const int32_t* d_ray,
                          const float* d_z, const float* d_zlut_dense, int K, long long n_samples, const long long* d_total,
                          float* d_x1, uint8_t* d_tiles1, int num_sms, cudaStream_t s) {
  // n_samples is an upper bound (capacity) when d_total is given
  if (n_samples <= 0) return cudaSuccess;
  long long blocks = (n_samples + kTileM - 1) / kTileM;
  const long long cap = 64ll * num_sms;
  if (d_total && blocks > cap) blocks = cap;   // grid-stride when the true count lives on the device
  const int tile_bytes = 3 * kBlkBytes;        // the largest shading tile
  const size_t smem = d_tiles1 ? shading_tiles(3 + 6 * sc.n_freq_pos, 3 + 6 * sc.n_freq_dir).tile_bytes() : 0;
  static unsigned long long attr_done[2] = {0, 0};   // per device
  auto run = [&](auto kernel, unsigned long long* attr) -> cudaError_t {
    if (set_max_dyn_smem_once(reinterpret_cast<const void*>(kernel), tile_bytes, attr) != cudaSuccess) return cudaGetLastError();
    kernel<<<unsigned(blocks), 128, smem, s>>>(sc, d_ray_o, d_ray_d, d_ray, d_z, d_zlut_dense, K, n_samples, d_total, d_x1, d_tiles1);
    return cudaGetLastError();
  };
  if (sc.n_freq_pos == kNFreqPos && sc.n_freq_dir == kNFreqDir) return run(stage3_kernel<false>, &attr_done[0]);
  return run(stage3_kernel<true>, &attr_done[1]);
}

// ------------------------------------------------------------------------------------- stage 5
// adaptive_raw2outputs (src/nerf_raymarch_common.py:91-144), accumulation_mult == "alpha".
__device__ __forceinline__ float sigmoidf_acc(float x) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x))); }

// adaptive_cuda_kernels.cu:846-851: clamp(x, 0, 1) * 255 truncated, alpha = 255.  nvcc compiles helper_math.h:748's
// clamp, fmaxf(0, fminf(x, 1)), to one saturating add (FADD.SAT), which maps NaN to +0 where the C semantics of the
// source would give 1; the viewer's pixels are what the compiled kernel writes, so this states the saturate explicitly.
__device__ __forceinline__ uint32_t rgba8_channel(float x) { return uint32_t(__saturatef(x) * 255.0f); }

__device__ __forceinline__ uint32_t to_rgba8(float r, float g, float b) {
  return rgba8_channel(r) | (rgba8_channel(g) << 8) | (rgba8_channel(b) << 16) | (255u << 24);
}

// z_vals of a live sample (features.py:546-547): the reference scatters the packed z into a zero-filled [N,K] tensor and
// then sets every slot == 0 to NaN, so a live sample at z = +-0 is NaN too.  Dense mode stores z_vals unchanged.
__device__ __forceinline__ float s5_z_val(float z) { return z == 0.0f ? __int_as_float(0x7fc00000) : z; }

// Per-ray epilogue shared by both composite kernels: acc / disparity / log-warped depth (src/nerf_raymarch_common.py:137-139,
// src/util/depth_transformations.py:15-35).  disp: torch.max propagates a NaN quotient (0 / 0 when acc == 0), fmaxf
// would not.
__device__ __forceinline__ void s5_write_ray_aux(const Stage5Aux& aux, long long r, float dm, float acc) {
  if (aux.depth_map) aux.depth_map[r] = dm;
  if (aux.acc_map) aux.acc_map[r] = acc;
  if (aux.disp_map) {
    const float q = __fdiv_rn(dm, acc);
    aux.disp_map[r] = __fdiv_rn(1.0f, isnan(q) ? q : fmaxf(1e-10f, q));
  }
  if (aux.depth_est && aux.linear_depth) {
    aux.depth_est[r] = dm;
  } else if (aux.depth_est) {
    float d = __fsub_rn(dm, aux.dr_min);
    if (d <= 0.0f) d = 0.001f;
    aux.depth_est[r] = __fdiv_rn(logf(__fadd_rn(d, 1.0f)), aux.log_range);
  }
}

// alpha of nerf_raw2outputs (src/nerf_raymarch_common.py:35-46): dist = (z1 - z0, or 1e10 for the last sample) * |rays_d|,
// 1 - exp(-relu(a) * dist).  torch.relu keeps a NaN, fmaxf would not.
__device__ __forceinline__ float nerf_alpha(float a, float z0, float z1, bool last, float norm) {
  const float dist = __fmul_rn(last ? 1e10f : __fsub_rn(z1, z0), norm);
  const float ra = isnan(a) ? a : fmaxf(a, 0.0f);
  return __fsub_rn(1.0f, expf(__fmul_rn(-ra, dist)));
}

// torch.norm(rays_d[r], dim=-1) in fp32 (the density composite); 0 when there is no ray_d (the adaptive composite).
__device__ __forceinline__ float ray_norm(const float* __restrict__ ray_d, long long r) {
  if (!ray_d) return 0.0f;
  const float x = __ldg(ray_d + 3 * r), y = __ldg(ray_d + 3 * r + 1), z = __ldg(ray_d + 3 * r + 2);
  return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
}

// One thread per ray, samples visited in order: the same sequential cumprod / sum order as torch.  NERF: the density
// composite over K samples at offset r K (launch_stage5).
template <bool NERF>
__global__ void __launch_bounds__(128)
stage5_thread_kernel(const float4* __restrict__ raw1, const float* __restrict__ zp, const float* __restrict__ z,
                     const int32_t* __restrict__ offset, const int32_t* __restrict__ count, long long n_rays, int K,
                     float* __restrict__ rgb, uint32_t* __restrict__ rgba8, const Stage5Aux aux, const float* __restrict__ ray_d) {
  const long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (r >= n_rays) return;
  constexpr bool nerf = NERF;
  const long long off = nerf ? r * K : (long long)offset[r];
  const int n = nerf ? K : count[r];
  const float norm = ray_norm(ray_d, r);
  const bool want_z = nerf || aux.depth_map || aux.disp_map || aux.depth_est || aux.z_vals;
  float T = 1.0f, cr = 0.0f, cg = 0.0f, cb = 0.0f, dm = 0.0f, acc = 0.0f;
  for (int j0 = 0; j0 < n; j0 += 4) {
    // four samples' loads are issued before the (sequential) transmittance chain consumes them
    float4 q4[4];
    float zp4[4], z4[4], zn4[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const bool live = j0 + u < n;
      q4[u] = live ? __ldg(raw1 + off + j0 + u) : make_float4(0.f, 0.f, 0.f, 0.f);
      zp4[u] = (live && !nerf) ? __ldg(zp + off + j0 + u) : 0.0f;
      z4[u] = (live && want_z) ? __ldg(z + off + j0 + u) : 0.0f;
      zn4[u] = (nerf && j0 + u + 1 < n) ? __ldg(z + off + j0 + u + 1) : 0.0f;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = j0 + u;
      if (j >= n) break;
      const float4 q = q4[u];
      const float sr = sigmoidf_acc(q.x), sg = sigmoidf_acc(q.y), sb = sigmoidf_acc(q.z);
      // K == 1: nerf_raw2outputs' dists is [N, 0] (the 1e10 column is expanded to the shape of an empty slice, :36-37), so
      // its alpha and weights are empty and the ray composites to nothing
      const float alpha = nerf ? (n == 1 ? 0.0f : nerf_alpha(q.w, z4[u], zn4[u], j + 1 == n, norm))
                               : __fmul_rn(sigmoidf_acc(q.w), zp4[u]);              // :123-125
      const float w = __fmul_rn(alpha, T);                                          // :128-129
      T = __fmul_rn(T, __fadd_rn(__fsub_rn(1.0f, alpha), 1e-10f));
      cr = __fadd_rn(cr, __fmul_rn(w, sr));                                         // :135
      cg = __fadd_rn(cg, __fmul_rn(w, sg));
      cb = __fadd_rn(cb, __fmul_rn(w, sb));
      acc = __fadd_rn(acc, w);                                                      // :139
      if (want_z) {
        dm = __fadd_rn(dm, __fmul_rn(w, z4[u]));                                    // :137
        if (aux.z_vals) aux.z_vals[r * K + j] = nerf ? z4[u] : s5_z_val(z4[u]);
      }
      if (aux.weights) aux.weights[r * K + j] = w;
      if (aux.alpha) aux.alpha[r * K + j] = alpha;
    }
  }
  for (int j = n; j < K; ++j) {
    if (aux.weights) aux.weights[r * K + j] = 0.0f;
    if (aux.alpha) aux.alpha[r * K + j] = 0.0f;
    if (aux.z_vals) aux.z_vals[r * K + j] = __int_as_float(0x7fc00000);          // features.py:546 (NaN padding)
  }
  if (rgb) {
    rgb[3 * r + 0] = cr;
    rgb[3 * r + 1] = cg;
    rgb[3 * r + 2] = cb;
  }
  if (rgba8) rgba8[r] = to_rgba8(cr, cg, cb);
  s5_write_ray_aux(aux, r, dm, acc);
}

// One warp per ray (dense 128 samples / large K): lanes own consecutive samples, transmittance by a
// warp-wide product scan with a running carry.  NERF: the density composite (launch_stage5).
template <bool NERF>
__global__ void __launch_bounds__(256)
stage5_warp_kernel(const float4* __restrict__ raw1, const float* __restrict__ zp, const float* __restrict__ z,
                   const float* __restrict__ zlut_dense, const int32_t* __restrict__ offset,
                   const int32_t* __restrict__ count, long long n_rays, int K, int dense, float* __restrict__ rgb,
                   uint32_t* __restrict__ rgba8, const Stage5Aux aux, const float* __restrict__ ray_d) {
  const long long r = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= n_rays) return;
  constexpr bool nerf = NERF;
  const long long off = (dense || nerf) ? r * K : (long long)offset[r];
  const int n = (dense || nerf) ? K : count[r];
  const float norm = ray_norm(ray_d, r);
  const bool want_z = nerf || aux.depth_map || aux.disp_map || aux.depth_est || aux.z_vals;
  float carry = 1.0f, cr = 0.0f, cg = 0.0f, cb = 0.0f, dm = 0.0f, acc = 0.0f;
  for (int j0 = 0; j0 < n; j0 += 32) {
    const int j = j0 + lane;
    float alpha = 0.0f, sr = 0.0f, sg = 0.0f, sb = 0.0f, zz = 0.0f;
    if (j < n) {
      const float4 q = __ldg(raw1 + off + j);
      sr = sigmoidf_acc(q.x);
      sg = sigmoidf_acc(q.y);
      sb = sigmoidf_acc(q.z);
      if (nerf) {
        zz = __ldg(z + off + j);
        const float zn = j + 1 < n ? __ldg(z + off + j + 1) : 0.0f;
        alpha = nerf_alpha(q.w, zz, zn, j + 1 == n, norm);
      } else {
        alpha = __fmul_rn(sigmoidf_acc(q.w), __ldg(zp + off + j));
        if (want_z) zz = dense ? __ldg(zlut_dense + j) : __ldg(z + off + j);
      }
    }
    float f = __fadd_rn(__fsub_rn(1.0f, alpha), 1e-10f);
    // inclusive product scan
    float p = f;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float y = __shfl_up_sync(0xffffffffu, p, o);
      if (lane >= o) p = __fmul_rn(p, y);
    }
    float excl = __shfl_up_sync(0xffffffffu, p, 1);
    if (lane == 0) excl = 1.0f;
    const float T = __fmul_rn(carry, excl);
    const float w = __fmul_rn(alpha, T);
    carry = __fmul_rn(carry, __shfl_sync(0xffffffffu, p, 31));
    cr = __fadd_rn(cr, __fmul_rn(w, sr));
    cg = __fadd_rn(cg, __fmul_rn(w, sg));
    cb = __fadd_rn(cb, __fmul_rn(w, sb));
    dm = __fadd_rn(dm, __fmul_rn(w, zz));
    acc = __fadd_rn(acc, w);
    if (j < K) {
      const bool live = j < n;
      if (aux.weights) aux.weights[r * K + j] = live ? w : 0.0f;
      if (aux.alpha) aux.alpha[r * K + j] = live ? alpha : 0.0f;
      if (aux.z_vals) aux.z_vals[r * K + j] = !live ? __int_as_float(0x7fc00000) : (dense || nerf) ? zz : s5_z_val(zz);
    }
  }
  for (int j = ((n + 31) & ~31) + lane; j < K; j += 32) {
    if (aux.weights) aux.weights[r * K + j] = 0.0f;
    if (aux.alpha) aux.alpha[r * K + j] = 0.0f;
    if (aux.z_vals) aux.z_vals[r * K + j] = __int_as_float(0x7fc00000);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    cr += __shfl_xor_sync(0xffffffffu, cr, o);
    cg += __shfl_xor_sync(0xffffffffu, cg, o);
    cb += __shfl_xor_sync(0xffffffffu, cb, o);
    dm += __shfl_xor_sync(0xffffffffu, dm, o);
    acc += __shfl_xor_sync(0xffffffffu, acc, o);
  }
  if (lane == 0) {
    if (rgb) {
      rgb[3 * r + 0] = cr;
      rgb[3 * r + 1] = cg;
      rgb[3 * r + 2] = cb;
    }
    if (rgba8) rgba8[r] = to_rgba8(cr, cg, cb);
    s5_write_ray_aux(aux, r, dm, acc);
  }
}

cudaError_t launch_stage5(const float* d_raw1, const float* d_zp, const float* d_z, const float* d_zlut_dense,
                          const int32_t* d_offset, const int32_t* d_count, long long n_rays, int K, int dense, float* d_rgb,
                          uint8_t* d_rgba8, const Stage5Aux& aux, cudaStream_t s, const float* d_ray_d) {
  if (n_rays <= 0) return cudaSuccess;
  const float4* raw = reinterpret_cast<const float4*>(d_raw1);
  uint32_t* rgba = reinterpret_cast<uint32_t*>(d_rgba8);
  const long long threads = n_rays * 32;
  const unsigned warp_blocks = unsigned((threads + 255) / 256), thread_blocks = unsigned((n_rays + 127) / 128);
  if (d_ray_d && K > 32) {
    stage5_warp_kernel<true><<<warp_blocks, 256, 0, s>>>(raw, nullptr, d_z, nullptr, nullptr, nullptr, n_rays, K, 0, d_rgb, rgba,
                                                         aux, d_ray_d);
  } else if (d_ray_d) {
    stage5_thread_kernel<true><<<thread_blocks, 128, 0, s>>>(raw, nullptr, d_z, nullptr, nullptr, n_rays, K, d_rgb, rgba, aux,
                                                             d_ray_d);
  } else if (dense || K > 32) {
    stage5_warp_kernel<false><<<warp_blocks, 256, 0, s>>>(raw, d_zp, d_z, d_zlut_dense, d_offset, d_count, n_rays, K, dense,
                                                          d_rgb, rgba, aux, nullptr);
  } else {
    stage5_thread_kernel<false><<<thread_blocks, 128, 0, s>>>(raw, d_zp, d_z, d_offset, d_count, n_rays, K, d_rgb, rgba, aux,
                                                              nullptr);
  }
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------- fixed-K sampler
// FromClassifiedDepth.generate (src/nerf_raymarch_common.py:606-660): nerf_sample_pdf(mids, w, K + 2, det=True) (:160-192)
// on mids = linspace(0, 1, 129), samples 1..K kept, then LogTransform.to_world.  One warp per ray, lane l owns cells
// 4l..4l+3 (one 16-byte load):
//   * w = transform(raw0) + 1e-5 and pdf = w / sum(w).  The sum is taken in double and rounded once; torch.sum's fp32
//     order (and the softmax denominator's) is ATen's own, so pdf can differ from the reference's in the last bit;
//   * cdf = [0, cumsum(pdf)]: ATen's CPU cumsum of fp32 accumulates in double, so the warp scans in double and rounds each
//     entry once (the association differs, the double sums almost never round differently); staged in shared memory;
//   * u_j = linspace(0, 1, K + 2)[j] as ATen's CPU kernel forms it: step j below the half, fma(-step, K + 1 - j, 1) above;
//   * lane t takes j = 1 + t, 33 + t, ... <= K: searchsorted(cdf, u, right=True) by binary search over the staged cdf,
//     then the interpolation in the reference's separate fp32 operations, then to_world as the z table does it (pow in
//     double, the rest in fp32).  Stores are coalesced (consecutive j, consecutive lanes).
constexpr int kPdfWarps = 8;
constexpr int kPdfStride = 132;   // one warp's staged cdf (129 entries)

__device__ __forceinline__ float linspace01(int j, int steps) {
  const float step = __fdiv_rn(1.0f, float(steps - 1));
  return j < steps / 2 ? __fmul_rn(step, float(j)) : __fmaf_rn(-step, float(steps - 1 - j), 1.0f);
}

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(32 * kPdfWarps)
pdf_sample_kernel(const float* __restrict__ raw0, long long n_rays, int K, int transform, double wbase, float dr_min,
                  bool aligned16, int32_t* __restrict__ count, int32_t* __restrict__ offset, int32_t* __restrict__ ray,
                  float* __restrict__ zout, long long* __restrict__ total) {
  __shared__ float s_cdf[kPdfWarps][kPdfStride];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long r = blockIdx.x * (long long)kPdfWarps + warp;
  if (r == 0 && lane == 0 && total) *total = n_rays * K;
  if (r >= n_rays) return;
  const float4 v4 = ld_row_quad(raw0 + r * 128, lane, aligned16);
  float w[4] = {v4.x, v4.y, v4.z, v4.w};
  if (transform == kPdfSoftmax) {   // softmax(dim=-1): exp(x - max) * (1 / sum)
    float m = fmaxf(fmaxf(w[0], w[1]), fmaxf(w[2], w[3]));
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    double se = 0.0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      w[k] = expf(__fsub_rn(w[k], m));
      se += w[k];
    }
    const float inv = __fdiv_rn(1.0f, float(warp_sum_f64(se)));   // ATen's vectorised softmax scales by the reciprocal
#pragma unroll
    for (int k = 0; k < 4; ++k) w[k] = __fmul_rn(w[k], inv);
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) w[k] = sigmoidf_acc(w[k]);
  }
  double sw = 0.0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    w[k] = __fadd_rn(w[k], 1e-5f);                                               // :162
    sw += w[k];
  }
  const float wsum = float(warp_sum_f64(sw));                                      // :163
  double a[4], run = 0.0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    run += double(__fdiv_rn(w[k], wsum));
    a[k] = run;
  }
  double inc = run;                                                                // :164 (inclusive warp scan)
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const double y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  double excl = __shfl_up_sync(0xffffffffu, inc, 1);
  if (lane == 0) excl = 0.0;
  float* cdf = s_cdf[warp];
  if (lane == 0) cdf[0] = 0.0f;                                                    // :165
#pragma unroll
  for (int k = 0; k < 4; ++k) cdf[4 * lane + k + 1] = float(excl + a[k]);
  __syncwarp();
  const int steps = K + 2;
  for (int j = 1 + lane; j <= K; j += 32) {
    const float u = linspace01(j, steps);                                          // :169
    int lo = 0, hi = 129;                                                          // :177 first cdf entry > u (right=True)
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (cdf[mid] > u) hi = mid;
      else lo = mid + 1;
    }
    const int below = max(0, lo - 1), above = min(128, lo);                       // :178-179
    const float c0 = cdf[below], c1 = cdf[above];
    const float b0 = linspace01(below, 129), b1 = linspace01(above, 129);
    float denom = __fsub_rn(c1, c0);                                               // :188-189
    if (denom < 1e-5f) denom = 1.0f;
    const float t = __fdiv_rn(__fsub_rn(u, c0), denom);                            // :190-191
    const float zs = __fadd_rn(b0, __fmul_rn(t, __fsub_rn(b1, b0)));
    const float zw = __fadd_rn(__fsub_rn(float(pow(wbase, double(zs))), 1.0f), dr_min);   // depth_transformations.py:44-46
    const long long o = r * K + (j - 1);
    zout[o] = zw;
    if (ray) ray[o] = int32_t(r);
  }
  if (lane == 0) {
    if (count) count[r] = K;
    if (offset) offset[r] = int32_t(r * K);
  }
}

cudaError_t launch_pdf_sample(const float* d_raw0, long long n_rays, int K, int transform, double wbase, float dr_min,
                              int32_t* d_count, int32_t* d_offset, int32_t* d_ray, float* d_z, long long* d_total, cudaStream_t s) {
  const long long n = n_rays > 0 ? n_rays : 1;   // an empty call still writes *d_total = 0
  const bool aligned16 = (reinterpret_cast<uintptr_t>(d_raw0) & 15u) == 0;
  pdf_sample_kernel<<<unsigned((n + kPdfWarps - 1) / kPdfWarps), 32 * kPdfWarps, 0, s>>>(
      d_raw0, n_rays, K, transform, wbase, dr_min, aligned16, d_count, d_offset, d_ray, d_z, d_total);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------- metrics
__global__ void __launch_bounds__(256)
sqdiff_partial_kernel(const float* __restrict__ a, const float* __restrict__ b, long long n, int clamp01,
                      double* __restrict__ partials) {
  __shared__ double s_w[8];
  double acc = 0.0;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += 256ll * gridDim.x) {
    float x = __ldg(a + i);
    if (clamp01) x = fminf(fmaxf(x, 0.0f), 1.0f);
    const double d = double(x) - double(__ldg(b + i));
    acc += d * d;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += s_w[w];
    partials[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(32) sqdiff_final_kernel(const double* __restrict__ partials, int n, double* __restrict__ out) {
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += 32) acc += partials[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (threadIdx.x == 0) *out = acc;
}

cudaError_t launch_image_sqdiff(const float* d_a, const float* d_b, long long n_values, int clamp01, double* d_partials,
                                double* d_sum, cudaStream_t s) {
  sqdiff_partial_kernel<<<kMetricBlocks, 256, 0, s>>>(d_a, d_b, n_values, clamp01, d_partials);
  sqdiff_final_kernel<<<1, 32, 0, s>>>(d_partials, kMetricBlocks, d_sum);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------- viewer surface
__global__ void rgba_to_surface_kernel(const uchar4* __restrict__ px, int W, int row0, int rows, cudaSurfaceObject_t surf) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x < W && y < rows) surf2Dwrite(px[size_t(y) * W + x], surf, x * int(sizeof(uchar4)), row0 + y);
}

cudaError_t launch_rgba_to_surface(const uint8_t* d_rgba8, int W, int row0, int rows, unsigned long long surface, cudaStream_t s) {
  if (rows <= 0 || W <= 0) return cudaSuccess;
  const dim3 block(32, 8), grid(unsigned((W + 31) / 32), unsigned((rows + 7) / 8));
  rgba_to_surface_kernel<<<grid, block, 0, s>>>(reinterpret_cast<const uchar4*>(d_rgba8), W, row0, rows, cudaSurfaceObject_t(surface));
  return cudaGetLastError();
}

}  // namespace adn
