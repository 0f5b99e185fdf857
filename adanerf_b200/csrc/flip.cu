// FLIP of two sRGB images (see flip.cuh).  Every 2-D filter of the metric is separable, so the work is two passes:
//   flip_rows_kernel:  sRGB -> YCxCz once per pixel into shared memory (one row segment plus its halo), then the seven
//                      horizontal 1-D filters of each image into planes [image][filter][H*W];
//   flip_cols_kernel:  the vertical filters from those planes, then everything per pixel -- linear RGB clamp, L*a*b*, Hunt,
//                      HyAB^0.7, the error remap, the feature term, the final power -- and one partial sum per block;
//   flip_sum_kernel:   the partial sums in a fixed order, in double.
// Replicate padding is a clamped pixel index in both passes (the two clamps compose to the 2-D one exactly).  Both images go
// through the same code and meet only in symmetric expressions, so swapping the arguments gives the same bits.  NaN
// propagates as in the reference's torch code: its clamps pass NaN through, so no clamp or max here uses fminf / fmaxf.
#include <cmath>
#include <cstdint>

#include "flip.cuh"

namespace adn {
namespace {

constexpr int kRowThreads = 128;            // pixels per row segment of flip_rows_kernel
constexpr int kTileX = 32, kTileY = 8;      // pixels per block of flip_cols_kernel
constexpr int kPlanes = 7;                  // horizontal-pass planes per image, in FlipFilter order
constexpr int kSumThreads = 256;

// torch.clamp(x, lo, hi): NaN stays NaN
__device__ __forceinline__ float clamp_nan(float x, float lo, float hi) { return x < lo ? lo : (x > hi ? hi : x); }
// torch.maximum: NaN if either is NaN
__device__ __forceinline__ float max_nan(float a, float b) { return (a > b || a != a) ? a : b; }

__device__ __forceinline__ void mat3(const float* m, float x, float y, float z, float& u, float& v, float& w) {
  u = m[0] * x + m[1] * y + m[2] * z;
  v = m[3] * x + m[4] * y + m[5] * z;
  w = m[6] * x + m[7] * y + m[8] * z;
}

__device__ __forceinline__ float srgb_to_linear(float c) {
  c = clamp_nan(c, 0.0f, 1.0f);
  return c > 0.04045f ? powf((c + 0.055f) / 1.055f, 2.4f) : c / 12.92f;
}

__device__ __forceinline__ float lab_f(float t) { return t > 0.00885f ? cbrtf(t) : t / (3.0f * (6.0f / 29.0f) * (6.0f / 29.0f)) + 4.0f / 29.0f; }

__device__ __forceinline__ void load_weights(float* s_w, const FlipConsts& c, int tid, int nthreads) {
  for (int i = tid; i < kFlipNumFilters * kFlipTaps; i += nthreads) s_w[i] = c.w[i];
}

// grid: (row segments * H, 2 images), block kRowThreads.  s_px holds (Y, Cx, Cz, (Y + 16) / 116) of the segment and its halo.
__global__ void __launch_bounds__(kRowThreads)
flip_rows_kernel(const float* __restrict__ img_a, const float* __restrict__ img_b, int W, int H, int n_seg, const FlipConsts c,
                 float* __restrict__ planes) {
  __shared__ float s_w[kFlipNumFilters * kFlipTaps];
  __shared__ float4 s_px[kRowThreads + 2 * kFlipMaxRadius];
  const int tid = threadIdx.x;
  const int row = blockIdx.x / n_seg;
  const int x0 = (blockIdx.x - row * n_seg) * kRowThreads;
  const float* img = blockIdx.y == 0 ? img_a : img_b;
  const int R = c.r > c.rf ? c.r : c.rf;
  load_weights(s_w, c, tid, kRowThreads);
  for (int i = tid; i < kRowThreads + 2 * R; i += kRowThreads) {
    int xs = x0 - R + i;
    xs = xs < 0 ? 0 : (xs >= W ? W - 1 : xs);
    const float* p = img + (size_t(row) * W + xs) * 3;
    float xn, yn, zn;
    mat3(c.rgb2xyz, srgb_to_linear(__ldg(p)), srgb_to_linear(__ldg(p + 1)), srgb_to_linear(__ldg(p + 2)), xn, yn, zn);
    const float Y = 116.0f * yn - 16.0f;
    s_px[i] = make_float4(Y, 500.0f * (xn - yn), 200.0f * (yn - zn), (Y + 16.0f) / 116.0f);
  }
  __syncthreads();
  const int x = x0 + tid;
  if (x >= W) return;
  float a = 0.0f, rg = 0.0f, by1 = 0.0f, by2 = 0.0f;
  const float4* px = s_px + tid + R - c.r;
  for (int k = 0; k <= 2 * c.r; ++k) {
    const float4 v = px[k];
    a = fmaf(s_w[kFlipA * kFlipTaps + k], v.x, a);
    rg = fmaf(s_w[kFlipRG * kFlipTaps + k], v.y, rg);
    by1 = fmaf(s_w[kFlipBY1 * kFlipTaps + k], v.z, by1);
    by2 = fmaf(s_w[kFlipBY2 * kFlipTaps + k], v.z, by2);
  }
  float fg = 0.0f, edge = 0.0f, point = 0.0f;
  px = s_px + tid + R - c.rf;
  for (int k = 0; k <= 2 * c.rf; ++k) {
    const float y = px[k].w;
    fg = fmaf(s_w[kFlipFG * kFlipTaps + k], y, fg);
    edge = fmaf(s_w[kFlipEdge * kFlipTaps + k], y, edge);
    point = fmaf(s_w[kFlipPoint * kFlipTaps + k], y, point);
  }
  const size_t n = size_t(W) * H;
  float* out = planes + size_t(blockIdx.y) * kPlanes * n + size_t(row) * W + x;
  out[kFlipA * n] = a;
  out[kFlipRG * n] = rg;
  out[kFlipBY1 * n] = by1;
  out[kFlipBY2 * n] = by2;
  out[kFlipFG * n] = fg;
  out[kFlipEdge * n] = edge;
  out[kFlipPoint * n] = point;
}

// One image's filtered values at one pixel: Hunt-adjusted L*a*b* and the edge / point feature magnitudes.
struct FlipPixel {
  float L, a, b, edge, point;
};

__device__ __forceinline__ FlipPixel flip_pixel(const float* __restrict__ p, const float* s_w, const FlipConsts& c, int W, int H,
                                                int x, int y) {
  const size_t n = size_t(W) * H;
  float A = 0.0f, RG = 0.0f, by1 = 0.0f, by2 = 0.0f;
  for (int k = 0; k <= 2 * c.r; ++k) {
    int ys = y - c.r + k;
    ys = ys < 0 ? 0 : (ys >= H ? H - 1 : ys);
    const float* q = p + size_t(ys) * W + x;
    A = fmaf(s_w[kFlipA * kFlipTaps + k], __ldg(q + kFlipA * n), A);
    RG = fmaf(s_w[kFlipRG * kFlipTaps + k], __ldg(q + kFlipRG * n), RG);
    by1 = fmaf(s_w[kFlipBY1 * kFlipTaps + k], __ldg(q + kFlipBY1 * n), by1);
    by2 = fmaf(s_w[kFlipBY2 * kFlipTaps + k], __ldg(q + kFlipBY2 * n), by2);
  }
  float ex = 0.0f, px = 0.0f, ey = 0.0f, py = 0.0f;
  for (int k = 0; k <= 2 * c.rf; ++k) {
    int ys = y - c.rf + k;
    ys = ys < 0 ? 0 : (ys >= H ? H - 1 : ys);
    const float* q = p + size_t(ys) * W + x;
    const float g = s_w[kFlipFG * kFlipTaps + k];
    ex = fmaf(g, __ldg(q + kFlipEdge * n), ex);          // edge in x: EDGE(x) FG(y)
    px = fmaf(g, __ldg(q + kFlipPoint * n), px);
    const float fg = __ldg(q + kFlipFG * n);             // edge in y: FG(x) EDGE(y)
    ey = fmaf(s_w[kFlipEdge * kFlipTaps + k], fg, ey);
    py = fmaf(s_w[kFlipPoint * kFlipTaps + k], fg, py);
  }
  const float BY = c.by_w1 * by1 + c.by_w2 * by2;
  // YCxCz -> XYZ / white -> linear RGB, clamped to the RGB box
  const float yy = (A + 16.0f) / 116.0f;
  float r, g, b;
  mat3(c.xyz2rgb, yy + RG / 500.0f, yy, yy - BY / 200.0f, r, g, b);
  r = clamp_nan(r, 0.0f, 1.0f);
  g = clamp_nan(g, 0.0f, 1.0f);
  b = clamp_nan(b, 0.0f, 1.0f);
  float xn, yn, zn;
  mat3(c.rgb2xyz, r, g, b, xn, yn, zn);
  const float fx = lab_f(xn), fy = lab_f(yn), fz = lab_f(zn);
  // Explicitly rounded: the caller subtracts the two images' values, and a product left to the compiler could be fused
  // into that subtraction for one image and not the other (identical inputs must give exactly 0, swapped ones the same bits).
  FlipPixel o;
  o.L = __fmaf_rn(116.0f, fy, -16.0f);
  o.a = __fmul_rn(0.01f * o.L, 500.0f * (fx - fy));   // Hunt adjustment
  o.b = __fmul_rn(0.01f * o.L, 200.0f * (fy - fz));
  o.edge = sqrtf(ex * ex + ey * ey);
  o.point = sqrtf(px * px + py * py);
  return o;
}

// grid: ceil(W / kTileX) * ceil(H / kTileY) blocks of kTileX x kTileY.
__global__ void __launch_bounds__(kTileX * kTileY)
flip_cols_kernel(const float* __restrict__ planes, int W, int H, int n_tx, const FlipConsts c, float* __restrict__ map,
                 double* __restrict__ partials) {
  __shared__ float s_w[kFlipNumFilters * kFlipTaps];
  __shared__ double s_sum[kTileX * kTileY / 32];
  const int tid = threadIdx.y * kTileX + threadIdx.x;
  load_weights(s_w, c, tid, kTileX * kTileY);
  __syncthreads();
  const int ty = blockIdx.x / n_tx;
  const int x = (blockIdx.x - ty * n_tx) * kTileX + threadIdx.x;
  const int y = ty * kTileY + threadIdx.y;
  double v = 0.0;
  if (x < W && y < H) {
    const size_t n = size_t(W) * H;
    const FlipPixel p = flip_pixel(planes, s_w, c, W, H, x, y);
    const FlipPixel q = flip_pixel(planes + kPlanes * n, s_w, c, W, H, x, y);
    // colour: HyAB distance, ^0.7, remapped so that [0, pc cmax) -> [0, pt) and [pc cmax, cmax] -> [pt, 1]
    const float da = p.a - q.a, db = p.b - q.b;
    const float hyab = fabsf(p.L - q.L) + sqrtf(da * da + db * db);
    const float pw = powf(hyab, 0.7f);
    const float pccmax = 0.4f * c.cmax;
    const float dec = pw < pccmax ? (0.95f / pccmax) * pw : 0.95f + ((pw - pccmax) / (c.cmax - pccmax)) * (1.0f - 0.95f);
    // features
    const float df = max_nan(fabsf(p.edge - q.edge), fabsf(p.point - q.point));
    const float def = clamp_nan(sqrtf(0.70710678118654752f * df), 0.0f, 1.0f);
    const float f = powf(dec, 1.0f - def);
    if (map) map[size_t(y) * W + x] = f;
    v = f;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((tid & 31) == 0) s_sum[tid >> 5] = v;
  __syncthreads();
  if (tid == 0) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < kTileX * kTileY / 32; ++w) t += s_sum[w];
    partials[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(kSumThreads) flip_sum_kernel(const double* __restrict__ partials, int n, double* __restrict__ out) {
  __shared__ double s_sum[kSumThreads / 32];
  double v = 0.0;
  for (int i = threadIdx.x; i < n; i += kSumThreads) v += partials[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < kSumThreads / 32; ++w) t += s_sum[w];
    *out = t;
  }
}

size_t n_tiles(int W, int H) { return size_t((W + kTileX - 1) / kTileX) * size_t((H + kTileY - 1) / kTileY); }
// the sum, the partial sums (n_tiles doubles), then the planes, 256-byte aligned
size_t planes_offset(int W, int H) { return ((n_tiles(W, H) + 1) * sizeof(double) + 255) / 256 * 256; }

}  // namespace

void flip_consts(double ppd, FlipConsts* out) {
  FlipConsts& c = *out;
  const double pi = 3.14159265358979323846;
  // linear RGB -> XYZ (D65); the white is its row sums
  const double M[9] = {10135552.0 / 24577794, 8788810.0 / 24577794, 4435075.0 / 24577794,
                       2613072.0 / 12288897,  8788810.0 / 12288897, 887015.0 / 12288897,
                       1425312.0 / 73733382,  8788810.0 / 73733382, 70074185.0 / 73733382};
  double white[3], inv[9];
  for (int i = 0; i < 3; ++i) white[i] = M[3 * i] + M[3 * i + 1] + M[3 * i + 2];
  const double det = M[0] * (M[4] * M[8] - M[5] * M[7]) - M[1] * (M[3] * M[8] - M[5] * M[6]) + M[2] * (M[3] * M[7] - M[4] * M[6]);
  inv[0] = (M[4] * M[8] - M[5] * M[7]) / det;
  inv[1] = (M[2] * M[7] - M[1] * M[8]) / det;
  inv[2] = (M[1] * M[5] - M[2] * M[4]) / det;
  inv[3] = (M[5] * M[6] - M[3] * M[8]) / det;
  inv[4] = (M[0] * M[8] - M[2] * M[6]) / det;
  inv[5] = (M[2] * M[3] - M[0] * M[5]) / det;
  inv[6] = (M[3] * M[7] - M[4] * M[6]) / det;
  inv[7] = (M[1] * M[6] - M[0] * M[7]) / det;
  inv[8] = (M[0] * M[4] - M[1] * M[3]) / det;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      c.rgb2xyz[3 * i + j] = float(M[3 * i + j] / white[i]);
      c.xyz2rgb[3 * i + j] = float(inv[3 * i + j] * white[j]);
    }
  // cmax: Hunt-adjusted L*a*b* of pure green and pure blue, HyAB distance ^ 0.7
  auto lab_hunt = [&](int ch, double* lab) {
    double f[3];
    for (int i = 0; i < 3; ++i) {
      const double t = M[3 * i + ch] / white[i];
      f[i] = t > 0.00885 ? std::cbrt(t) : t / (3 * (6.0 / 29) * (6.0 / 29)) + 4.0 / 29;
    }
    lab[0] = 116 * f[1] - 16;
    lab[1] = 0.01 * lab[0] * 500 * (f[0] - f[1]);
    lab[2] = 0.01 * lab[0] * 200 * (f[1] - f[2]);
  };
  double g[3], b[3];
  lab_hunt(1, g);
  lab_hunt(2, b);
  c.cmax = float(std::pow(std::fabs(g[0] - b[0]) + std::hypot(g[1] - b[1], g[2] - b[2]), 0.7));

  for (float& w : c.w) w = 0.0f;
  // CSF filters: a1 sqrt(pi / b1) exp(-pi^2 z / b1) + a2 sqrt(pi / b2) exp(-pi^2 z / b2), z = (x^2 + y^2) / ppd^2
  c.r = int(std::ceil(3 * std::sqrt(0.04 / (2 * pi * pi)) * ppd));
  const double dx = 1.0 / ppd;
  auto gauss = [&](int f, double bb) {   // writes the normalised 1-D term, returns its unnormalised sum
    double e[kFlipTaps], s = 0;
    for (int k = 0; k <= 2 * c.r; ++k) s += (e[k] = std::exp(-pi * pi * (k - c.r) * dx * (k - c.r) * dx / bb));
    for (int k = 0; k <= 2 * c.r; ++k) c.w[f * kFlipTaps + k] = float(e[k] / s);
    return s;
  };
  gauss(kFlipA, 0.0047);
  gauss(kFlipRG, 0.0053);
  const double s1 = gauss(kFlipBY1, 0.04), s2 = gauss(kFlipBY2, 0.025);
  const double t1 = 34.1 * std::sqrt(pi / 0.04) * s1 * s1, t2 = 13.5 * std::sqrt(pi / 0.025) * s2 * s2;
  c.by_w1 = float(t1 / (t1 + t2));
  c.by_w2 = float(t2 / (t1 + t2));
  // feature filters: sd = 0.5 * 0.082 * ppd pixels
  const double sd = 0.5 * 0.082 * ppd;
  c.rf = int(std::ceil(3 * sd));
  double gs = 0, ge[kFlipTaps], gp[kFlipTaps];
  double pos_e = 0, neg_e = 0, pos_p = 0, neg_p = 0;
  for (int k = 0; k <= 2 * c.rf; ++k) {
    const double t = k - c.rf, e = std::exp(-t * t / (2 * sd * sd));
    gs += e;
    ge[k] = -t * e;
    gp[k] = (t * t / (sd * sd) - 1) * e;
    (ge[k] > 0 ? pos_e : neg_e) += ge[k];
    (gp[k] > 0 ? pos_p : neg_p) += gp[k];
  }
  for (int k = 0; k <= 2 * c.rf; ++k) {
    const double t = k - c.rf;
    c.w[kFlipFG * kFlipTaps + k] = float(std::exp(-t * t / (2 * sd * sd)) / gs);
    c.w[kFlipEdge * kFlipTaps + k] = float(ge[k] < 0 ? ge[k] / -neg_e : ge[k] / pos_e);
    c.w[kFlipPoint * kFlipTaps + k] = float(gp[k] < 0 ? gp[k] / -neg_p : gp[k] / pos_p);
  }
}

size_t flip_scratch_bytes(int W, int H) { return planes_offset(W, H) + size_t(2) * kPlanes * size_t(W) * H * sizeof(float); }

cudaError_t launch_flip(const float* d_a, const float* d_b, int W, int H, const FlipConsts& c, void* d_scratch, float* d_map,
                        cudaStream_t s) {
  double* sum = static_cast<double*>(d_scratch);
  double* partials = sum + 1;
  float* planes = reinterpret_cast<float*>(static_cast<char*>(d_scratch) + planes_offset(W, H));
  const int n_seg = (W + kRowThreads - 1) / kRowThreads;
  flip_rows_kernel<<<dim3(unsigned(n_seg) * unsigned(H), 2), kRowThreads, 0, s>>>(d_a, d_b, W, H, n_seg, c, planes);
  const int n_tx = (W + kTileX - 1) / kTileX;
  const int n_blk = int(n_tiles(W, H));
  flip_cols_kernel<<<n_blk, dim3(kTileX, kTileY), 0, s>>>(planes, W, H, n_tx, c, d_map, partials);
  flip_sum_kernel<<<1, kSumThreads, 0, s>>>(partials, n_blk, sum);
  return cudaGetLastError();
}

}  // namespace adn
