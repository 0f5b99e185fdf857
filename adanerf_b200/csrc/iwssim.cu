// IW-SSIM of two images (see iwssim.cuh).  The reference image is the metric's original: its bands weight the scales and
// supply the parent band.  Ten launches, each over every scale that needs it:
//   iwssim_gray_kernel:   the metric's image, as doubles: evaluate.py's rgb2gray (fp32, round half to even) or the gray plane;
//   iwssim_down_kernel:   one pyramid reduction (corrDn, binom5, reflect about the edge sample, step 2), fp64; four launches;
//   iwssim_band_kernel:   band = level - upConv(next level) (zero-insert, reflect, binom5) for every level, rounded to fp32
//                         once; the low-pass is rounded as it is;
//   iwssim_cov_kernel:    per block, fp64 partial sums of the 55 distinct entries of Y^T Y (3 x 3 neighbours, plus the
//                         parent at scales 1-3) over the interior pixels of scales 1-4;
//   iwssim_eig_kernel:    one block per scale: the partial sums in a fixed order, cyclic Jacobi (round-robin, five disjoint
//                         rotations at a time) in fp64, the eigenvalue adjustment, the rebuilt matrix and its Gauss-Jordan
//                         inverse (NaN at a zero pivot);
//   iwssim_main_kernel:   per 32 x 8 tile of a scale's cs map: the separable 11-tap Gaussian statistics of the five moment
//                         planes, cs (and l at scale 5), then at scales 1-4 the 3 x 3 gain and error, y^T C^-1 y and the
//                         information weight; per block fp64 partial sums of cs * iw and iw (cs * l and 1 at scale 5);
//   iwssim_final_kernel:  the partial sums of each scale in a fixed order, the wmcs and the score, in double.
// Everything after the fp32 bands is fp64; every sum runs in an order fixed by the image size alone.
#include <cmath>
#include <cstdint>

#include "iwssim.cuh"

namespace adn {
namespace {

constexpr int kThreads = 256;
constexpr int kCovThreads = 128, kCovPix = 8;     // covariance: pixels per thread
constexpr int kTileX = 32, kTileY = 8;            // cs pixels per main block
constexpr int kHalo = 10;                         // the 11 x 11 window
constexpr int kInX = kTileX + kHalo, kInY = kTileY + kHalo;
constexpr int kNsym = kIwMaxN * (kIwMaxN + 1) / 2;   // 55 distinct entries of Y^T Y
constexpr int kEigThreads = 128;
constexpr int kMaxSweeps = 16;
constexpr double kTol = 1e-15;
constexpr double kSigmaNsq = 0.4;
constexpr double kC1 = (0.01 * 255) * (0.01 * 255), kC2 = (0.03 * 255) * (0.03 * 255);

__constant__ double c_binom5[5];

__device__ __forceinline__ int reflect(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * (n - 1) - i : i); }

// ---- input conversion -----------------------------------------------------------------------------------------------------
// grid (ceil(n / kThreads), 2): y = 0 the reference (original), 1 the image (distorted).  In both layouts the metric's image
// is the buffer's pixels in order, rows x cols.
__global__ void __launch_bounds__(kThreads)
iwssim_gray_kernel(const float* __restrict__ img, const float* __restrict__ ref, int n, int layout, double* __restrict__ g0,
                   size_t lvl_total) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const float* src = blockIdx.y == 0 ? ref : img;
  float v;
  if (layout == kIwEvaluateRgb) {
    // 0.2989 r + 0.5870 g + 0.1140 b, each product and sum rounded to fp32 as torch does, then np.round (half to even)
    const float* p = src + size_t(i) * 3;
    v = rintf(__fadd_rn(__fadd_rn(__fmul_rn(0.2989f, __ldg(p)), __fmul_rn(0.5870f, __ldg(p + 1))), __fmul_rn(0.1140f, __ldg(p + 2))));
  } else {
    v = __ldg(src + i);
  }
  g0[blockIdx.y * lvl_total + i] = double(v);
}

// ---- pyramid --------------------------------------------------------------------------------------------------------------
// grid (ceil(rd * cd / kThreads), 2).  corrDn along rows, then along columns: 5 x 5 taps with per-axis reflection.
__global__ void __launch_bounds__(kThreads)
iwssim_down_kernel(double* __restrict__ levels, size_t lvl_total, size_t src_off, int rs, int cs, size_t dst_off, int rd, int cd) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= rd * cd) return;
  const int y = i / cd, x = i - y * cd;
  const double* src = levels + blockIdx.y * lvl_total + src_off;
  double acc = 0.0;
  for (int b = 0; b < 5; ++b) {
    const int xs = reflect(2 * x + b - 2, cs);
    double t = 0.0;
    for (int a = 0; a < 5; ++a) t += c_binom5[a] * src[size_t(reflect(2 * y + a - 2, rs)) * cs + xs];
    acc += c_binom5[b] * t;
  }
  levels[blockIdx.y * lvl_total + dst_off + i] = acc;
}

// grid (band_blk[5], 2).  Band l = level l - upConv(level l + 1): the coarse samples sit at even positions of level l's
// grid, zeros between; the zero-inserted signal is reflected about its edge sample and correlated with binom5.
__global__ void __launch_bounds__(kThreads)
iwssim_band_kernel(const double* __restrict__ levels, const IwPlan p, float* __restrict__ bands) {
  int l = 0;
  while (l < kIwNsc - 1 && int(blockIdx.x) >= p.band_blk[l + 1]) ++l;
  const int i = (blockIdx.x - p.band_blk[l]) * kThreads + threadIdx.x;
  const int R = p.rows[l], Cc = p.cols[l];
  if (i >= R * Cc) return;
  const double* lv = levels + blockIdx.y * p.lvl_total;
  double v = lv[p.lvl_off[l] + i];
  if (l < kIwNsc - 1) {
    const int y = i / Cc, x = i - y * Cc;
    const double* nx = lv + p.lvl_off[l + 1];
    const int cn = p.cols[l + 1];
    double acc = 0.0;
    for (int b = 0; b < 5; ++b) {
      const int xs = reflect(x + b - 2, Cc);
      double t = 0.0;
      if ((xs & 1) == 0)
        for (int a = 0; a < 5; ++a) {
          const int ys = reflect(y + a - 2, R);
          if ((ys & 1) == 0) t += c_binom5[a] * nx[size_t(ys >> 1) * cn + (xs >> 1)];
        }
      acc += c_binom5[b] * t;
    }
    v -= acc;
  }
  bands[blockIdx.y * p.lvl_total + p.lvl_off[l] + i] = float(v);
}

// ---- parent band ----------------------------------------------------------------------------------------------------------
// The bilinear resize (align_corners=False) of an M-sample axis to 4M - 3 samples: the two source samples and weights of
// output sample o.
__device__ __forceinline__ void bilinear_src(int o, int M, int& i0, int& i1, double& l0, double& l1) {
  const double scale = double(M) / double(4 * M - 3);
  double src = scale * (o + 0.5) - 0.5;
  src = src < 0.0 ? 0.0 : src;
  i0 = int(src);
  i1 = i0 + (i0 < M - 1 ? 1 : 0);
  l1 = src - i0;
  l0 = 1.0 - l1;
}

// Sample t2-index 2e of the extended axis (4M - 1 samples: the resized axis with one linearly extrapolated sample at each
// end) as up to two resized samples and weights.
__device__ __forceinline__ int enlarge_taps(int e, int M, int* idx, double* w) {
  if (e == 0) {
    idx[0] = 0; w[0] = 2.0; idx[1] = 1; w[1] = -1.0;
    return 2;
  }
  if (2 * e == 4 * M - 2) {
    idx[0] = 4 * M - 4; w[0] = 2.0; idx[1] = 4 * M - 5; w[1] = -1.0;
    return 2;
  }
  idx[0] = 2 * e - 1; w[0] = 1.0;
  return 1;
}

// The parent band (M x N, fp32) enlarged to its child's grid, at child pixel (i, j): rows extrapolated first, then columns.
__device__ double parent_at(const float* __restrict__ b, int M, int N, int i, int j) {
  int ri[2], ci[2];
  double rw[2], cw[2];
  const int nr = enlarge_taps(i, M, ri, rw), nc = enlarge_taps(j, N, ci, cw);
  double acc = 0.0;
  for (int c = 0; c < nc; ++c) {
    int w0, w1;
    double lw0, lw1;
    bilinear_src(ci[c], N, w0, w1, lw0, lw1);
    double col = 0.0;
    for (int r = 0; r < nr; ++r) {
      int h0, h1;
      double lh0, lh1;
      bilinear_src(ri[r], M, h0, h1, lh0, lh1);
      const double t = lh0 * (lw0 * double(__ldg(b + size_t(h0) * N + w0)) + lw1 * double(__ldg(b + size_t(h0) * N + w1))) +
                       lh1 * (lw0 * double(__ldg(b + size_t(h1) * N + w0)) + lw1 * double(__ldg(b + size_t(h1) * N + w1)));
      col += rw[r] * t;
    }
    acc += cw[c] * col;
  }
  return acc;
}

// ---- covariance -----------------------------------------------------------------------------------------------------------
template <int N>
__device__ __forceinline__ void block_sum_store(double (&acc)[N], double* s_red, double* __restrict__ out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int kWarps = kCovThreads / 32;
#pragma unroll
  for (int e = 0; e < N; ++e) {
    double v = acc[e];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) s_red[warp * N + e] = v;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < N; e += kCovThreads) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) t += s_red[w * N + e];
    out[e] = t;
  }
}

// grid (cov_blk[4]): blocks of scales 1-4, each over kCovThreads * kCovPix interior pixels of the original's band.
__global__ void __launch_bounds__(kCovThreads)
iwssim_cov_kernel(const float* __restrict__ bands, const IwPlan p, double* __restrict__ partials) {
  __shared__ double s_red[kCovThreads / 32 * kNsym];
  int s = 0;
  while (s < kIwNsc - 2 && int(blockIdx.x) >= p.cov_blk[s + 1]) ++s;
  const int R = p.rows[s], Cc = p.cols[s];
  const int ni = Cc - 2, n_int = (R - 2) * ni;
  const bool prnt = s < kIwNsc - 2;
  const float* b = bands + p.lvl_off[s];
  const float* bp = bands + p.lvl_off[s + 1];
  double acc[kNsym];
#pragma unroll
  for (int e = 0; e < kNsym; ++e) acc[e] = 0.0;
  const int base = (blockIdx.x - p.cov_blk[s]) * kCovThreads * kCovPix + threadIdx.x;
  for (int k = 0; k < kCovPix; ++k) {
    const int q = base + k * kCovThreads;
    if (q >= n_int) break;
    const int i = q / ni + 1, j = q - (q / ni) * ni + 1;
    double y[kIwMaxN];
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) y[dy * 3 + dx] = double(__ldg(b + size_t(i - 1 + dy) * Cc + (j - 1 + dx)));
    y[9] = prnt ? parent_at(bp, p.rows[s + 1], p.cols[s + 1], i, j) : 0.0;
    int e = 0;
#pragma unroll
    for (int r = 0; r < kIwMaxN; ++r)
#pragma unroll
      for (int c = r; c < kIwMaxN; ++c, ++e) acc[e] = fma(y[r], y[c], acc[e]);
  }
  block_sum_store(acc, s_red, partials + size_t(blockIdx.x) * kNsym);
}

// ---- eigen step -----------------------------------------------------------------------------------------------------------
// One block per scale 1-4.  Writes, at eig + s * (kIwMaxN * kIwMaxN + kIwMaxN): the inverse of the rebuilt covariance
// (10 x 10, zero outside n x n; all NaN when it cannot be inverted), then the n raw eigenvalues.
__global__ void __launch_bounds__(kEigThreads)
iwssim_eig_kernel(const double* __restrict__ partials, const IwPlan p, double* __restrict__ eig) {
  constexpr int n10 = kIwMaxN;
  __shared__ double A[n10][n10], B[n10][n10], V[n10][n10], VB[n10][n10];
  __shared__ double M[n10][2 * n10];
  __shared__ double rc[n10 / 2], rs[n10 / 2], f[n10], lam_adj[n10];
  __shared__ int rp[n10 / 2], rq[n10 / 2], pair_of[n10], piv_row;
  __shared__ bool rotated, fail;
  const int s = blockIdx.x, tid = threadIdx.x;
  const int n = s < kIwNsc - 2 ? 10 : 9;
  const double nexp = double(p.rows[s] - 2) * double(p.cols[s] - 2);
  // the partial sums of this scale's blocks, warp w over entries w, w + 4, ..., each lane over a strided run of blocks
  {
    const int lane = tid & 31, warp = tid >> 5;
    const int b0 = p.cov_blk[s], nb = p.cov_blk[s + 1] - b0;
    for (int e = warp; e < kNsym; e += kEigThreads / 32) {
      double v = 0.0;
      for (int k = lane; k < nb; k += 32) v += partials[size_t(b0 + k) * kNsym + e];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) {
        int r = 0, c = e, row_len = n10;
        while (c >= row_len) { c -= row_len; ++r; --row_len; }
        c += r;
        A[r][c] = A[c][r] = v / nexp;
      }
    }
  }
  if (tid < n10 * n10) V[tid / n10][tid % n10] = (tid / n10 == tid % n10) ? 1.0 : 0.0;
  if (tid == 0) { rotated = true; fail = false; }
  __syncthreads();
  // cyclic Jacobi, round-robin: in round r, index 9 meets r and (r + k) % 9 meets (r - k) % 9, k = 1..4.  At scale 4 the
  // tenth row and column are zero, so every rotation that touches index 9 is the identity.  A pair is rotated while
  // |a_pq| > 1e-17 sqrt(|a_pp a_qq|); the sweeps end after one that rotates nothing (4-6 sweeps here).
  for (int sweep = 0; sweep < kMaxSweeps; ++sweep) {
    __syncthreads();
    if (!rotated) break;
    __syncthreads();
    if (tid == 0) rotated = false;
    __syncthreads();
    for (int round = 0; round < n10 - 1; ++round) {
      if (tid < n10 / 2) {
        int a = tid == 0 ? n10 - 1 : (round + tid) % (n10 - 1);
        int b = tid == 0 ? round : (round - tid + (n10 - 1)) % (n10 - 1);
        const int pp = a < b ? a : b, qq = a < b ? b : a;
        const double apq = A[pp][qq];
        double c = 1.0, sn = 0.0;
        if (fabs(apq) > 1e-17 * sqrt(fabs(A[pp][pp] * A[qq][qq]))) {
          rotated = true;
          const double theta = (A[qq][qq] - A[pp][pp]) / (2.0 * apq);
          const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
          c = 1.0 / sqrt(t * t + 1.0);
          sn = t * c;
        }
        rp[tid] = pp; rq[tid] = qq; rc[tid] = c; rs[tid] = sn;
        pair_of[pp] = tid; pair_of[qq] = tid;
      }
      __syncthreads();
      if (tid < n10 * n10) {   // B = A P, VB = V P
        const int i = tid / n10, j = tid % n10, k = pair_of[j];
        const int pp = rp[k], qq = rq[k];
        const double c = rc[k], sn = rs[k];
        B[i][j] = j == pp ? c * A[i][pp] - sn * A[i][qq] : sn * A[i][pp] + c * A[i][qq];
        VB[i][j] = j == pp ? c * V[i][pp] - sn * V[i][qq] : sn * V[i][pp] + c * V[i][qq];
      }
      __syncthreads();
      if (tid < n10 * n10) {   // A = P^T B, its rotated pairs set to exactly 0
        const int i = tid / n10, j = tid % n10, k = pair_of[i];
        const int pp = rp[k], qq = rq[k];
        const double c = rc[k], sn = rs[k];
        A[i][j] = pair_of[j] == k && i != j ? 0.0 : (i == pp ? c * B[pp][j] - sn * B[qq][j] : sn * B[pp][j] + c * B[qq][j]);
        V[i][j] = VB[i][j];
      }
      __syncthreads();
    }
  }
  __syncthreads();
  // eigenvalue adjustment: negative ones to 0, positive ones rescaled to keep the sum
  if (tid == 0) {
    double sum = 0.0, pos = 0.0;
    for (int j = 0; j < n; ++j) {
      sum += A[j][j];
      pos += A[j][j] > 0.0 ? A[j][j] : 0.0;
    }
    const double k = sum / (pos + (pos == 0.0 ? 1.0 : 0.0));
    for (int j = 0; j < n; ++j) lam_adj[j] = (A[j][j] > 0.0 ? A[j][j] : 0.0) * k;
  }
  __syncthreads();
  // rebuilt matrix V diag(lam_adj) V^T, augmented with the identity
  for (int t = tid; t < n * 2 * n; t += kEigThreads) {
    const int i = t / (2 * n), j = t % (2 * n);
    double v = 0.0;
    if (j < n)
      for (int k = 0; k < n; ++k) v += V[i][k] * lam_adj[k] * V[j][k];
    else
      v = (j - n == i) ? 1.0 : 0.0;
    M[i][j] = v;
  }
  __syncthreads();
  // Gauss-Jordan with partial pivoting
  for (int k = 0; k < n; ++k) {
    if (tid == 0) {
      int best = k;
      double bv = -1.0;
      for (int i = k; i < n; ++i)
        if (fabs(M[i][k]) > bv) { bv = fabs(M[i][k]); best = i; }
      piv_row = best;
      if (!(fabs(M[best][k]) > 0.0)) fail = true;
    }
    __syncthreads();
    if (fail) break;
    if (tid < 2 * n && piv_row != k) {
      const double t = M[k][tid];
      M[k][tid] = M[piv_row][tid];
      M[piv_row][tid] = t;
    }
    __syncthreads();
    const double piv = M[k][k];
    if (tid < n) f[tid] = M[tid][k];
    __syncthreads();
    if (tid < 2 * n) M[k][tid] = M[k][tid] / piv;
    __syncthreads();
    for (int t = tid; t < n * 2 * n; t += kEigThreads) {
      const int i = t / (2 * n), j = t % (2 * n);
      if (i != k) M[i][j] -= f[i] * M[k][j];
    }
    __syncthreads();
  }
  double* out = eig + size_t(s) * (n10 * n10 + n10);
  if (tid < n10 * n10) {
    const int i = tid / n10, j = tid % n10;
    out[tid] = fail ? __longlong_as_double(0x7ff8000000000000LL) : (i < n && j < n ? M[i][n + j] : 0.0);
  }
  if (tid < n) out[n10 * n10 + tid] = A[tid][tid];
}

// ---- quality maps and information weights ---------------------------------------------------------------------------------
__device__ __forceinline__ double block_sum(double v, double* s_red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int tid = threadIdx.y * kTileX + threadIdx.x;
  if ((tid & 31) == 0) s_red[tid >> 5] = v;
  __syncthreads();
  double t = 0.0;
#pragma unroll
  for (int w = 0; w < kTileX * kTileY / 32; ++w) t += s_red[w];
  return t;
}

// grid (main_blk[5]), block kTileX x kTileY: one tile of one scale's cs map; partials[2 * block + {0, 1}].
__global__ void __launch_bounds__(kTileX * kTileY)
iwssim_main_kernel(const float* __restrict__ bands, const double* __restrict__ eig, const IwPlan p, double* __restrict__ partials) {
  __shared__ double s_x[kInY][kInX], s_y[kInY][kInX];
  __shared__ double s_h[5][kInY][kTileX];
  __shared__ double s_inv[kIwMaxN * kIwMaxN + kIwMaxN];
  __shared__ double s_red[2][kTileX * kTileY / 32];
  int s = 0;
  while (s < kIwNsc - 1 && int(blockIdx.x) >= p.main_blk[s + 1]) ++s;
  const int R = p.rows[s], Cc = p.cols[s];
  const int mh = R - kHalo, mw = Cc - kHalo;              // the cs map
  const int t = blockIdx.x - p.main_blk[s];
  const int ty0 = (t / p.main_tx[s]) * kTileY, tx0 = (t % p.main_tx[s]) * kTileX;
  const int tid = threadIdx.y * kTileX + threadIdx.x;
  const float* bo = bands + p.lvl_off[s];
  const float* bd = bands + p.lvl_total + p.lvl_off[s];
  for (int i = tid; i < kInY * kInX; i += kTileX * kTileY) {
    const int r = ty0 + i / kInX, c = tx0 + i % kInX;
    const bool in = r < R && c < Cc;
    s_x[i / kInX][i % kInX] = in ? double(__ldg(bo + size_t(r) * Cc + c)) : 0.0;
    s_y[i / kInX][i % kInX] = in ? double(__ldg(bd + size_t(r) * Cc + c)) : 0.0;
  }
  const bool iw_scale = s < kIwNsc - 1;
  if (iw_scale)
    for (int i = tid; i < kIwMaxN * kIwMaxN + kIwMaxN; i += kTileX * kTileY) s_inv[i] = eig[size_t(s) * (kIwMaxN * kIwMaxN + kIwMaxN) + i];
  __syncthreads();
  for (int i = tid; i < kInY * kTileX; i += kTileX * kTileY) {
    const int r = i / kTileX, c = i % kTileX;
    double m1 = 0.0, m2 = 0.0, xx = 0.0, yy = 0.0, xy = 0.0;
#pragma unroll
    for (int k = 0; k <= kHalo; ++k) {
      const double w = p.gauss[k], x = s_x[r][c + k], y = s_y[r][c + k];
      m1 += w * x;
      m2 += w * y;
      xx += w * (x * x);
      yy += w * (y * y);
      xy += w * (x * y);
    }
    s_h[0][r][c] = m1; s_h[1][r][c] = m2; s_h[2][r][c] = xx; s_h[3][r][c] = yy; s_h[4][r][c] = xy;
  }
  __syncthreads();
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int a = ty0 + ty, b = tx0 + tx;
  double num = 0.0, den = 0.0;
  if (a < mh && b < mw) {
    double mu1 = 0.0, mu2 = 0.0, exx = 0.0, eyy = 0.0, exy = 0.0;
#pragma unroll
    for (int k = 0; k <= kHalo; ++k) {
      const double w = p.gauss[k];
      mu1 += w * s_h[0][ty + k][tx];
      mu2 += w * s_h[1][ty + k][tx];
      exx += w * s_h[2][ty + k][tx];
      eyy += w * s_h[3][ty + k][tx];
      exy += w * s_h[4][ty + k][tx];
    }
    const double s12 = exy - mu1 * mu2;
    double s1 = exx - mu1 * mu1, s2 = eyy - mu2 * mu2;
    s1 = s1 < 0.0 ? 0.0 : s1;       // torch.max(0, x): NaN stays NaN
    s2 = s2 < 0.0 ? 0.0 : s2;
    const double cs = (2.0 * s12 + kC2) / (s1 + s2 + kC2);
    if (!iw_scale) {
      num = cs * ((2.0 * mu1 * mu2 + kC1) / (mu1 * mu1 + mu2 * mu2 + kC1));
      den = 1.0;
    } else {
      // band pixel (a + 5, b + 5): its 3 x 3 statistics (never padded here), neighbourhood vector and parent
      const int cy = ty + 5, cx = tx + 5;
      constexpr double kNinth = 1.0 / 9.0;
      double mx = 0.0, my = 0.0, sxx = 0.0, syy = 0.0, sxy = 0.0, yv[kIwMaxN];
#pragma unroll
      for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx) {
          const double x = s_x[cy + dy][cx + dx], y = s_y[cy + dy][cx + dx];
          mx += x * kNinth;
          my += y * kNinth;
          sxx += (x * x) * kNinth;
          syy += (y * y) * kNinth;
          sxy += (x * y) * kNinth;
          yv[(dy + 1) * 3 + dx + 1] = x;
        }
      const int n = s < kIwNsc - 2 ? 10 : 9;
      yv[9] = n == 10 ? parent_at(bands + p.lvl_off[s + 1], p.rows[s + 1], p.cols[s + 1], a + 5, b + 5) : 0.0;
      const double cov = sxy - mx * my;
      double ssx = sxx - mx * mx, ssy = syy - my * my;
      ssx = ssx < 0.0 ? 0.0 : ssx;
      ssy = ssy < 0.0 ? 0.0 : ssy;
      double g = cov / (ssx + kTol);
      double vv = ssy - g * cov;
      if (ssx < kTol) { g = 0.0; vv = ssy; }
      if (ssy < kTol) { g = 0.0; vv = 0.0; }
      double ss = 0.0;
#pragma unroll
      for (int i = 0; i < kIwMaxN; ++i) {
        double r = 0.0;
#pragma unroll
        for (int j = 0; j < kIwMaxN; ++j) r += yv[j] * s_inv[j * kIwMaxN + i];
        ss += r * yv[i];
      }
      ss /= double(n);
      const double gain = (vv + (1.0 + g * g) * kSigmaNsq) * ss;
      double iw = 0.0;
      for (int j = 0; j < n; ++j) iw += log2(1.0 + (gain * s_inv[kIwMaxN * kIwMaxN + j] + kSigmaNsq * vv) / (kSigmaNsq * kSigmaNsq));
      iw = iw < kTol ? 0.0 : iw;
      num = cs * iw;
      den = iw;
    }
  }
  num = block_sum(num, s_red[0]);
  den = block_sum(den, s_red[1]);
  if (tid == 0) {
    partials[2 * size_t(blockIdx.x)] = num;
    partials[2 * size_t(blockIdx.x) + 1] = den;
  }
}

// ---- the score ------------------------------------------------------------------------------------------------------------
// One block, warp s over scale s.  out: score, wmcs 1..5.
__global__ void __launch_bounds__(kIwNsc * 32)
iwssim_final_kernel(const double* __restrict__ partials, const IwPlan p, double* __restrict__ out) {
  __shared__ double s_w[kIwNsc];
  const int lane = threadIdx.x & 31, s = threadIdx.x >> 5;
  double num = 0.0, den = 0.0;
  for (int k = p.main_blk[s] + lane; k < p.main_blk[s + 1]; k += 32) {
    num += partials[2 * size_t(k)];
    den += partials[2 * size_t(k) + 1];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    num += __shfl_xor_sync(0xffffffffu, num, o);
    den += __shfl_xor_sync(0xffffffffu, den, o);
  }
  if (lane == 0) s_w[s] = num / den;
  __syncthreads();
  if (threadIdx.x == 0) {
    // the reference holds the scale weights as an fp32 tensor: its weights are the fp32-rounded values
    const double w[kIwNsc] = {double(0.0448f), double(0.2856f), double(0.3001f), double(0.2363f), double(0.1333f)};
    double score = 1.0;
    for (int k = 0; k < kIwNsc; ++k) {
      score *= pow(fabs(s_w[k]), w[k]);
      out[1 + k] = s_w[k];
    }
    out[0] = score;
  }
}

int blocks(size_t n, int per) { return int((n + per - 1) / per); }
size_t align256(size_t b) { return (b + 255) / 256 * 256; }

}  // namespace

IwPlan iwssim_plan(int rows, int cols) {
  IwPlan p{};
  size_t off = 0;
  p.band_blk[0] = 0;
  for (int l = 0; l < kIwNsc; ++l) {
    p.rows[l] = l == 0 ? rows : (p.rows[l - 1] + 1) / 2;
    p.cols[l] = l == 0 ? cols : (p.cols[l - 1] + 1) / 2;
    p.lvl_off[l] = off;
    const size_t n = size_t(p.rows[l]) * p.cols[l];
    off += n;
    p.band_blk[l + 1] = p.band_blk[l] + blocks(n, kThreads);
  }
  p.lvl_total = off;
  p.cov_blk[0] = 0;
  for (int s = 0; s < kIwNsc - 1; ++s)
    p.cov_blk[s + 1] = p.cov_blk[s] + blocks(size_t(p.rows[s] - 2) * (p.cols[s] - 2), kCovThreads * kCovPix);
  p.main_blk[0] = 0;
  for (int s = 0; s < kIwNsc; ++s) {
    p.main_tx[s] = (p.cols[s] - kHalo + kTileX - 1) / kTileX;
    p.main_blk[s + 1] = p.main_blk[s] + p.main_tx[s] * ((p.rows[s] - kHalo + kTileY - 1) / kTileY);
  }
  double g[11], sum = 0.0;
  for (int k = 0; k <= kHalo; ++k) sum += (g[k] = std::exp(-double((k - 5) * (k - 5)) / (2.0 * 1.5 * 1.5)));
  for (int k = 0; k <= kHalo; ++k) p.gauss[k] = g[k] / sum;
  p.off_g = 0;
  p.off_b = align256(p.off_g + 2 * p.lvl_total * sizeof(double));
  p.off_cov = align256(p.off_b + 2 * p.lvl_total * sizeof(float));
  p.off_eig = align256(p.off_cov + size_t(p.cov_blk[kIwNsc - 1]) * kNsym * sizeof(double));
  p.off_part = align256(p.off_eig + size_t(kIwNsc - 1) * (kIwMaxN * kIwMaxN + kIwMaxN) * sizeof(double));
  p.off_out = align256(p.off_part + 2 * size_t(p.main_blk[kIwNsc]) * sizeof(double));
  p.bytes = align256(p.off_out + (1 + kIwNsc) * sizeof(double));
  return p;
}

cudaError_t launch_iwssim(const float* d_image, const float* d_reference, int layout, const IwPlan& p, void* d_scratch,
                          cudaStream_t st) {
  static const double binom5[5] = {1.0 / 16 * 1.4142135623730951, 4.0 / 16 * 1.4142135623730951, 6.0 / 16 * 1.4142135623730951,
                                   4.0 / 16 * 1.4142135623730951, 1.0 / 16 * 1.4142135623730951};
  cudaError_t e = cudaMemcpyToSymbolAsync(c_binom5, binom5, sizeof(binom5), 0, cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) return e;
  char* base = static_cast<char*>(d_scratch);
  double* levels = reinterpret_cast<double*>(base + p.off_g);
  float* bands = reinterpret_cast<float*>(base + p.off_b);
  double* cov = reinterpret_cast<double*>(base + p.off_cov);
  double* eig = reinterpret_cast<double*>(base + p.off_eig);
  double* part = reinterpret_cast<double*>(base + p.off_part);
  double* out = reinterpret_cast<double*>(base + p.off_out);
  const int n = p.rows[0] * p.cols[0];
  iwssim_gray_kernel<<<dim3(blocks(n, kThreads), 2), kThreads, 0, st>>>(d_image, d_reference, n, layout, levels, p.lvl_total);
  for (int l = 0; l < kIwNsc - 1; ++l)
    iwssim_down_kernel<<<dim3(blocks(size_t(p.rows[l + 1]) * p.cols[l + 1], kThreads), 2), kThreads, 0, st>>>(
        levels, p.lvl_total, p.lvl_off[l], p.rows[l], p.cols[l], p.lvl_off[l + 1], p.rows[l + 1], p.cols[l + 1]);
  iwssim_band_kernel<<<dim3(p.band_blk[kIwNsc], 2), kThreads, 0, st>>>(levels, p, bands);
  iwssim_cov_kernel<<<p.cov_blk[kIwNsc - 1], kCovThreads, 0, st>>>(bands, p, cov);
  iwssim_eig_kernel<<<kIwNsc - 1, kEigThreads, 0, st>>>(cov, p, eig);
  iwssim_main_kernel<<<p.main_blk[kIwNsc], dim3(kTileX, kTileY), 0, st>>>(bands, eig, p, part);
  iwssim_final_kernel<<<1, kIwNsc * 32, 0, st>>>(part, p, out);
  return cudaGetLastError();
}

}  // namespace adn
