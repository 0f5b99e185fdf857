// Positional-encoding helpers shared by the feature kernels (stages.cu) and the shading MLP's fused input encoder
// (mlp.cu).
#pragma once
#include <cuda_runtime.h>

#include "stages.cuh"

namespace adn {

// enc_L(v) = [v, sin(2^0 v), cos(2^0 v), ..., sin(2^(L-1) v), cos(2^(L-1) v)], each term a 3-vector
// (src/util/feature_encoding.py:60-73).  Writes 3 + 6L floats.
// The frequencies are powers of two, so sin / cos of 2^f v follow from those of 2^(f-1) v by the double-angle
// identities (3 FMA-class ops instead of a ~40-instruction sincosf).  The error at least doubles per step, so an
// accurate sincosf re-anchors the recurrence every kAnchor octaves.  Against float64 sin / cos the fourth step after an
// anchor (bands 4 and 9) is off by up to ~4e-6 when the anchors are correctly rounded, and by up to 1.7e-5 when they
// sit anywhere within sincosf's documented 2 ulp (per-band bounds: oracle/stage_emulation.py, recurrence_band_bounds)
// -- still far inside the 2^f argument-rounding amplification that the reference's own fp32 evaluation carries
// (SURVEY 8d: 5e-4 at 2^9).
constexpr int kAnchor = 5;
template <int L>
__device__ __forceinline__ void posenc3(const float (&v)[3], float* out) {
  out[0] = v[0];
  out[1] = v[1];
  out[2] = v[2];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    float s = 0.f, c = 1.f;
#pragma unroll
    for (int f = 0; f < L; ++f) {
      if (f % kAnchor == 0) {
        sincosf(__fmul_rn(v[a], float(1 << f)), &s, &c);
      } else {
        const float s2 = 2.0f * s * c;
        const float c2 = fmaf(-2.0f * s, s, 1.0f);
        s = s2;
        c = c2;
      }
      out[3 + 6 * f + a] = s;
      out[3 + 6 * f + 3 + a] = c;
    }
  }
}

// posenc3 with a run-time band count L >= 0 (posEnc none = 0 bands: v alone): the same operations, so the same bits as
// posenc3<L>.  Feature j of the 3 + 6L goes to emit(j, value), in no particular order, so no array of them is held.
template <typename Emit>
__device__ __forceinline__ void posenc3_rt(const float (&v)[3], int L, Emit emit) {
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    emit(a, v[a]);
    float s = 0.f, c = 1.f;
    for (int f = 0; f < L; ++f) {
      if (f % kAnchor == 0) {
        sincosf(__fmul_rn(v[a], float(1 << f)), &s, &c);
      } else {
        const float s2 = 2.0f * s * c;
        const float c2 = fmaf(-2.0f * s, s, 1.0f);
        s = s2;
        c = c2;
      }
      emit(3 + 6 * f + a, s);
      emit(3 + 6 * f + 3 + a, c);
    }
  }
}

// ndc_rays(H, W, focal, near = 1) (src/nerf_raymarch_common.py:71-88) of one ray in the reference's operation order:
// origin o and direction d -> the NDC origin oo and the un-normalised NDC direction dd.
__device__ __forceinline__ void ndc_ray(const SceneDev& sc, const float (&o)[3], const float (&d)[3], float (&oo)[3],
                                        float (&dd)[3]) {
  const float t = __fdiv_rn(-__fadd_rn(1.0f, o[2]), d[2]);
  float on[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) on[a] = __fadd_rn(o[a], __fmul_rn(t, d[a]));
  const float q0 = __fdiv_rn(on[0], on[2]), q1 = __fdiv_rn(on[1], on[2]);
  oo[0] = __fdiv_rn(__fmul_rn(sc.ndc_cw, on[0]), on[2]);
  oo[1] = __fdiv_rn(__fmul_rn(sc.ndc_ch, on[1]), on[2]);
  oo[2] = __fadd_rn(1.0f, __fdiv_rn(2.0f, on[2]));
  dd[0] = __fmul_rn(sc.ndc_cw, __fsub_rn(__fdiv_rn(d[0], d[2]), q0));
  dd[1] = __fmul_rn(sc.ndc_ch, __fsub_rn(__fdiv_rn(d[1], d[2]), q1));
  dd[2] = __fdiv_rn(-2.0f, on[2]);
}

// torch.norm(v, dim=-1) of a 3-vector in fp32: sqrt((x x + y y) + z z).
__device__ __forceinline__ float norm3(const float (&v)[3]) {
  return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(v[0], v[0]), __fmul_rn(v[1], v[1])), __fmul_rn(v[2], v[2])));
}

// The shading net's inputs of one sample at world depth zw on ray r (RayMarchFromPoses.batch, src/features.py:458-479), in
// the reference's operation order: the position into pos and the direction to encode into dir.  Stage 3 and the fused
// encoder both call this, so their features are the same bits.
__device__ __forceinline__ void sample_inputs(const SceneDev& sc, bool ndc, const float* __restrict__ ray_o,
                                              const float* __restrict__ ray_d, long long r, float zw, float (&pos)[3],
                                              float (&dir)[3]) {
  float o[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    o[a] = __ldg(ray_o + 3 * r + a);
    dir[a] = __ldg(ray_d + 3 * r + a);   // un-normalised nds, as SpherePosDir hands it on
  }
  if (ndc) {
    // ndc_rays, then pos = o' + d' z with the un-normalised NDC direction, no position normalisation, view encoding of
    // d' / |d'|
    float oo[3], dd[3];
    ndc_ray(sc, o, dir, oo, dd);
#pragma unroll
    for (int a = 0; a < 3; ++a) pos[a] = __fadd_rn(oo[a], __fmul_rn(dd[a], zw));                 // :458
    const float dn = norm3(dd);
#pragma unroll
    for (int a = 0; a < 3; ++a) dir[a] = __fdiv_rn(dd[a], dn);                                    // :431
  } else {
#pragma unroll
    for (int a = 0; a < 3; ++a) pos[a] = __fsub_rn(__fadd_rn(o[a], __fmul_rn(dir[a], zw)), sc.c[a]);   // :458, loc = pos - c
    // normalization_inverse_sqrt_dist_centered (src/nerf_raymarch_common.py:226-230)
    const float nrm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(pos[0], pos[0]), __fmul_rn(pos[1], pos[1])), __fmul_rn(pos[2], pos[2])));
    const float den = __fmul_rn(sc.sqrt_max_depth, __fsqrt_rn(nrm));
#pragma unroll
    for (int a = 0; a < 3; ++a) pos[a] = __fdiv_rn(pos[a], den);
  }
}

}  // namespace adn
