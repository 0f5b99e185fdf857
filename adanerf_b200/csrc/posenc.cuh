// Positional-encoding helpers shared by the feature kernels (stages.cu) and the shading MLP's fused input encoder
// (mlp.cu).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <cstdint>

namespace adn {

__device__ __forceinline__ uint32_t bf16x2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// enc_L(v) = [v, sin(2^0 v), cos(2^0 v), ..., sin(2^(L-1) v), cos(2^(L-1) v)], each term a 3-vector
// (src/util/feature_encoding.py:60-73).  Writes 3 + 6L floats.
// The frequencies are powers of two, so sin / cos of 2^f v follow from those of 2^(f-1) v by the double-angle
// identities (3 FMA-class ops instead of a ~40-instruction sincosf).  The rounding error doubles per step, so
// an accurate sincosf re-anchors the recurrence every kAnchor octaves: the result stays within 2^(kAnchor-1)
// ulp-class (<= ~2e-6 abs) of the directly evaluated value -- far inside the 2^f argument-rounding amplification
// that the reference's own fp32 evaluation carries (SURVEY 8d: 5e-4 at 2^9).
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

}  // namespace adn
