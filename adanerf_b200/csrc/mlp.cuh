// Fused multi-layer perceptron on the Hopper tensor cores (wgmma), sm_90a.
//
// One persistent CTA per SM walks 128-row tiles of the batch through ALL layers of the network:
//   * weights stream layer by layer from L2 into a shared-memory ring with 1-D bulk async copies
//     (TMA engine), pre-packed on the host as K-major SWIZZLE_128B tiles (the split net: [128 x 32] SWIZZLE_64B hi + lo
//     tiles) in consumption order,
//   * activations never leave the SM: two consumer warpgroups each own 64 rows of the tile, accumulate
//     a layer in registers (wgmma m64n128k16, one 64-register accumulator per 128-column N half), add
//     bias / ReLU, round to bf16 and keep the result as the next layer's A operand: in registers for plain
//     bf16 nets (the accumulator fragment is the register-A fragment, 64 registers at W = 256), in
//     swizzled shared memory as a hi+lo split for the split-precision net; a warpgroup only ever touches its own
//     rows, so the layers of one warpgroup need no synchronisation with the other beyond the shared weight ring,
//   * warp roles: warpgroups 0, 1 = consumers, warpgroup 2 = producers: warp 8 issues the weight copies; with NSPLIT == 1
//     warps 9-11 fill the next tile's inputs into the second of two input slots while the consumers run the current one
//     (the fused encoder computes them; otherwise one bulk copy of the packed tile).  The producers hand most of their
//     registers to the consumers (setmaxnreg), whose accumulators take 128 per thread.
//
// NSPLIT = 2 is the split-precision mode of the sampling network: x = hi + lo (both bf16) for
// activations and weights and three MMAs per K step (hi*hi + lo*hi + hi*lo), fp32 accumulate --
// fp32-class accuracy, which the bit-exact threshold decisions downstream need (SURVEY.md 8d).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "stages.cuh"
#include "tiles.cuh"

namespace adn {

constexpr int kMaxLayers = 12;
constexpr int kMlpThreads = 384;  // three warpgroups: two consumers, one weight producer
// fp32 side parameters (biases, alpha / rgb heads), copied to shared memory per CTA.  The largest supported net sets it: a
// 10 x 256 shading net has 10 x 256 pts biases, 256 + 128 feature / view biases, 256 + 4 alpha and 384 + 4 rgb floats.
constexpr int kSideFloats = 3592;

enum : uint8_t {
  LF_RELU = 1,
  LF_ALPHA_DOT = 2,      // accumulate alpha = <post-activation row, alpha_w> on CUDA cores (fp32)
  LF_OUT_ACT = 4,        // write bf16 activations for the next layer
  LF_FINAL_RAW = 8,      // write fp32 rows to global (sampling net output / test programs)
  LF_FINAL_RGB = 16      // rgb_linear on CUDA cores + write float4 (rgb, alpha)
};

// Where a layer's A operand comes from, in K order: in_first input blocks (input blocks 0, 1) in shared memory, then
// n_hid hidden blocks, then input block in_nblk0 (V) when in_last; n_kb = in_first + n_hid + in_last.  With NSPLIT == 1
// (the shading net, and the plain bf16 sampling net) the hidden blocks are in the registers the previous layer's epilogue wrote; the
// split-precision sampling net (NSPLIT == 2) keeps them as activation blocks 0 .. n_hid - 1, which each epilogue
// overwrites in place, so there K block kb reads activation block kb.
struct MlpLayer {
  uint32_t w_off;     // byte offset of this layer's packed weight stages (N half outermost, then K block; layer_stages)
  uint32_t bias_off;  // float offset of the fp32 bias vector in MlpProgram::side
  uint8_t n_kb;       // number of 64-wide K blocks
  uint8_t in_first, n_hid, in_last;   // 0-2, 0 or W / 64, 0 / 1
  uint8_t n_half;     // N / 128  (1 or 2)
  uint8_t flags;
  // 16-wide K steps issued per K block (4 = the whole 64-wide block; fewer when the tail columns of the block are zero
  // padding, e.g. 90 input features -> blocks of 4 and 2 steps; 30 features -> 2 and 0).
  uint8_t k_cnt[6];
};

// 16-wide K steps per weight ring stage: a [128 x 64] block for plain bf16; for the split net a [128 x 32] hi block and
// its lo block (SWIZZLE_64B), so that its ring holds more, smaller stages next to its activation blocks.
__host__ __device__ constexpr int stage_k_steps(int nsplit) { return nsplit == 2 ? 2 : 4; }

// Ring stages of layer L, one per N half and K block's group of stage_k_steps K steps that holds a K step (a K block
// with k_cnt 0 has none; with nsplit == 1 every K block has a stage).  pack_layer packs this many, the kernel's weight
// producer streams and its consumers take this many.
__host__ __device__ inline int layer_stages(const MlpLayer& L, int nsplit) {
  if (nsplit == 1) return int(L.n_kb) * int(L.n_half);
  int s = 0;
  for (int kb = 0; kb < L.n_kb; ++kb) s += (L.k_cnt[kb] + stage_k_steps(nsplit) - 1) / stage_k_steps(nsplit);
  return s * int(L.n_half);
}

struct MlpProgram {
  int32_t n_layers;
  TileFormat in;              // the packed input tiles (in.n_terms == NSPLIT)
  int32_t in_nblk0;           // input blocks (per term) the first layer reads; the shading net's V is the block after them
  uint32_t alpha_w_off, alpha_b_off, rgb_w_off, rgb_b_off;  // float offsets in `side`
  int32_t out_cols;           // row stride of the FINAL_RAW output
  MlpLayer layers[kMaxLayers];
  float side[kSideFloats];
};

// Fused input encoder of the shading MLP (stage 3 inside the kernel): producer warps 9-11 compute the positional encoding
// of the packed samples (RayMarchFromPoses.batch, src/features.py:458-479) straight into the next tile's input slot, so
// the [M, 90] feature tensor and its packed tiles never exist in HBM.  ray_idx == nullptr: dense mode
// (ray = sample / K, z = zlut_dense[sample % K]).
struct EncodeParams {
  const float* ray_o = nullptr;       // [N,3]
  const float* ray_d = nullptr;       // [N,3] (un-normalised, as SpherePosDir hands it on)
  const int32_t* ray_idx = nullptr;   // [M] packed sample -> ray
  const float* z = nullptr;           // [M] world depth of the packed samples
  const float* zlut_dense = nullptr;  // [K]
  int K = 1;
  SceneDev sc{};                      // non-NDC scenes only
};

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device attribute: set it once per (kernel, device).
// `done` is the caller's per-kernel bit mask (one static per launcher).
cudaError_t set_max_dyn_smem_once(const void* func, int bytes, unsigned long long* done);

// Launchers (defined in mlp.cu).  rows_dev may be null (then rows_host is used).  prog.in.n_terms == 2: split precision.
// enc != nullptr: shading net with the fused input encoder (in_tiles unused).
cudaError_t launch_mlp(const MlpProgram& prog, const uint8_t* wblob, const uint8_t* in_tiles, float* out,
                       const long long* rows_dev, long long rows_host, int* err_flag, int num_sms, cudaStream_t stream,
                       const EncodeParams* enc = nullptr);
// fp32 feature rows [rows, n_feat] -> packed tiles of format `fmt`.
cudaError_t launch_pack_rows(const float* x, long long rows, const long long* rows_dev, int n_feat, const TileFormat& fmt,
                             uint8_t* tiles, int num_sms, cudaStream_t stream);

}  // namespace adn
