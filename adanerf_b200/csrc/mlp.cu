// Warpgroup-MMA fused MLP kernel (see mlp.cuh for the design).
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "mlp.cuh"
#include "posenc.cuh"
#include "ptx.cuh"
#include "tiles.cuh"

namespace adn {

// A set of layer flags known at compile time: the epilogue's tests of it fold away.
template <uint8_t V>
struct ConstFlags {
  __device__ constexpr operator uint8_t() const { return V; }
};

constexpr int kInSlots = 2;   // mlp_kernel<1>: input slots, so the producer fills one tile ahead of the consumers

template <int NSPLIT>
struct MlpCfg {
  // NSPLIT == 2: activation blocks per term, the split net's input / hidden blocks.  NSPLIT == 1: the most input blocks a
  // layer reads first (the sampling net's two, the shading net's one or two P blocks); the hidden activations stay in
  // registers and the inputs sit in kInSlots slots of one packed tile each.
  static constexpr int kNB = (NSPLIT == 2) ? 4 : 2;
  // One ring stage, 16 KB either way: a [128 x 64] weight block (SWIZZLE_128B), or for the split net a [128 x 32] hi
  // block and its lo block (SWIZZLE_64B, stage_k_steps(2) = 2 K steps).
  static constexpr int kStageBytes = kBlkBytes;
  // As many ring stages as fit next to the inputs and the side parameters (227 KB per block): two slots of a three-block
  // tile (P > 64 columns) take two stages' room; the split net's 128 KB of activations leave room for five.
  __host__ __device__ static constexpr int stages(int n_blk) { return NSPLIT == 2 ? 5 : (n_blk > 2 ? 6 : 8); }
  __host__ __device__ static constexpr size_t in_bytes(int n_blk) {
    return NSPLIT == 2 ? size_t(NSPLIT) * kNB * kBlkBytes : size_t(kInSlots) * n_blk * kBlkBytes;
  }
  // full / empty per ring stage, and per input slot (NSPLIT == 1) or an input-landed barrier per consumer warpgroup
  __host__ __device__ static constexpr int n_bars(int n_blk) { return 2 * stages(n_blk) + (NSPLIT == 1 ? 2 * kInSlots : 2); }
  __host__ __device__ static constexpr size_t smem_bytes(int n_blk) {
    return in_bytes(n_blk) + size_t(stages(n_blk)) * kStageBytes + size_t(kSideFloats) * 4 + size_t(n_bars(n_blk)) * 8 +
           1024 /*alignment slack*/;
  }
  // the largest over the tile formats the kernel runs (the split net's is fixed)
  static constexpr size_t kMaxSmemBytes = smem_bytes(2) > smem_bytes(3) ? smem_bytes(2) : smem_bytes(3);
};
static_assert(MlpCfg<1>::kMaxSmemBytes <= 232448 && MlpCfg<2>::kMaxSmemBytes <= 232448, "shared memory per block (sm_90)");

// Row `row` of the fused encoder's input blocks (n_freq_pos <= 20, n_freq_dir <= 10 bands): P (3 + 6 n_freq_pos
// features, in one block or two) into the blocks from `blk` on, or V into block `blk`, each feature written as stage 3
// writes it (posenc3_rt, the bits of posenc3<L>; put_feature, the bits of pack_chunk8), then zeros up to the block's end.
__device__ __forceinline__ void encode_row(const EncodeParams& enc, long long i, long long rows, uint8_t* blk, int row,
                                           bool view) {
  const TileFormat act{1, 2, {0, 64, 0}, {64, 64, 0}};   // consecutive blocks: block b at blk + b * kBlkBytes
  const int n_p = 3 + 6 * enc.sc.n_freq_pos;
  zero_row(act, blk, uint32_t(row), 0, view ? 1 : shading_p_blocks(n_p));
  if (i < rows) {
    long long ray;
    float zw;
    if (enc.ray_idx) {
      ray = enc.ray_idx[i];
      zw = enc.z[i];
    } else {
      ray = i / enc.K;
      zw = enc.zlut_dense[i - ray * enc.K];
    }
    float pos[3], dir[3];
    sample_inputs(enc.sc, false, enc.ray_o, enc.ray_d, ray, zw, pos, dir);
    auto put = [&](int j, float v) { put_feature(act, blk, j >> 6, uint32_t(row), j & 63, v); };
    if (view) posenc3_rt(dir, enc.sc.n_freq_dir, put);
    else posenc3_rt(pos, enc.sc.n_freq_pos, put);
  }
}

template <int NSPLIT, bool ENC>
__global__ void __launch_bounds__(kMlpThreads, 1)
mlp_kernel(const __grid_constant__ MlpProgram prog, const uint8_t* __restrict__ wblob, const uint8_t* __restrict__ in_tiles,
           float* __restrict__ out, const long long* __restrict__ rows_dev, long long rows_host, int* err_flag,
           const __grid_constant__ EncodeParams enc) {
  static_assert(!ENC || NSPLIT == 1, "fused input encoder: shading net (plain bf16) only");
  using Cfg = MlpCfg<NSPLIT>;
  constexpr int NB = Cfg::kNB;
  const int STAGES = Cfg::stages(prog.in.n_blk);   // a constant for NSPLIT == 2
  constexpr int STAGE_BYTES = Cfg::kStageBytes;
  constexpr int STAGE_K = stage_k_steps(NSPLIT);   // K steps per ring stage
  constexpr int kConsumerWarps = 8, kProducerWarp = 8;
  constexpr int kEncThreads = 96;   // ENC: producer warps 9-11 encode the inputs
  // The launch gives every thread 168 registers (__launch_bounds__(384, 1)); setmaxnreg only moves them between
  // warpgroups, so 2 x kConsumerRegs + kProducerRegs <= 3 x 168 (a consumer increase beyond what the producers released
  // would wait forever).  The shading net's consumers keep 128 accumulator and 64 A-fragment registers live through the
  // MMAs; the encoder warps need more than the weight issuer's 24.
  constexpr int kConsumerRegs = ENC ? 232 : 240, kProducerRegs = ENC ? 40 : 24;
  static_assert(2 * kConsumerRegs + kProducerRegs <= 3 * 168, "registers the launch allocates");

  extern __shared__ uint8_t smem_raw[];
  // 1024-byte aligned.  Offsetting smem_raw (rather than rounding an integer address) keeps every pointer below in the
  // shared state space, so the epilogue's reads of `side` and writes of `act` compile to LDS / STS, not generic accesses.
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* act = smem;   // NSPLIT == 2: [NSPLIT][NB] activation blocks; NSPLIT == 1: [kInSlots] input tiles
  uint8_t* ring = act + Cfg::in_bytes(prog.in.n_blk);                    // [STAGES] stages
  float* side = reinterpret_cast<float*>(ring + size_t(STAGES) * STAGE_BYTES);
  uint64_t* w_full = reinterpret_cast<uint64_t*>(side + kSideFloats);   // [STAGES] the stage has landed
  uint64_t* w_empty = w_full + STAGES;                                   // [STAGES] every consumer warp's MMAs on it retired
  // NSPLIT == 1, [kInSlots]: the slot holds its tile.  NSPLIT == 2, [2]: consumer warpgroup wg's rows of the tile landed
  uint64_t* in_full = w_empty + STAGES;
  uint64_t* in_empty = in_full + kInSlots;                               // [kInSlots] every consumer warp is done with it

  const int warp = __shfl_sync(0xffffffffu, int(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const long long rows = rows_dev ? *rows_dev : rows_host;
  const long long n_tiles = (rows + kTileM - 1) / kTileM;

  // biases and heads: the epilogue reads a different column per lane, which the constant bank would serialise
  for (int i = threadIdx.x; i < kSideFloats; i += blockDim.x) side[i] = prog.side[i];
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&w_full[s], 1);
      mbar_init(&w_empty[s], kConsumerWarps);
    }
    if (NSPLIT == 1) {
      for (int s = 0; s < kInSlots; ++s) {
        mbar_init(&in_full[s], ENC ? kEncThreads : 1);
        mbar_init(&in_empty[s], kConsumerWarps);
      }
    } else {
      for (int g = 0; g < 2; ++g) mbar_init(&in_full[g], 1);
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp >= kProducerWarp) {
    // ===================================================================== producers
    setmaxnreg_dec<kProducerRegs>();
    if (NSPLIT == 1 && warp > kProducerWarp) {
      // ------------------------------------------------------------------- input producer (NSPLIT == 1)
      // Fills the CTA's tiles into the slots in turn, one tile ahead of the consumers: ENC, warps 9-11 encode the rows
      // (P, then V, of every row; 256 row tasks); otherwise one thread copies the packed tile with one bulk copy.
      if (!ENC && !(warp == kProducerWarp + 1 && lane == 0)) return;
      const uint32_t tile_bytes = prog.in.tile_bytes();
      int slot = 0;
      uint32_t phase = 0;
      for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        mbar_wait(&in_empty[slot], phase ^ 1, err_flag, 3);
        uint8_t* dst = act + size_t(slot) * tile_bytes;
        if constexpr (ENC) {
          for (int task = int(threadIdx.x) - 32 * (kProducerWarp + 1); task < 2 * kTileM; task += kEncThreads) {
            const int row = task & (kTileM - 1);
            const bool view = task >= kTileM;
            encode_row(enc, t * kTileM + row, rows, dst + (view ? prog.in_nblk0 : 0) * kBlkBytes, row, view);
          }
          fence_proxy_async_smem();   // generic-proxy stores -> visible to the consumers' wgmma reads
          mbar_arrive(&in_full[slot]);
        } else {
          mbar_arrive_expect_tx(&in_full[slot], tile_bytes);
          bulk_g2s(dst, in_tiles + size_t(t) * tile_bytes, tile_bytes, &in_full[slot]);
        }
        if (++slot == kInSlots) {
          slot = 0;
          phase ^= 1;
        }
      }
      return;
    }
    // -------------------------------------------------------------------- weight producer
    // Stage i of a layer is [128 N rows x 64 K], or [128 x 32] hi then lo when NSPLIT == 2 (pack_layer), N half
    // outermost: the order the consumers walk them in.  It never waits on an input slot.
    if (warp == kProducerWarp && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        for (int l = 0; l < prog.n_layers; ++l) {
          const MlpLayer& L = prog.layers[l];
          const int n_st = layer_stages(L, NSPLIT);
          for (int i = 0; i < n_st; ++i) {
            mbar_wait(&w_empty[stage], phase ^ 1, err_flag, 1);
            mbar_arrive_expect_tx(&w_full[stage], STAGE_BYTES);
            bulk_g2s(ring + size_t(stage) * STAGE_BYTES, wblob + L.w_off + size_t(i) * STAGE_BYTES, STAGE_BYTES, &w_full[stage]);
            if (++stage == STAGES) {
              stage = 0;
              phase ^= 1;
            }
          }
        }
      }
    }
    return;
  }

  // ============================================================================ consumer warpgroups
  setmaxnreg_inc<kConsumerRegs>();
  const int wg = warp >> 2;                               // rows [64 wg, 64 wg + 64) of every tile
  const int tw = threadIdx.x & 127;
  const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2); // accumulator rows r0 and r0 + 8 of this thread
  const int cq = 2 * (lane & 3);                          // column pair inside every 8-column group
  const int bar_id = 1 + wg;                              // named barrier of this warpgroup
  const uint32_t act_s = smem_u32(act);
  const uint32_t ring_s = smem_u32(ring);
  const uint32_t wg_off = uint32_t(wg) * (kBlkBytes / 2); // this warpgroup's rows inside a block
  uint32_t in_s = act_s;                                  // the current tile's input blocks (NSPLIT == 1: its slot)
  auto blk_addr = [&](int term, int blk) -> uint32_t { return in_s + uint32_t(term * NB + blk) * kBlkBytes; };
  const uint64_t desc_hi = make_desc_sw128(0) & ~uint64_t(0x3FFF);
  auto desc = [&](uint32_t addr) -> uint64_t { return desc_hi | uint64_t((addr & 0x3FFFF) >> 4); };
  const uint64_t desc64_hi = make_desc_sw64(0) & ~uint64_t(0x3FFF);   // the split net's weight stages
  auto desc64 = [&](uint32_t addr) -> uint64_t { return desc64_hi | uint64_t((addr & 0x3FFFF) >> 4); };

  // Shading net: the bf16 output of the last LF_OUT_ACT layer as register-A fragments, [K block][K step][register]
  // (hidden column 64 kb + 16 k + ...).  Indexed with compile-time constants only, so it stays in registers.
  uint32_t afrag[4][4][4];
  // The compiler cannot see which layers read afrag (the layer program is read at run time), so every epilogue and every
  // tile start define all of it; the registers a layer does not write are never read.  Otherwise the previous values
  // stay alive through MMAs and epilogues, and spill.
  auto clear_afrag = [&](int kb0, int kb1) {
#pragma unroll
    for (int kb = 0; kb < 4; ++kb)
#pragma unroll
      for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (kb >= kb0 && kb < kb1) afrag[kb][k][j] = 0u;
  };

  int stage = 0;
  uint32_t phase = 0;
  int prev = -1;   // ring stage whose MMAs may still be running
  // One ring stage: wait for it, issue up to STAGE_K K steps through mma(k, B stage address, accumulate), and hand the
  // previous stage back to the producer once its MMAs have retired.
  auto k_block = [&](bool first, int nk, auto mma) {
    mbar_wait(&w_full[stage], phase, err_flag, 2);
    wgmma_fence();
    const uint32_t b = ring_s + uint32_t(stage) * STAGE_BYTES;
#pragma unroll
    for (int k = 0; k < STAGE_K; ++k) {
      if (k < nk) mma(k, b, (first && k == 0) ? 0u : 1u);   // zero-padded tail columns of an input block are not multiplied
    }
    wgmma_commit();
    wgmma_wait<1>();   // the previous stage's MMAs have retired: hand it back to the producer
    if (prev >= 0 && lane == 0) mbar_arrive(&w_empty[prev]);
    prev = stage;
    if (++stage == STAGES) {
      stage = 0;
      phase ^= 1;
    }
  };

  // NSPLIT == 2: one thread of the warpgroup bulk-copies the warpgroup's 64 rows of tile tt's input blocks (8 KB of each
  // block of each term) into its rows of activation blocks 0 .. in_nblk0 - 1 of both terms, completing on in_full[wg].
  auto fetch_input = [&](long long tt) {
    if (tw != 0) return;
    const uint8_t* src = in_tiles + size_t(tt) * prog.in.tile_bytes() + wg_off;
    mbar_arrive_expect_tx(&in_full[wg], uint32_t(NSPLIT * prog.in_nblk0) * (kBlkBytes / 2));
    for (int term = 0; term < NSPLIT; ++term)
      for (int b = 0; b < prog.in_nblk0; ++b)
        bulk_g2s(act + size_t(term * NB + b) * kBlkBytes + wg_off, src + prog.in.blk_off(term, b), kBlkBytes / 2, &in_full[wg]);
  };
  if (NSPLIT == 2 && blockIdx.x < n_tiles) fetch_input(blockIdx.x);

  int in_slot = 0;
  uint32_t in_phase = 0;
  for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    if constexpr (NSPLIT == 2) {
      mbar_wait(&in_full[wg], in_phase, err_flag, 4);   // this warpgroup's rows of the tile's inputs have landed
      in_phase ^= 1;
    } else {
      mbar_wait(&in_full[in_slot], in_phase, err_flag, 4);   // the producer has filled this tile's slot
      in_s = act_s + uint32_t(in_slot) * prog.in.tile_bytes();
      clear_afrag(0, 4);
    }
    float alpha[2] = {0.0f, 0.0f};
    for (int l = 0; l < prog.n_layers; ++l) {
      const MlpLayer& L = prog.layers[l];
      float acc[2][64];   // written by the first MMA of each half (accumulate = 0): K block 0 has at least one K step
#pragma unroll
      for (int nh = 0; nh < 2; ++nh) {
        if (nh >= L.n_half) break;
        if (NSPLIT == 2) {
          // K block kb in stages of STAGE_K K steps, [128 x 32] hi then lo (SWIZZLE_64B); K steps past k_cnt have none
          for (int kb = 0; kb < L.n_kb; ++kb) {
            for (int k0 = 0; k0 < L.k_cnt[kb]; k0 += STAGE_K) {
              const uint32_t a_hi = blk_addr(0, kb) + wg_off + 32 * k0;
              const uint32_t a_lo = a_hi + uint32_t(NB) * kBlkBytes;
              k_block(kb == 0 && k0 == 0, L.k_cnt[kb] - k0, [&](int k, uint32_t b_hi, uint32_t accumulate) {
                const uint32_t b_lo = b_hi + uint32_t(kBlkBytes / 2);
                wgmma_m64n128_bf16(acc[nh], desc(a_hi + 32 * k), desc64(b_hi + 32 * k), accumulate);
                wgmma_m64n128_bf16(acc[nh], desc(a_lo + 32 * k), desc64(b_hi + 32 * k), 1u);
                wgmma_m64n128_bf16(acc[nh], desc(a_hi + 32 * k), desc64(b_lo + 32 * k), 1u);
              });
            }
          }
        } else {
          auto from_smem = [&](int blk) {
            const uint32_t a = blk_addr(0, blk) + wg_off;
            return [&, a](int k, uint32_t b, uint32_t accumulate) {
              wgmma_m64n128_bf16(acc[nh], desc(a + 32 * k), desc(b + 32 * k), accumulate);
            };
          };
#pragma unroll
          for (int ib = 0; ib < NB; ++ib) {
            if (ib >= L.in_first) break;
            k_block(ib == 0, L.k_cnt[ib], from_smem(ib));
          }
#pragma unroll
          for (int hb = 0; hb < 4; ++hb) {
            if (hb >= L.n_hid) break;
            k_block(hb == 0 && L.in_first == 0, 4, [&](int k, uint32_t b, uint32_t accumulate) {
              wgmma_m64n128_bf16_rs(acc[nh], afrag[hb][k], desc(b + 32 * k), accumulate);
            });
          }
          if (L.in_last) k_block(L.n_kb == 1, L.k_cnt[L.n_kb - 1], from_smem(prog.in_nblk0));   // V
        }
      }
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(&w_empty[prev]);
      prev = -1;
      // NSPLIT == 2: the tile's last layer fetches the next tile's inputs, before its epilogue when that writes no
      // activations (the sampling net's LF_FINAL_RAW layer), else after it
      const bool fetch_next = l + 1 == prog.n_layers && t + gridDim.x < n_tiles;
      const bool fetch_early = fetch_next && !(L.flags & LF_OUT_ACT);
      if constexpr (NSPLIT == 2) {
        // all of the warpgroup's MMAs retired: the A blocks in shared memory may be overwritten in place
        named_bar_sync(bar_id, 128);
        // The bulk copy (async proxy) overwrites this warpgroup's rows of the input blocks.  The wgmma reads of them (async
        // proxy) retired: wait_group 0 in every warp, then the barrier.  The generic-proxy stores of earlier epilogues
        // that wrote them were each followed by fence.proxy.async and the barrier after that epilogue, so they are
        // ordered before the copy.  This layer's epilogue writes only global memory and registers.
        if (fetch_early) fetch_input(t + gridDim.x);
      } else {
        // the tile's last MMAs retired: its slot goes back to the input producer
        if (l + 1 == prog.n_layers && lane == 0) mbar_arrive(&in_empty[in_slot]);
      }

      // ------------------------------------------------------------------ epilogue
      // Instantiated per set of layer flags (a compile-time constant for the sets the networks use): with no branches in
      // the unrolled column loop the compiler batches the bias / head loads ahead of the dependent adds and stores.
      auto epilogue = [&](auto flags) {
        float rgb[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
        if (NSPLIT == 1 && !(flags & LF_OUT_ACT)) clear_afrag(0, 4);
#pragma unroll
        for (int nh = 0; nh < 2; ++nh) {
          if (nh >= L.n_half) {
            if (NSPLIT == 1 && (flags & LF_OUT_ACT)) clear_afrag(2 * nh, 4);
            break;
          }
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const int col = nh * 128 + 8 * i + cq;
            const float2 b = *reinterpret_cast<const float2*>(side + L.bias_off + col);
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
              const int row = r0 + 8 * rr;
              float v0 = acc[nh][4 * i + 2 * rr] + b.x;
              float v1 = acc[nh][4 * i + 2 * rr + 1] + b.y;
              if (flags & LF_FINAL_RAW) {
                const long long grow = t * kTileM + row;
                if (grow < rows) *reinterpret_cast<float2*>(out + grow * prog.out_cols + col) = make_float2(v0, v1);
                continue;
              }
              if (flags & LF_RELU) {
                v0 = fmaxf(v0, 0.0f);
                v1 = fmaxf(v1, 0.0f);
              }
              if (flags & LF_ALPHA_DOT) {
                const float2 w = *reinterpret_cast<const float2*>(side + prog.alpha_w_off + col);
                alpha[rr] = fmaf(v1, w.y, fmaf(v0, w.x, alpha[rr]));
              }
              if (flags & LF_OUT_ACT) {
                const uint32_t hi = bf16x2(v0, v1);
                if (NSPLIT == 1) {
                  afrag[2 * nh + (i >> 3)][(i >> 1) & 3][2 * (i & 1) + rr] = hi;   // ptx.cuh: wgmma_m64n128_bf16_rs
                } else {
                  const uint32_t off = uint32_t(col >> 6) * kBlkBytes + sw128_offset(uint32_t(row), uint32_t(col & 63));
                  *reinterpret_cast<uint32_t*>(act + off) = hi;
                  *reinterpret_cast<uint32_t*>(act + NB * kBlkBytes + off) = bf16x2_lo(v0, v1, hi);
                }
              }
              if (flags & LF_FINAL_RGB) {
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                  const float2 w = *reinterpret_cast<const float2*>(side + prog.rgb_w_off + k * 128 + col);
                  rgb[rr][k] = fmaf(v1, w.y, fmaf(v0, w.x, rgb[rr][k]));
                }
              }
            }
          }
        }
        if (flags & LF_FINAL_RGB) {
          // the four lanes of a row hold partial dot products over interleaved column pairs
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            float a = alpha[rr], c0 = rgb[rr][0], c1 = rgb[rr][1], c2 = rgb[rr][2];
#pragma unroll
            for (int m = 1; m <= 2; m <<= 1) {
              a += __shfl_xor_sync(0xffffffffu, a, m);
              c0 += __shfl_xor_sync(0xffffffffu, c0, m);
              c1 += __shfl_xor_sync(0xffffffffu, c1, m);
              c2 += __shfl_xor_sync(0xffffffffu, c2, m);
            }
            const long long grow = t * kTileM + r0 + 8 * rr;
            if ((lane & 3) == 0 && grow < rows)
              reinterpret_cast<float4*>(out)[grow] = make_float4(c0 + side[prog.rgb_b_off], c1 + side[prog.rgb_b_off + 1],
                                                                 c2 + side[prog.rgb_b_off + 2], a + side[prog.alpha_b_off]);
          }
        }
      };
      using F = uint8_t;
      constexpr F kEpiFlags = LF_RELU | LF_ALPHA_DOT | LF_OUT_ACT | LF_FINAL_RAW | LF_FINAL_RGB;
      switch (L.flags & kEpiFlags) {
        case LF_RELU | LF_OUT_ACT: epilogue(ConstFlags<LF_RELU | LF_OUT_ACT>{}); break;
        case LF_RELU | LF_OUT_ACT | LF_ALPHA_DOT: epilogue(ConstFlags<LF_RELU | LF_OUT_ACT | LF_ALPHA_DOT>{}); break;
        case LF_OUT_ACT: epilogue(ConstFlags<LF_OUT_ACT>{}); break;
        case LF_RELU | LF_FINAL_RGB: epilogue(ConstFlags<LF_RELU | LF_FINAL_RGB>{}); break;
        case LF_FINAL_RAW: epilogue(ConstFlags<LF_FINAL_RAW>{}); break;
        default: epilogue(F(L.flags)); break;   // any other combination: the same code with run-time tests
      }
      if constexpr (NSPLIT == 2) {
        fence_proxy_async_smem();        // generic-proxy stores -> visible to the next layer's wgmma reads
        named_bar_sync(bar_id, 128);
        if (fetch_next && !fetch_early) fetch_input(t + gridDim.x);   // its activation stores are fenced: as above
      }
    }
    if (NSPLIT == 1 && ++in_slot == kInSlots) {
      in_slot = 0;
      in_phase ^= 1;
    }
  }
}

// -------------------------------------------------------------------------------------------------
// fp32 feature rows [rows, n_feat] -> packed tiles of format `fmt`.
// One thread per (row, block, 16-byte chunk): 8 consecutive source columns.
__global__ void pack_rows_kernel(const float* __restrict__ x, long long rows_host, const long long* __restrict__ rows_dev,
                                 int n_feat, const __grid_constant__ TileFormat fmt, uint8_t* __restrict__ tiles) {
  const long long rows = rows_dev ? *rows_dev : rows_host;
  const long long n_tiles = (rows + kTileM - 1) / kTileM;
  const long long total = n_tiles * kTileM * fmt.n_blk * 8;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int chunk = int(i & 7);
    const long long rb = i >> 3;
    const int blk = int(rb % fmt.n_blk);
    const long long row = rb / fmt.n_blk;
    const long long t = row >> 7;
    pack_tile_chunk(fmt, tiles + size_t(t) * fmt.tile_bytes(), blk, uint32_t(row & (kTileM - 1)), chunk,
                    [&](int c) { return row < rows ? x[row * n_feat + c] : 0.0f; });
  }
}

// -------------------------------------------------------------------------------------------------
cudaError_t set_max_dyn_smem_once(const void* func, int bytes, unsigned long long* done) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 64 && ((__atomic_load_n(done, __ATOMIC_ACQUIRE) >> dev) & 1ull)) return cudaSuccess;
  e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return e;
  if (dev < 64) __atomic_fetch_or(done, 1ull << dev, __ATOMIC_RELEASE);   // two threads may both set the (idempotent) attribute
  return cudaSuccess;
}

template <int NSPLIT, bool ENC>
static cudaError_t launch_mlp_t(const MlpProgram& prog, const uint8_t* wblob, const uint8_t* in_tiles, float* out,
                                const long long* rows_dev, long long rows_host, int* err_flag, int num_sms, cudaStream_t stream,
                                const EncodeParams& enc) {
  static unsigned long long attr_done = 0;   // per device
  if (prog.in.n_blk < 1 || prog.in.n_blk > 3) return cudaErrorInvalidValue;
  const size_t smem = MlpCfg<NSPLIT>::smem_bytes(prog.in.n_blk);
  auto kernel = mlp_kernel<NSPLIT, ENC>;
  cudaError_t e = set_max_dyn_smem_once(reinterpret_cast<const void*>(kernel), int(MlpCfg<NSPLIT>::kMaxSmemBytes), &attr_done);
  if (e != cudaSuccess) return e;
  long long grid = num_sms;   // persistent: one CTA per SM
  if (!rows_dev) {
    const long long n_tiles = (rows_host + kTileM - 1) / kTileM;
    if (n_tiles < grid) grid = n_tiles < 1 ? 1 : n_tiles;
  }
  kernel<<<unsigned(grid), kMlpThreads, smem, stream>>>(prog, wblob, in_tiles, out, rows_dev, rows_host, err_flag, enc);
  return cudaGetLastError();
}

cudaError_t launch_mlp(const MlpProgram& prog, const uint8_t* wblob, const uint8_t* in_tiles, float* out,
                       const long long* rows_dev, long long rows_host, int* err_flag, int num_sms, cudaStream_t stream,
                       const EncodeParams* enc) {
  if (enc) {   // shading net with the fused input encoder
    if (prog.in.n_terms != 1) return cudaErrorInvalidValue;
    return launch_mlp_t<1, true>(prog, wblob, in_tiles, out, rows_dev, rows_host, err_flag, num_sms, stream, *enc);
  }
  if (prog.in.n_terms == 2) return launch_mlp_t<2, false>(prog, wblob, in_tiles, out, rows_dev, rows_host, err_flag, num_sms, stream, EncodeParams{});
  return launch_mlp_t<1, false>(prog, wblob, in_tiles, out, rows_dev, rows_host, err_flag, num_sms, stream, EncodeParams{});
}

cudaError_t launch_pack_rows(const float* x, long long rows, const long long* rows_dev, int n_feat, const TileFormat& fmt,
                             uint8_t* tiles, int num_sms, cudaStream_t stream) {
  long long work = ((rows + kTileM - 1) / kTileM) * kTileM * fmt.n_blk * 8;
  int grid = int((work + 255) / 256);
  if (grid < 1) grid = 1;
  if (grid > 16 * num_sms) grid = 16 * num_sms;
  pack_rows_kernel<<<grid, 256, 0, stream>>>(x, rows, rows_dev, n_feat, fmt, tiles);
  return cudaGetLastError();
}

}  // namespace adn
