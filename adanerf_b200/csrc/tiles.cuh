// Packed input tiles of the MLP kernels: the one definition of their format, and the bf16 packing every writer of them uses
// (stage 0, stage 3, pack_rows_kernel and the shading kernel's fused encoder).
//
// A tile holds kTileM rows.  It is n_terms x n_blk blocks of [128 rows x 64 bf16 columns], K-major with the SWIZZLE_128B
// layout (the wgmma A operand), term-major: block (term, b) sits at (term * n_blk + b) * kBlkBytes.  Term 0 holds bf16(x);
// with two terms, term 1 holds the residual lo = bf16(x - hi), so that x = hi + lo to ~16 mantissa bits.  Input block b
// holds the feature columns [col0[b], col0[b] + n_col[b]) and zeros after them.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <cstdint>

#include "ptx.cuh"

namespace adn {

constexpr int kTileM = 128;
constexpr int kBlkBytes = 16384;  // one [128 x 64] bf16 SWIZZLE_128B block

struct TileFormat {
  int32_t n_terms;   // 1: bf16; 2: bf16 hi + lo
  int32_t n_blk;     // input blocks per term (at most 3)
  int32_t col0[3];   // first feature column of each input block
  int32_t n_col[3];  // feature columns of each input block (at most 64)
  __host__ __device__ uint32_t blk_off(int term, int b) const { return uint32_t(term * n_blk + b) * kBlkBytes; }
  __host__ __device__ uint32_t tile_bytes() const { return uint32_t(n_terms * n_blk) * kBlkBytes; }
};

// Sampling net: [hi blk0 | hi blk1 | lo blk0 | lo blk1], features 0-63 in block 0 and 64-127 in block 1.
__host__ __device__ inline TileFormat sampling_tiles(int n_in, int n_terms) {
  return TileFormat{n_terms, 2, {0, 64, 0}, {n_in < 64 ? n_in : 64, n_in > 64 ? n_in - 64 : 0, 0}};
}

// Shading net with n_p position and n_v view-direction features (3 + 6 bands each, n_p <= 128, n_v <= 64): [P | V] when
// P fits one block, else [P0 | P1 | V] with P0 = features 0-63.  Each block holds its features and zeros after them.
// The kernel holds the whole tile in one input slot: the P blocks feed layer 0 (and the skip consumer), V the view layer.
// posEnc 10-4: [P | V] = [63 features and a zero column | 27 features and zeros].
__host__ __device__ inline TileFormat shading_tiles(int n_p, int n_v) {
  if (n_p <= 64) return TileFormat{1, 2, {0, n_p, 0}, {n_p, n_v, 0}};
  return TileFormat{1, 3, {0, 64, n_p}, {64, n_p - 64, n_v}};
}
// The number of P blocks of shading_tiles(n_p, .).
__host__ __device__ inline int shading_p_blocks(int n_p) { return n_p > 64 ? 2 : 1; }

// Round to nearest even, a in the low half.
__device__ __forceinline__ uint32_t bf16x2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// The lo term of the pair (a, b) whose hi term is `hi`: bf16(a - hi.a), bf16(b - hi.b).
__device__ __forceinline__ uint32_t bf16x2_lo(float a, float b, uint32_t hi) {
  return bf16x2(a - __uint_as_float(hi << 16), b - __uint_as_float(hi & 0xFFFF0000u));
}

// Features v[0..7] = columns 8 ch .. 8 ch + 7 of an input block, row `row`: packed into their 16-byte chunk of the hi block
// at `hi` and, when `lo` is not null, of the lo block at `lo`.
__device__ __forceinline__ void pack_chunk8(const float* v, uint32_t row, int ch, uint8_t* hi, uint8_t* lo) {
  const uint4 h = make_uint4(bf16x2(v[0], v[1]), bf16x2(v[2], v[3]), bf16x2(v[4], v[5]), bf16x2(v[6], v[7]));
  const uint32_t off = sw128_offset(row, uint32_t(ch * 8));
  *reinterpret_cast<uint4*>(hi + off) = h;
  if (lo)
    *reinterpret_cast<uint4*>(lo + off) =
        make_uint4(bf16x2_lo(v[0], v[1], h.x), bf16x2_lo(v[2], v[3], h.y), bf16x2_lo(v[4], v[5], h.z), bf16x2_lo(v[6], v[7], h.w));
}

// Chunk ch of input block b, row `row`, of the tile at `tile`: feat(c) is feature column c of the row.
template <typename Feat>
__device__ __forceinline__ void pack_tile_chunk(const TileFormat& fmt, uint8_t* tile, int b, uint32_t row, int ch, Feat feat) {
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = (8 * ch + j < fmt.n_col[b]) ? feat(fmt.col0[b] + 8 * ch + j) : 0.0f;
  pack_chunk8(v, row, ch, tile + fmt.blk_off(0, b), fmt.n_terms == 2 ? tile + fmt.blk_off(1, b) : nullptr);
}

// One thread per tile row (a 128-thread CTA): the tile image in shared memory goes to `dst` with one bulk shared -> global
// copy (TMA engine) from thread 0 instead of strided 16-byte global stores.  Before s_tile is filled again, thread 0 waits
// for the copy to have read it (bulk_wait_read_all) and the CTA synchronises; the CTA calls store_tiles_drain() before it
// exits.
__device__ __forceinline__ void flush_tile(const TileFormat& fmt, uint8_t* s_tile, uint8_t* dst) {
  fence_proxy_async_smem();
  __syncthreads();
  if (threadIdx.x == 0) {
    bulk_s2g(dst, s_tile, fmt.tile_bytes());
    bulk_commit();
  }
}

// Packs the thread's features f (a register array, feature c = f[c]) into the image of input blocks 0 and 1, then
// flush_tile.
template <int NF>
__device__ __forceinline__ void store_tile(const TileFormat& fmt, const float (&f)[NF], uint8_t* s_tile, uint8_t* dst) {
#pragma unroll
  for (int b = 0; b < 2; ++b) {
    if (b < fmt.n_blk) {
#pragma unroll
      for (int ch = 0; ch < 8; ++ch)
        pack_tile_chunk(fmt, s_tile, b, threadIdx.x, ch, [&](int c) { return c < NF ? f[c] : 0.0f; });
    }
  }
  flush_tile(fmt, s_tile, dst);
}

// Run-time encodings: a row written one feature at a time.  zero_row clears row `row` of blocks [b0, b1) of every term of
// the image at `tile` (block (term, b) at fmt.blk_off); put_feature then writes feature column `col` of block b, its bf16
// hi term and, with two terms, its lo term -- the bits pack_chunk8 writes for the same value.
__device__ __forceinline__ void zero_row(const TileFormat& fmt, uint8_t* tile, uint32_t row, int b0, int b1) {
  for (int term = 0; term < fmt.n_terms; ++term)
    for (int b = b0; b < b1; ++b)
#pragma unroll
      for (int ch = 0; ch < 8; ++ch)
        *reinterpret_cast<uint4*>(tile + fmt.blk_off(term, b) + sw128_offset(row, uint32_t(ch * 8))) = make_uint4(0u, 0u, 0u, 0u);
}

__device__ __forceinline__ void put_feature(const TileFormat& fmt, uint8_t* tile, int b, uint32_t row, int col, float v) {
  const __nv_bfloat16 hi = __float2bfloat16_rn(v);
  const uint32_t off = sw128_offset(row, uint32_t(col));
  *reinterpret_cast<__nv_bfloat16*>(tile + fmt.blk_off(0, b) + off) = hi;
  if (fmt.n_terms == 2) *reinterpret_cast<__nv_bfloat16*>(tile + fmt.blk_off(1, b) + off) = __float2bfloat16_rn(v - __bfloat162float(hi));
}

__device__ __forceinline__ void store_tiles_drain() {
  if (threadIdx.x == 0) bulk_wait_all();
}

}  // namespace adn
