// Forward block stage: 8 lanes per 8x8 block.
//   pass 1: lane (b, r) loads row r of block b (8 bytes; RGB: 24 bytes + jccolor.c conversion),
//           runs the 1-D islow DCT on it in registers and parks the row in a warp-private,
//           bank-padded shared-memory tile
//   pass 2: lane (b, c) reads column c, runs the 1-D DCT, quantises with the exact reciprocal
//           (floor(a/d) == umulhi(a, ceil(2^32/d)) while a*d < 2^32), scatters the 8 coefficients
//           to their (zigzag) positions
//   k_fdct8 (coefficient output): lane (b, j) writes 16 bytes; a warp writes 4 blocks = 512 contiguous bytes
//   k_fdct8_code (device entropy coder follows): the quantised blocks stay in shared memory, one LANE per
//           block turns them into finished AC bit strings (see code_block_lane)
// All planes of an image go in ONE launch, the three components of an RGB888 gain map are produced
// from one read of the pixels.
// Arithmetic is libjpeg-turbo's jccolor.c / jfdctint.c / jcdctmgr.c integer arithmetic: bit-exact.
#include <cstring>

#include "kernels.cuh"
#include "runtime.h"

namespace uhdr_b200 {

namespace {

#define C_BITS 13
#define P1_BITS 2
#define DESC(x, n) (((x) + (1 << ((n)-1))) >> (n))

template <int PASS>
__device__ __forceinline__ void dct1d(int d[8]) {
  const int tmp0 = d[0] + d[7], tmp7 = d[0] - d[7], tmp1 = d[1] + d[6], tmp6 = d[1] - d[6];
  const int tmp2 = d[2] + d[5], tmp5 = d[2] - d[5], tmp3 = d[3] + d[4], tmp4 = d[3] - d[4];
  const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  constexpr int sh = PASS == 0 ? C_BITS - P1_BITS : C_BITS + P1_BITS;
  if (PASS == 0) {
    d[0] = (tmp10 + tmp11) << P1_BITS;
    d[4] = (tmp10 - tmp11) << P1_BITS;
  } else {
    d[0] = DESC(tmp10 + tmp11, P1_BITS);
    d[4] = DESC(tmp10 - tmp11, P1_BITS);
  }
  int z1 = (tmp12 + tmp13) * 4433;
  d[2] = DESC(z1 + tmp13 * 6270, sh);
  d[6] = DESC(z1 + tmp12 * (-15137), sh);
  z1 = tmp4 + tmp7;
  int z2 = tmp5 + tmp6, z3 = tmp4 + tmp6, z4 = tmp5 + tmp7;
  const int z5 = (z3 + z4) * 9633;
  const int t4 = tmp4 * 2446, t5 = tmp5 * 16819, t6 = tmp6 * 25172, t7 = tmp7 * 12299;
  z1 *= -7373;
  z2 *= -20995;
  z3 = z3 * (-16069) + z5;
  z4 = z4 * (-3196) + z5;
  d[7] = DESC(t4 + z1 + z3, sh);
  d[5] = DESC(t5 + z2 + z4, sh);
  d[3] = DESC(t6 + z2 + z3, sh);
  d[1] = DESC(t7 + z1 + z4, sh);
}

// natural index -> zigzag position
__device__ const uint8_t kUnzigTab[64] = {0,  1,  5,  6,  14, 15, 27, 28, 2,  4,  7,  13, 16, 26, 29, 42, 3,  8,  12, 17, 25, 30,
                                          41, 43, 9,  11, 18, 24, 31, 40, 44, 53, 10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38,
                                          46, 51, 55, 60, 21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57, 58, 62, 63};
__device__ __forceinline__ int unzig_rt(int n) { return kUnzigTab[n]; }

constexpr int kTileStride = 72;  // ints per block tile: 64 + 8 padding (4 blocks of a warp on distinct banks)

// Entropy-coder front end (jchuff.c encode_one_block).  Per block it leaves
//   * "meta", one uint4: x = number of code bits of its AC part (run/size Huffman codes, magnitude
//     bits, a ZRL per 16 zeros, EOB unless coefficient 63 is non-zero) << 16 | the DC value; y, z, w =
//     the first 96 bits of the AC part's finished bit string (EOB included), MSB first;
//   * bit strings longer than 96 bits: all their words in the block's slot.
// huffman.cu then only prepends the DC code (which needs the neighbouring block) and concatenates bit
// strings; coefficients are never stored for the device path.
// One LANE codes one block, 32 blocks of a warp at a time: the transform needs 8 lanes per block, but a
// typical block has a handful of non-zero coefficients, and cooperating lanes spend their instructions on
// shuffles and on work that is uniform over the group.  So a warp first transforms and quantises 32 blocks
// (8 rounds of 4) into a staging area (zigzag order, 16 bit, 144-byte pitch: the 128-bit reads of the mask
// scan are conflict free), then every lane walks the non-zero mask of its own block and shifts code words
// into a 64-bit register; the trip count of a warp is the largest non-zero count of its 32 blocks.
constexpr int kStagePitch = 72;   // int16 per staged block

struct BitSink {
  unsigned long long acc = 0;   // low `nacc` bits pending
  unsigned nacc = 0, w = 0, bits = 0, c0 = 0, c1 = 0, c2 = 0;
  uint32_t* slot;               // global: the block's 64-word slot (null: dead block)
  __device__ __forceinline__ void emit(unsigned word) {
    if (w == 0) c0 = word;
    else if (w == 1) c1 = word;
    else if (w == 2) c2 = word;
    else if (slot) slot[w] = word;
    w++;
  }
  __device__ __forceinline__ void put(unsigned code, unsigned len) {   // len <= 26
    acc = (acc << len) | code;
    nacc += len;
    bits += len;
    if (nacc >= 32) {
      nacc -= 32;
      emit((unsigned)(acc >> nacc));
    }
  }
  __device__ __forceinline__ void finish() {
    if (nacc) emit((unsigned)(acc << (32 - nacc)));
    if (bits > 96 && slot) { slot[0] = c0; slot[1] = c1; slot[2] = c2; }
  }
};

__device__ __forceinline__ void code_block_lane(const int16_t* t16, const uint32_t* acb, uint32_t* slot, uint4* meta_out) {
  auto nz2 = [](unsigned w) { return ((w & 0xffffu) ? 1u : 0u) | ((w >> 16) ? 2u : 0u); };
  unsigned lo = 0, hi = 0;
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const uint4 q = *(const uint4*)(t16 + 8 * j);
    const unsigned m8 = nz2(q.x) | (nz2(q.y) << 2) | (nz2(q.z) << 4) | (nz2(q.w) << 6);
    if (j < 4) lo |= m8 << (8 * j);
    else hi |= m8 << (8 * (j - 4));
  }
  BitSink S;
  S.slot = slot;
  const unsigned zrl = acb[0xF0] & 0xff, zcode = acb[0xF0] >> 8;
  int prev = 0;
  unsigned long long m = (((unsigned long long)hi << 32) | lo) & ~1ull;
  while (m) {
    const int k = __ffsll((long long)m) - 1;
    m &= m - 1;
    int run = k - prev - 1;
    prev = k;
    while (run >= 16) {
      S.put(zcode, zrl);
      run -= 16;
    }
    const int v = t16[k];
    const int nb = 32 - __clz(abs(v));
    const uint32_t e = acb[(run << 4) | nb];
    const unsigned low = (unsigned)(v < 0 ? v - 1 : v) & ((1u << nb) - 1u);
    S.put(((e >> 8) << nb) | low, (e & 0xff) + nb);
  }
  if (!(hi >> 31)) S.put(acb[0] >> 8, acb[0] & 0xff);
  S.finish();
  if (meta_out) *meta_out = make_uint4((S.bits << 16) | ((unsigned)(int)t16[0] & 0xffffu), S.c0, S.c1, S.c2);
}

// transform + quantise the block whose row this lane holds; the quantised block goes to `st` (16 bit,
// zigzag order) -- the staging entry of the device-coder kernel
__device__ __forceinline__ void block_to_stage(int d[8], int* tile, int lane_b, int lane_r, const unsigned* sdiv,
                                               const unsigned* smag, const uint8_t* sunzig, int16_t* st) {
  dct1d<0>(d);
  int* t = tile + lane_b * kTileStride;
  *(int4*)(t + lane_r * 8) = make_int4(d[0], d[1], d[2], d[3]);
  *(int4*)(t + lane_r * 8 + 4) = make_int4(d[4], d[5], d[6], d[7]);
  __syncwarp();
  const int c = lane_r;
#pragma unroll
  for (int k = 0; k < 8; k++) d[k] = t[k * 8 + c];
  dct1d<1>(d);
  __syncwarp();
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const int n = k * 8 + c;
    const unsigned dv = sdiv[n];
    const unsigned a = (unsigned)abs(d[k]) + (dv >> 1);
    int q = (int)__umulhi(a, smag[n]);
    q = d[k] < 0 ? -q : q;
    st[sunzig[n]] = (int16_t)q;
  }
}

template <bool ZIGZAG>
__device__ __forceinline__ void block_stage(int d[8], int* tile, int lane_b, int lane_r, const unsigned* sdiv,
                                            const unsigned* smag, const uint8_t* sunzig, int16_t* gout_block_base) {
  // pass 1 on this lane's row, park it
  dct1d<0>(d);
  int* t = tile + lane_b * kTileStride;
  *(int4*)(t + lane_r * 8) = make_int4(d[0], d[1], d[2], d[3]);
  *(int4*)(t + lane_r * 8 + 4) = make_int4(d[4], d[5], d[6], d[7]);
  __syncwarp();
  // pass 2 on column c = lane_r
  const int c = lane_r;
#pragma unroll
  for (int k = 0; k < 8; k++) d[k] = t[k * 8 + c];
  dct1d<1>(d);
  __syncwarp();
  // quantise; element k of this column is natural index k*8 + c
  int16_t* t16 = reinterpret_cast<int16_t*>(t);
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const int n = k * 8 + c;
    const unsigned dv = sdiv[n];
    const unsigned a = (unsigned)abs(d[k]) + (dv >> 1);
    int q = (int)__umulhi(a, smag[n]);
    q = d[k] < 0 ? -q : q;
    const int pos = ZIGZAG ? (int)sunzig[n] : n;
    t16[pos] = (int16_t)q;
  }
  __syncwarp();
  // 16 bytes per lane: coefficients [8*lane_r, 8*lane_r + 8) of block lane_b
  const uint4 q = *(const uint4*)(t16 + lane_r * 8);
  if (gout_block_base) *(uint4*)(gout_block_base + lane_r * 8) = q;
  __syncwarp();
}

// row `lane_r` of block (by, bx) of a plane, level shifted; rows past the plane: the encoder helper's pad row
// (jpegencoderhelper.cpp:254-296)
__device__ __forceinline__ void load_plane_row(const Fdct8Plane& pl, int by, int bx, int lane_r, int d[8]) {
  const int y = by * 8 + lane_r;
  if (y >= pl.h) {
#pragma unroll
    for (int k = 0; k < 8; k++) d[k] = pl.fill - 128;
  } else {
    const uint2 v = __ldg((const uint2*)(pl.src + (size_t)y * pl.stride + bx * 8));
#pragma unroll
    for (int k = 0; k < 4; k++) {
      d[k] = (int)((v.x >> (8 * k)) & 0xff) - 128;
      d[4 + k] = (int)((v.y >> (8 * k)) & 0xff) - 128;
    }
  }
}
// RGB888: libjpeg's scanline path replicates the last column / row (jcsample.c, jcprepct.c)
__device__ __forceinline__ void load_rgb_row(const Fdct8Plane& pl, int by, int bx, int lane_r, int r[8], int g[8], int b[8]) {
  const int y = min(by * 8 + lane_r, pl.h - 1);
  const uint8_t* row = pl.src + (size_t)y * pl.stride * 3;
  if (bx * 8 + 8 <= pl.w) {
    const uint2* p = (const uint2*)(row + (size_t)bx * 24);
    const uint2 a = __ldg(p), bb = __ldg(p + 1), cc = __ldg(p + 2);
    const unsigned w[6] = {a.x, a.y, bb.x, bb.y, cc.x, cc.y};
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const int o = 3 * k;
      r[k] = (w[o >> 2] >> (8 * (o & 3))) & 0xff;
      g[k] = (w[(o + 1) >> 2] >> (8 * ((o + 1) & 3))) & 0xff;
      b[k] = (w[(o + 2) >> 2] >> (8 * ((o + 2) & 3))) & 0xff;
    }
  } else {
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const uint8_t* px = row + (size_t)min(bx * 8 + k, pl.w - 1) * 3;
      r[k] = __ldg(px); g[k] = __ldg(px + 1); b[k] = __ldg(px + 2);
    }
  }
}
template <int COMP>
__device__ __forceinline__ void rgb_to_ycc_row(const int r[8], const int g[8], const int b[8], int d[8]) {
#pragma unroll
  for (int k = 0; k < 8; k++) {  // jccolor.c rgb_ycc_convert, SCALEBITS 16
    int v;
    if (COMP == 0) v = (19595 * r[k] + 38470 * g[k] + 7471 * b[k] + 32768) >> 16;
    else if (COMP == 1) v = (-11059 * r[k] - 21709 * g[k] + 32768 * b[k] + (128 << 16) + 32767) >> 16;
    else v = (32768 * r[k] - 27439 * g[k] - 5329 * b[k] + (128 << 16) + 32767) >> 16;
    d[k] = v - 128;
  }
}

// coefficient output (natural order: the parity hook and the host entropy coder's input; zigzag order on request)
template <bool ZIGZAG>
__global__ void __launch_bounds__(256, 4) k_fdct8(const Fdct8Params P) {
  __shared__ unsigned sdiv[2][64], smag[2][64];
  __shared__ int tiles[8][4 * kTileStride];
  __shared__ uint8_t sunzig[64];
  if (threadIdx.x >= 128 && threadIdx.x < 192) sunzig[threadIdx.x - 128] = (uint8_t)unzig_rt(threadIdx.x - 128);
  if (threadIdx.x < 128) {
    const int t = threadIdx.x >> 6, i = threadIdx.x & 63;
    sdiv[t][i] = (unsigned)P.q[t][i] << 3;
    smag[t][i] = P.mag[t][i];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int lane_b = lane >> 3, lane_r = lane & 7;
  const int total_tiles = P.tile_end[P.nplanes - 1];
  // persistent CTAs: tiles of 32 horizontally adjacent blocks, all planes in one flat index space
#pragma unroll 1
  for (int tidx = blockIdx.x; tidx < total_tiles; tidx += gridDim.x) {
    const int pi = tidx < P.tile_end[0] ? 0 : (tidx < P.tile_end[1] ? 1 : 2);
    const Fdct8Plane& pl = P.plane[pi];
    const int local = tidx - (pi ? P.tile_end[pi - 1] : 0);
    const int tiles_x = (pl.wblocks + 31) >> 5;
    const int by = local / tiles_x, tx = local - by * tiles_x;
    const int bx = tx * 32 + warp * 4 + lane_b;
    const bool live = bx < pl.wblocks;
    const int bxc = live ? bx : pl.wblocks - 1;  // dead lanes compute on a valid block, store nothing
    int* tile = tiles[warp];
    const size_t bidx = (size_t)by * pl.wblocks + bx;
    int d[8];
    if (!pl.rgb) {
      load_plane_row(pl, by, bxc, lane_r, d);
      block_stage<ZIGZAG>(d, tile, lane_b, lane_r, sdiv[pl.tq[0]], smag[pl.tq[0]], sunzig, live ? pl.coefs[0] + bidx * 64 : nullptr);
    } else {
      int r[8], g[8], b[8];
      load_rgb_row(pl, by, bxc, lane_r, r, g, b);
      rgb_to_ycc_row<0>(r, g, b, d);
      block_stage<ZIGZAG>(d, tile, lane_b, lane_r, sdiv[pl.tq[0]], smag[pl.tq[0]], sunzig, live ? pl.coefs[0] + bidx * 64 : nullptr);
      rgb_to_ycc_row<1>(r, g, b, d);
      block_stage<ZIGZAG>(d, tile, lane_b, lane_r, sdiv[pl.tq[1]], smag[pl.tq[1]], sunzig, live ? pl.coefs[1] + bidx * 64 : nullptr);
      rgb_to_ycc_row<2>(r, g, b, d);
      block_stage<ZIGZAG>(d, tile, lane_b, lane_r, sdiv[pl.tq[2]], smag[pl.tq[2]], sunzig, live ? pl.coefs[2] + bidx * 64 : nullptr);
    }
  }
}

// device entropy coder follows: per block the AC bit string (meta word, long strings in the slot) instead of
// coefficients.  Work item of a WARP = 32 consecutive blocks (raster order) of a plane, or 8 consecutive
// pixel blocks x 3 components of an RGB888 image (24 of the 32 lanes code).
struct CodeSmem {
  unsigned sdiv[2][64], smag[2][64];
  uint32_t acb[2][256];                 // AC code books (code << 8 | length)
  int tiles[8][4 * kTileStride];
  alignas(16) int16_t stage[8][32 * kStagePitch];
  uint8_t unzig[64];
};

__global__ void __launch_bounds__(256, 4) k_fdct8_code(const __grid_constant__ Fdct8Params P) {
  extern __shared__ uint4 smem_u4[];
  CodeSmem& S = *reinterpret_cast<CodeSmem*>(smem_u4);
  S.acb[0][threadIdx.x] = __ldg(P.acbooks + threadIdx.x);
  S.acb[1][threadIdx.x] = __ldg(P.acbooks + 256 + threadIdx.x);
  if (threadIdx.x >= 128 && threadIdx.x < 192) S.unzig[threadIdx.x - 128] = (uint8_t)unzig_rt(threadIdx.x - 128);
  if (threadIdx.x < 128) {
    const int t = threadIdx.x >> 6, i = threadIdx.x & 63;
    S.sdiv[t][i] = (unsigned)P.q[t][i] << 3;
    S.smag[t][i] = P.mag[t][i];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int lane_b = lane >> 3, lane_r = lane & 7;
  const int total_items = P.tile_end[P.nplanes - 1];
  int* tile = S.tiles[warp];
  int16_t* stage = S.stage[warp];
#pragma unroll 1
  for (int it = blockIdx.x * 8 + warp; it < total_items; it += gridDim.x * 8) {
    const int pi = it < P.tile_end[0] ? 0 : (it < P.tile_end[1] ? 1 : 2);
    const Fdct8Plane& pl = P.plane[pi];
    const int local = it - (pi ? P.tile_end[pi - 1] : 0);
    const int nb = pl.wblocks * pl.hblocks;
    int d[8];
    if (!pl.rgb) {
      const int base = local * 32;
#pragma unroll 1
      for (int s = 0; s < 8; s++) {
        const int f = min(base + s * 4 + lane_b, nb - 1);   // past the end: a valid block, nothing stored later
        const int by = f / pl.wblocks, bx = f - by * pl.wblocks;
        load_plane_row(pl, by, bx, lane_r, d);
        block_to_stage(d, tile, lane_b, lane_r, S.sdiv[pl.tq[0]], S.smag[pl.tq[0]], S.unzig, stage + (s * 4 + lane_b) * kStagePitch);
      }
      __syncwarp();
      const int f = base + lane;
      const bool live = f < nb;
      code_block_lane(stage + lane * kStagePitch, S.acb[pl.hsel[0]], live ? reinterpret_cast<uint32_t*>(pl.coefs[0] + (size_t)f * 128) : nullptr,
                      live && pl.meta[0] ? pl.meta[0] + f : nullptr);
      __syncwarp();
    } else {
      const int base = local * 8;
#pragma unroll 1
      for (int s = 0; s < 2; s++) {
        const int f = min(base + s * 4 + lane_b, nb - 1);
        const int by = f / pl.wblocks, bx = f - by * pl.wblocks;
        int r[8], g[8], b[8];
        load_rgb_row(pl, by, bx, lane_r, r, g, b);
        int16_t* st = stage + (s * 12 + lane_b) * kStagePitch;
        rgb_to_ycc_row<0>(r, g, b, d);
        block_to_stage(d, tile, lane_b, lane_r, S.sdiv[pl.tq[0]], S.smag[pl.tq[0]], S.unzig, st);
        rgb_to_ycc_row<1>(r, g, b, d);
        block_to_stage(d, tile, lane_b, lane_r, S.sdiv[pl.tq[1]], S.smag[pl.tq[1]], S.unzig, st + 4 * kStagePitch);
        rgb_to_ycc_row<2>(r, g, b, d);
        block_to_stage(d, tile, lane_b, lane_r, S.sdiv[pl.tq[2]], S.smag[pl.tq[2]], S.unzig, st + 8 * kStagePitch);
      }
      __syncwarp();
      if (lane < 24) {
        const int s = lane / 12, comp = (lane - s * 12) >> 2;
        const int f = base + s * 4 + (lane & 3);
        const bool live = f < nb;
        code_block_lane(stage + lane * kStagePitch, S.acb[pl.hsel[comp]],
                        live ? reinterpret_cast<uint32_t*>(pl.coefs[comp] + (size_t)f * 128) : nullptr, live && pl.meta[comp] ? pl.meta[comp] + f : nullptr);
      }
      __syncwarp();
    }
  }
}

// k_fdct8_code over the planes of many images (no RGB888): a warp item is 32 consecutive blocks of one plane, found by a
// binary search over the planes' cumulative item counts; a plane's tq[0] picks one of four quantisers (base luma,
// base chroma, map luma, map chroma)
struct Fdct8BatchParams {
  const Fdct8Plane* planes;
  const unsigned* item_end;   // cumulative warp items of the planes
  unsigned nplanes, total;
  uint16_t q[4][64];
  unsigned mag[4][64];
  const uint32_t* acbooks;
};
struct CodeBatchSmem {
  unsigned sdiv[4][64], smag[4][64];
  uint32_t acb[2][256];
  int tiles[8][4 * kTileStride];
  alignas(16) int16_t stage[8][32 * kStagePitch];
  uint8_t unzig[64];
};

__global__ void __launch_bounds__(256, 4) k_fdct8_code_batch(const __grid_constant__ Fdct8BatchParams P) {
  extern __shared__ uint4 smem_u4[];
  CodeBatchSmem& S = *reinterpret_cast<CodeBatchSmem*>(smem_u4);
  S.acb[0][threadIdx.x] = __ldg(P.acbooks + threadIdx.x);
  S.acb[1][threadIdx.x] = __ldg(P.acbooks + 256 + threadIdx.x);
  if (threadIdx.x < 64) S.unzig[threadIdx.x] = (uint8_t)unzig_rt(threadIdx.x);
  {
    const int t = threadIdx.x >> 6, i = threadIdx.x & 63;
    S.sdiv[t][i] = (unsigned)P.q[t][i] << 3;
    S.smag[t][i] = P.mag[t][i];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int lane_b = lane >> 3, lane_r = lane & 7;
  int* tile = S.tiles[warp];
  int16_t* stage = S.stage[warp];
#pragma unroll 1
  for (unsigned it = blockIdx.x * 8 + warp; it < P.total; it += gridDim.x * 8) {
    const unsigned pi = batch_find(P.item_end, P.nplanes, it);
    const Fdct8Plane& pl = P.planes[pi];
    const int local = (int)(it - (pi ? P.item_end[pi - 1] : 0u));
    const int nb = pl.wblocks * pl.hblocks;
    const int tq = pl.tq[0];
    const int base = local * 32;
    int d[8];
#pragma unroll 1
    for (int s = 0; s < 8; s++) {
      const int f = min(base + s * 4 + lane_b, nb - 1);   // past the end: a valid block, nothing stored later
      const int by = f / pl.wblocks, bx = f - by * pl.wblocks;
      load_plane_row(pl, by, bx, lane_r, d);
      block_to_stage(d, tile, lane_b, lane_r, S.sdiv[tq], S.smag[tq], S.unzig, stage + (s * 4 + lane_b) * kStagePitch);
    }
    __syncwarp();
    const int f = base + lane;
    const bool live = f < nb;
    code_block_lane(stage + lane * kStagePitch, S.acb[pl.hsel[0]], live ? reinterpret_cast<uint32_t*>(pl.coefs[0] + (size_t)f * 128) : nullptr,
                    live ? pl.meta[0] + f : nullptr);
    __syncwarp();
  }
}

}  // namespace

void jpeg_std_codebook(int which, uint32_t out[256]);  // jpeg_host.cpp: (code << 8 | length) per symbol

// the two AC code books (luminance, chrominance), once per device; nullptr + last error on failure
static const uint32_t* fdct_device_books() {
  static PerDevice<const void*> books;
  return (const uint32_t*)device_table(books, 2 * 256 * sizeof(uint32_t), [](void* host) {
    jpeg_std_codebook(1, (uint32_t*)host);
    jpeg_std_codebook(3, (uint32_t*)host + 256);
  });
}

cudaError_t launch_fdct8(const Fdct8Params& Pin, cudaStream_t s) {
  count_launches(1);
  Fdct8Params P = Pin;
  const bool code = P.zigzag != 0;   // zigzag launches feed the device entropy coder
  if (code && !(P.acbooks = fdct_device_books())) return cudaErrorUnknown;
  for (int t = 0; t < 2; t++)
    for (int i = 0; i < 64; i++) {
      const unsigned d = (unsigned)P.q[t][i] << 3;
      P.mag[t][i] = d ? (unsigned)((0x100000000ull + d - 1) / d) : 0u;
    }
  int total = 0;
  for (int i = 0; i < 3; i++) {
    if (i < P.nplanes) {
      const Fdct8Plane& pl = P.plane[i];
      if (code) {
        if (pl.wblocks > 0 && pl.hblocks > 0) {
          const int per = pl.rgb ? 8 : 32;   // blocks of the plane per warp item
          total += (pl.wblocks * pl.hblocks + per - 1) / per;
        }
      } else {
        total += ((pl.wblocks + 31) / 32) * pl.hblocks;
      }
    }
    P.tile_end[i] = total;
  }
  if (total == 0) return cudaSuccess;
  static PerDevice<int> wave[2];  // k_fdct8<false>, k_fdct8_code
  const int resident = code ? wave_ctas(wave[1], (const void*)k_fdct8_code, 256, sizeof(CodeSmem))
                            : wave_ctas(wave[0], (const void*)k_fdct8<false>, 256, 0);
  if (!resident) return cudaErrorUnknown;
  if (code) {
    const int need = (total + 7) / 8;
    const int ctas = need < resident ? need : resident;
    k_fdct8_code<<<ctas, 256, sizeof(CodeSmem), s>>>(P);
  } else {
    const int ctas = total < resident ? total : resident;
    k_fdct8<false><<<ctas, 256, 0, s>>>(P);
  }
  return cudaGetLastError();
}

cudaError_t launch_fdct8_code_batch(const Fdct8Plane* planes, const unsigned* item_end, unsigned nplanes, unsigned total_items,
                                    const uint16_t q[4][64], cudaStream_t s) {
  if (!total_items) return cudaSuccess;
  count_launches(1);
  Fdct8BatchParams P;
  memset(&P, 0, sizeof P);
  P.planes = planes;
  P.item_end = item_end;
  P.nplanes = nplanes;
  P.total = total_items;
  if (!(P.acbooks = fdct_device_books())) return cudaErrorUnknown;
  for (int t = 0; t < 4; t++)
    for (int i = 0; i < 64; i++) {
      P.q[t][i] = q[t][i];
      const unsigned d = (unsigned)q[t][i] << 3;
      P.mag[t][i] = d ? (unsigned)((0x100000000ull + d - 1) / d) : 0u;
    }
  static PerDevice<int> wave;
  const int resident = wave_ctas(wave, (const void*)k_fdct8_code_batch, 256, sizeof(CodeBatchSmem));
  if (!resident) return cudaErrorUnknown;
  const unsigned need = (total_items + 7) / 8;
  const unsigned ctas = need < (unsigned)resident ? need : (unsigned)resident;
  k_fdct8_code_batch<<<ctas, 256, sizeof(CodeBatchSmem), s>>>(P);
  return cudaGetLastError();
}

}  // namespace uhdr_b200
