// Reduced-size inverse DCT of the scaled decoder (libjpeg scale_num = 1, scale_denom = 2 / 4 / 8): dequantise an 8x8
// coefficient block and output 4x4, 2x2 or 1x1 samples, the arithmetic of libjpeg-turbo's jidctred.c
// (jpeg_idct_4x4 / _2x2 / _1x1).  Integer, bit-exact:
//  - 4x4: the even part from inputs 0, 2, 6 and the odd part from 1, 3, 5, 7 of each column, column 4 left out,
//    then the same on the four rows; 2x2: DC and the odd inputs only, columns 2, 4 and 6 left out.  Dequantised with
//    the islow multipliers (the raw quantiser values), CONST_BITS 13, PASS1_BITS 2, 32-bit intermediates as in
//    k_idct_dequant; +128 and a saturating clamp, the semantics of the SIMD forms the library runs.
//  - 1x1: (dc * q0 + 4) >> 3 through the C range-limit table (the library has no SIMD form of it): the value is read
//    modulo 1024 as a signed number, then +128 and clamped.
// One thread per block; one launch covers every plane of a JPEG whose DCT scaled size is S (k_idct_scaled_batch: of
// many JPEGs).
#include "idct_block.cuh"
#include "kernels.cuh"

namespace uhdr_b200 {

namespace {

template <int S>
__global__ void __launch_bounds__(128) k_idct_scaled(const __grid_constant__ IdctScaledParams p) {
  __shared__ uint16_t sq[3][64];
  for (int i = threadIdx.x; i < p.nplanes * 64; i += blockDim.x) sq[i >> 6][i & 63] = p.plane[i >> 6].q[i & 63];
  __syncthreads();
  const int gb = blockIdx.x * blockDim.x + threadIdx.x;
  if (gb >= p.block_end[p.nplanes - 1]) return;
  const int c = gb < p.block_end[0] ? 0 : gb < p.block_end[1] ? 1 : 2;
  const IdctScaledParams::Plane& pl = p.plane[c];  // __grid_constant__: read in place, no local copy
  idct_scaled_block<S>(pl.coefs, sq[c], gb - (c == 0 ? 0 : p.block_end[c - 1]), pl.wblocks, pl.dst, pl.dst_stride, pl.dst_w, pl.dst_h);
}

// every plane of a batch in one launch: each CTA covers 128 blocks of one plane
template <int S>
__global__ void __launch_bounds__(128) k_idct_scaled_batch(const IdctBatchPlane* __restrict__ planes, const unsigned* __restrict__ cta_end,
                                                           unsigned n) {
  const unsigned j = batch_find(cta_end, n, blockIdx.x);
  const IdctBatchPlane& p = planes[j];
  __shared__ uint16_t sq[64];
  if (threadIdx.x < 64) sq[threadIdx.x] = p.q[threadIdx.x];
  __syncthreads();
  const int local = (int)(blockIdx.x - (j ? cta_end[j - 1] : 0)) * 128 + threadIdx.x;
  if (local >= p.blocks) return;
  idct_scaled_block<S>(p.coefs, sq, local, p.wblocks, p.dst, p.dst_stride, p.dst_w, p.dst_h);
}

// every plane of a ladder at every size it asks for, in one launch: each CTA covers 128 blocks of one plane, and a
// thread writes each output of its block in turn (the block's 128 bytes come from HBM once, the re-reads hit L1)
__global__ void __launch_bounds__(128) k_idct_multi(const IdctMultiPlane* __restrict__ planes, const unsigned* __restrict__ cta_end,
                                                    unsigned n) {
  const unsigned j = batch_find(cta_end, n, blockIdx.x);
  const IdctMultiPlane& p = planes[j];
  __shared__ uint16_t sq[64];
  if (threadIdx.x < 64) sq[threadIdx.x] = p.q[threadIdx.x];
  __syncthreads();
  const int local = (int)(blockIdx.x - (j ? cta_end[j - 1] : 0)) * 128 + threadIdx.x;
  if (local >= p.blocks) return;
#pragma unroll 1
  for (int i = 0; i < p.nout; i++) {
    const IdctMultiPlane::Out& o = p.out[i];
    switch (o.s) {
      case 8: {
        const int by = local / p.wblocks, bx = local - by * p.wblocks;
        idct_dequant_block(p.coefs, sq, p.wblocks, bx, by, o.dst, o.dst_stride, o.dst_w, o.dst_h);
        break;
      }
      case 4: idct_scaled_block<4>(p.coefs, sq, local, p.wblocks, o.dst, o.dst_stride, o.dst_w, o.dst_h); break;
      case 2: idct_scaled_block<2>(p.coefs, sq, local, p.wblocks, o.dst, o.dst_stride, o.dst_w, o.dst_h); break;
      default: idct_scaled_block<1>(p.coefs, sq, local, p.wblocks, o.dst, o.dst_stride, o.dst_w, o.dst_h); break;
    }
  }
}

}  // namespace

cudaError_t launch_idct_multi(const IdctMultiPlane* planes, const unsigned* cta_end, unsigned n, unsigned ctas, cudaStream_t s) {
  if (!ctas) return cudaSuccess;
  count_launches(1);
  k_idct_multi<<<ctas, 128, 0, s>>>(planes, cta_end, n);
  return cudaGetLastError();
}

cudaError_t launch_idct_scaled_batch(const IdctBatchPlane* planes, const unsigned* cta_end, unsigned n, unsigned ctas, int size,
                                     cudaStream_t s) {
  if (!ctas) return cudaSuccess;
  count_launches(1);
  switch (size) {
    case 4: k_idct_scaled_batch<4><<<ctas, 128, 0, s>>>(planes, cta_end, n); break;
    case 2: k_idct_scaled_batch<2><<<ctas, 128, 0, s>>>(planes, cta_end, n); break;
    case 1: k_idct_scaled_batch<1><<<ctas, 128, 0, s>>>(planes, cta_end, n); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

cudaError_t launch_idct_scaled(const IdctScaledParams& p, int size, cudaStream_t s) {
  if (p.nplanes < 1 || p.nplanes > 3) return cudaErrorInvalidValue;
  const int blocks = p.block_end[p.nplanes - 1];
  if (blocks <= 0) return cudaSuccess;
  const dim3 g((blocks + 127) / 128), b(128);
  count_launches(1);
  switch (size) {
    case 4: k_idct_scaled<4><<<g, b, 0, s>>>(p); break;
    case 2: k_idct_scaled<2><<<g, b, 0, s>>>(p); break;
    case 1: k_idct_scaled<1><<<g, b, 0, s>>>(p); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

}  // namespace uhdr_b200
