// Inverse DCT of the JPEG decoder: dequantise an 8x8 coefficient block and write it at a DCT scaled size S of 8, 4, 2 or
// 1 samples per block side (libjpeg scale_denom 1, 2, 4, 8).  The block bodies are in idct_block.cuh:
//  - 8: libjpeg-turbo jidctint.c "islow" (LL&M, CONST_BITS 13, PASS1_BITS 2);
//  - 4x4 / 2x2 / 1x1: jidctred.c (jpeg_idct_4x4 / _2x2 / _1x1).  4x4: the even part from inputs 0, 2, 6 and the odd part
//    from 1, 3, 5, 7 of each column, column 4 left out, then the same on the four rows; 2x2: DC and the odd inputs only,
//    columns 2, 4 and 6 left out.  1x1: (dc * q0 + 4) >> 3 through the C range-limit table (the library has no SIMD
//    form of it): the value is read modulo 1024 as a signed number, then +128 and clamped.
// Dequantised with the raw quantiser values (the islow multipliers), 32-bit intermediates; +128 and a saturating clamp,
// the semantics of the SIMD forms the library runs.  Integer arithmetic, bit-exact.
//
// One thread per block, one flat grid of 128-block CTAs over every plane of a launch: a CTA covers 128 blocks of one
// plane, found from the planes' CTA ends.  k_idct<S> writes each plane's out[0] at size S; k_idct<0> writes every output
// of every plane (a ladder of 1/k decodes), reading each block's 128 bytes from HBM once (the re-reads hit L1).
#include "idct_block.cuh"
#include "kernels.cuh"

namespace uhdr_b200 {

namespace {

// output o of block `local` of plane p at size S, quantiser sq in shared memory
template <int S>
__device__ __forceinline__ void idct_out(const IdctPlane& p, const uint16_t* sq, int local, const IdctPlane::Out& o) {
  if (S == 8) {
    const int by = local / p.wblocks, bx = local - by * p.wblocks;
    idct_dequant_block(p.coefs, sq, p.wblocks, bx, by, o.dst, o.dst_stride, o.dst_w, o.dst_h);
  } else {
    idct_scaled_block<S>(p.coefs, sq, local, p.wblocks, o.dst, o.dst_stride, o.dst_w, o.dst_h);
  }
}

template <int S>
__global__ void __launch_bounds__(128) k_idct(const IdctPlane* __restrict__ planes, const unsigned* __restrict__ cta_end, unsigned n) {
  const unsigned j = batch_find(cta_end, n, blockIdx.x);
  const IdctPlane& p = planes[j];
  __shared__ uint16_t sq[64];
  if (threadIdx.x < 64) sq[threadIdx.x] = p.q[threadIdx.x];
  __syncthreads();
  const int local = (int)(blockIdx.x - (j ? cta_end[j - 1] : 0)) * 128 + threadIdx.x;
  if (local >= p.blocks) return;
  if constexpr (S != 0) {
    idct_out<S>(p, sq, local, p.out[0]);
  } else {
#pragma unroll 1
    for (int i = 0; i < p.nout; i++) {
      const IdctPlane::Out& o = p.out[i];
      switch (o.s) {
        case 8: idct_out<8>(p, sq, local, o); break;
        case 4: idct_out<4>(p, sq, local, o); break;
        case 2: idct_out<2>(p, sq, local, o); break;
        default: idct_out<1>(p, sq, local, o); break;
      }
    }
  }
}

}  // namespace

cudaError_t launch_idct(int size, const IdctPlane* planes, const unsigned* cta_end, unsigned n, unsigned ctas, cudaStream_t s) {
  if (!ctas) return cudaSuccess;
  count_launches(1);
  switch (size) {
    case 8: k_idct<8><<<ctas, 128, 0, s>>>(planes, cta_end, n); break;
    case 4: k_idct<4><<<ctas, 128, 0, s>>>(planes, cta_end, n); break;
    case 2: k_idct<2><<<ctas, 128, 0, s>>>(planes, cta_end, n); break;
    case 1: k_idct<1><<<ctas, 128, 0, s>>>(planes, cta_end, n); break;
    case 0: k_idct<0><<<ctas, 128, 0, s>>>(planes, cta_end, n); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

}  // namespace uhdr_b200
