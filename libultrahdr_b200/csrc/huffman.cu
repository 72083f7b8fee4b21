// Baseline-JPEG entropy coding on the device, bit-identical to libjpeg-turbo's jchuff.c for the
// reference's settings (default Annex-K tables, one interleaved scan, no restart markers), including
// libjpeg's dummy blocks for MCUs that reach past a component's block grid (jccoefct.c
// compress_data: zero AC, DC repeated from the block coded before, jpegencoderhelper.cpp:254-296 for
// the padded sample rows that feed the real edge blocks).
//
// ONE kernel, one pass over the coefficients.  The forward stage (fdct8.cu) leaves, per block, the
// 64-bit mask of its non-zero coefficients, the number of code bits of its AC part and its DC value,
// so a block's total code length is known from 16 bytes and the coefficients are visited exactly
// once, non-zero ones only.  k_huff_encode, per CTA of 256 consecutive blocks of the scan:
//   1. per thread: locate the block (or dummy block) and its DC predecessor, total its code bits
//   2. CTA scan + decoupled look-back over CTAs -> absolute bit offset of every block
//   3. per thread: emit the block's codes into a word-aligned shared-memory image of the CTA's segment
//   4. partial boundary words travel from CTA to CTA (no pre-zeroed stream, no global atomics)
//   5. byte stuffing folded in: the 0xFF bytes of the words a CTA owns are counted, a second
//      look-back gives the number of stuffed zeros in front of them, the CTA writes its final bytes
// Only the final stuffed segment (a few MB at 4K) exists in global memory and crosses PCIe.
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "jpeg.h"

namespace uhdr_b200 {

void jpeg_std_codebook(int which, uint32_t out[256]);

namespace {

constexpr int kEncThreads = 256;
// A CTA takes 256 * bpt consecutive blocks of the scan, bpt (1..8) chosen per launch so that the whole grid
// is resident at once: the per-CTA chain of dependent global round trips (look-backs, boundary words) is
// then paid once per launch instead of once per wave.
constexpr int kMaxBpt = 8;
constexpr int kMaxChunk = kEncThreads * kMaxBpt;
// shared-memory image of the CTA's segment: 2048 words = 256 bits per block on average.  Heavier
// segments (noise at high quality; the worst case is 52 words per block) are produced in several
// windows of this size; a block is encoded only for the windows its bits fall into.
constexpr unsigned kSegWords = 2048;
constexpr unsigned long long kFlagAgg = 1ull << 62, kFlagPrefix = 2ull << 62, kFlagMask = 3ull << 62;

// floor(n / d) for the runtime divisors of the scan geometry: a multiply instead of the ~20-instruction
// integer division.  umulhi(n, ceil(2^32 / d)) is floor(n / d) or one more; the product check takes the
// excess back.  Exact for n < 2^32 - d (q * d must not wrap); here n < 2^27.  Needed: MCUs per row reach
// 8191 (a Y400 frame 65535 wide), so n * d passes 2^32 and the multiply alone is off by one.
struct FastDiv {
  unsigned d, m;  // m = ceil(2^32 / d); d == 1 is flagged with m = 0
  __device__ __forceinline__ unsigned div(unsigned n) const {
    if (!m) return n;
    const unsigned q = __umulhi(n, m);
    return q * d > n ? q - 1 : q;
  }
};

struct HuffFrame {
  const uint32_t* slots[3];  // [block raster][64 words] AC bit string of the block, MSB first (only strings longer than 96 bits)
  const uint4* meta[3];      // {AC code bits << 16 | DC, first three words of the AC bit string} per block (fdct8.cu block_code)
  int wblocks[3], hblocks[3], koff[3];
  FastDiv mw[3];             // blocks per MCU row of the component
  int per[3];                // blocks per MCU of the component (mw * mh)
  FastDiv bpm, mpr;          // blocks per MCU, MCUs per row
  int ncomp, has_dummy;
  int bpt;                   // blocks per thread
  unsigned nblocks;          // blocks of the scan = MCUs x blocks per MCU (dummy blocks included)
};

struct Loc {
  int c;            // component
  bool real;        // false: dummy block (outside the component's block grid)
  unsigned blk;     // raster index inside the component (real blocks)
  long long pred;   // raster index of the last real block of the component before this one in scan order, -1: none
};

// Position s of the scan -> block.  DC prediction runs over the blocks of a component in scan order;
// a dummy block repeats the DC of the block before it (difference 0), so the predecessor that matters
// is the most recent REAL block.  The first block of every MCU is real, so the walk back is short.
__device__ __forceinline__ Loc locate(const HuffFrame& f, unsigned s) {
  Loc L;
  const unsigned m = f.bpm.div(s), k = s - m * f.bpm.d;
  const int c = (f.ncomp > 2 && k >= (unsigned)f.koff[2]) ? 2 : ((f.ncomp > 1 && k >= (unsigned)f.koff[1]) ? 1 : 0);
  const FastDiv mwd = f.mw[c];
  const unsigned mw = mwd.d, per = f.per[c], mh = per / mw;
  const unsigned wb = f.wblocks[c], hb = f.hblocks[c];
  unsigned kk = k - f.koff[c];
  unsigned my = f.mpr.div(m), mx = m - my * f.mpr.d;
  unsigned ky = mwd.div(kk), kx = kk - ky * mw;
  unsigned bx = mx * mw + kx, by = my * mh + ky;
  L.c = c;
  L.real = bx < wb && by < hb;
  L.blk = by * wb + bx;
  L.pred = -1;
  unsigned pm = m;
  const unsigned tries = f.has_dummy ? 2 * per : 1;
  for (unsigned it = 0; it < tries; it++) {
    if (kk > 0) {
      kk--;
    } else {
      if (pm == 0) break;
      pm--;
      my = f.mpr.div(pm);
      mx = pm - my * f.mpr.d;
      kk = per - 1;
    }
    ky = mwd.div(kk);
    kx = kk - ky * mw;
    bx = mx * mw + kx;
    by = my * mh + ky;
    if (bx < wb && by < hb) {
      L.pred = (long long)by * wb + bx;
      break;
    }
  }
  return L;
}

__device__ __forceinline__ unsigned block_exclusive_scan(unsigned v, unsigned* total) {
  __shared__ unsigned warp_sums[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  unsigned x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[wid] = x;
  __syncthreads();
  if (wid == 0) {
    const int nw = blockDim.x >> 5;
    unsigned ws = lane < nw ? warp_sums[lane] : 0;
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned y = __shfl_up_sync(0xffffffffu, ws, o);
      if (lane >= o) ws += y;
    }
    warp_sums[lane] = ws;  // inclusive
  }
  __syncthreads();
  const unsigned base = wid ? warp_sums[wid - 1] : 0;
  if (total) *total = warp_sums[(blockDim.x >> 5) - 1];
  const unsigned r = base + x - v;
  __syncthreads();
  return r;
}

// Chain of per-CTA values (code bits; stuffed zeros).  status[i] carries a 2-bit flag and a 32-bit value:
// kFlagAgg = the value of CTA i alone, kFlagPrefix = the inclusive prefix up to i.  A CTA publishes its
// aggregate as early as it can, does other work, and only then sums its predecessors: by that time they
// have normally all published and the look-back costs one memory round trip.  The whole CTA looks back,
// 256 predecessors per round trip (the grid starts as one wave: nobody holds a prefix yet when the first
// CTAs look back, a one-warp look-back would crawl forward 32 CTAs per round trip).  Predecessors are
// running or finished (ticket order), so the polling loops terminate.
__device__ __forceinline__ void chain_publish(unsigned long long* status, unsigned idx, unsigned agg) {
  if (threadIdx.x == 0) *reinterpret_cast<volatile unsigned long long*>(status + idx) = (idx == 0 ? kFlagPrefix : kFlagAgg) | agg;
}
// returns the exclusive prefix to every thread and publishes the inclusive one
__device__ __forceinline__ unsigned chain_lookback(unsigned long long* status, unsigned idx, unsigned agg) {
  __shared__ unsigned s_w[kEncThreads / 32], s_f[kEncThreads / 32];
  const int j = threadIdx.x, lane = j & 31, wid = j >> 5;
  if (idx == 0) return 0;
  unsigned base = 0;
  long long hi = (long long)idx - 1;  // highest predecessor not yet accounted for
  for (;;) {
    const long long k = hi - j;
    unsigned long long st = kFlagPrefix;  // before element 0: nothing
    if (k >= 0) {
      for (;;) {
        st = *reinterpret_cast<const volatile unsigned long long*>(status + k);
        if (st & kFlagMask) break;
        __nanosleep(200);  // do not starve the stores we are waiting for
      }
    }
    const unsigned pm = __ballot_sync(0xffffffffu, (st & kFlagMask) == kFlagPrefix);
    const int first_prefix = pm ? __ffs(pm) - 1 : 32;  // nearest predecessor of this warp carrying an inclusive prefix
    unsigned v = (lane <= first_prefix && k >= 0) ? (unsigned)(st & 0xffffffffu) : 0u;
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) {
      s_w[wid] = v;
      s_f[wid] = pm;
    }
    __syncthreads();
    bool found = false;
#pragma unroll
    for (int w = 0; w < kEncThreads / 32; w++) {
      if (!found) {
        base += s_w[w];
        found = s_f[w] != 0;
      }
    }
    __syncthreads();
    if (found) break;
    hi -= kEncThreads;
  }
  if (j == 0) *reinterpret_cast<volatile unsigned long long*>(status + idx) = kFlagPrefix | (unsigned long long)(base + agg);
  return base;
}

// One block's codes, jchuff.c encode_one_block, into the window [win, win + wn) of the segment image
// (word indices relative to the CTA's first word).  Words that lie wholly inside the block's bit range
// belong to this thread alone and are stored; the first and the last word are shared with the
// neighbouring blocks and are ORed into the zero-initialised image.
struct Emitter {
  uint32_t* seg;
  unsigned win, wn, first_w, last_w;
  unsigned long long acc;
  int fill;
  unsigned widx;
  __device__ __forceinline__ void store(unsigned v) {
    const unsigned r = widx - win;
    if (r < wn) {
      if (widx == first_w || widx == last_w) atomicOr(seg + r, v);
      else seg[r] = v;
    }
  }
  __device__ __forceinline__ void put(unsigned bits, int n) {
    acc = (acc << n) | bits;
    fill += n;
    if (fill >= 32) {
      store((unsigned)(acc >> (fill - 32)));
      widx++;
      fill -= 32;
    }
  }
};

// DC code, then the block's finished AC bit string (fdct8.cu block_code; EOB included), 32 bits at a time:
// the first three words travel in the block's meta word, longer strings continue in the block's slot
__device__ __forceinline__ void emit_block(Emitter& E, int dc_diff, unsigned nbits, bool real, const uint4* __restrict__ meta,
                                           const uint4* __restrict__ slot, const uint32_t* dcb, const uint32_t* acb) {
  const int mag = abs(dc_diff);
  const int nb = mag ? 32 - __clz(mag) : 0;
  const uint32_t e = dcb[nb];
  const unsigned dclen = (e & 0xff) + nb;
  const unsigned acbits = nbits - dclen;
  uint4 m = make_uint4(0, 0, 0, 0);
  if (real) m = __ldg(meta);
  const unsigned low = (unsigned)(dc_diff < 0 ? dc_diff - 1 : dc_diff) & ((1u << nb) - 1u);
  E.put(((e >> 8) << nb) | low, (int)dclen);
  if (real) {
    uint4 cur = make_uint4(0, m.y, m.z, m.w);
    for (unsigned w = 0; w * 32 < acbits; w++) {
      unsigned word;
      if (w < 3) {
        word = w == 0 ? cur.y : (w == 1 ? cur.z : cur.w);
      } else {
        if (w == 3 || (w & 3) == 0) cur = __ldg(slot + (w >> 2));
        word = (w & 2) ? ((w & 1) ? cur.w : cur.z) : ((w & 1) ? cur.y : cur.x);
      }
      const unsigned n = min(32u, acbits - 32 * w);
      E.put(word >> (32 - n), (int)n);
    }
  } else {  // dummy block: EOB
    const uint32_t eb = acb[0];
    E.put(eb >> 8, (int)(eb & 0xff));
  }
  if (E.fill) E.store((unsigned)(E.acc << (32 - E.fill)));
}

__device__ __forceinline__ unsigned ff_count(unsigned v, int nvalid) {
  unsigned c = 0;
#pragma unroll
  for (int b = 0; b < 4; b++)
    if (b < nvalid && ((v >> (24 - 8 * b)) & 0xff) == 0xff) c++;
  return c;
}

// One scan of k_huff_encode_batch: its frame, its slices of the look-back words, its control words and its output
struct HuffScanDesc {
  HuffFrame f;
  unsigned long long *status, *ffstatus, *tails;
  uint8_t* out;
  unsigned* ctl;     // 16 words, as k_huff_encode's
  unsigned out_cap;
  unsigned pad[3];
};
static_assert(sizeof(HuffScanDesc) % 16 == 0, "HuffScanDesc is copied to shared memory in 16-byte words");

// k_huff_encode_batch: the scan of the CTA's ticket
__device__ __forceinline__ unsigned& batch_scan_slot() {
  __shared__ unsigned s_scan;
  return s_scan;
}

// The body of k_huff_encode (BATCH false: one scan, the kernel's parameters, CTA tickets in ctl[5]) and of
// k_huff_encode_batch (BATCH true: ctl is the global ticket, the CTA's scan is found in `scans` by its ticket).
// status   : bit-count look-back words, one per CTA        ffstatus : the same for the stuffed-zero counts
// tails[i] : (1 << 32 | trailing partial word of CTA i) once known
// ctl[0] <- total bits, ctl[3] <- stuffed bytes, ctl[4] <- overflow flag, ctl[5] = CTA tickets (all zeroed by the caller)
template <bool BATCH>
__device__ __forceinline__ void huff_encode_cta(const HuffFrame& f_arg, const uint32_t* __restrict__ books,
                                                unsigned long long* status_arg, unsigned long long* ffstatus_arg,
                                                unsigned long long* tails_arg, uint8_t* __restrict__ out_arg,
                                                unsigned out_cap_arg, unsigned* ctl_arg, unsigned long long* trace,
                                                const HuffScanDesc* __restrict__ scans, const unsigned* __restrict__ cta_end,
                                                unsigned nscan) {
#define TRACE(k) do { if (trace && threadIdx.x == 0) { unsigned long long t_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_)); trace[(size_t)s_cta * 16 + (k)] = t_; } } while (0)
  __shared__ uint32_t s_books[1024];  // (code << 8 | length): DC lum, AC lum, DC chr, AC chr
  __shared__ uint32_t seg[kSegWords];        // window of the CTA-relative image (bit 0 = the CTA's first code bit)
  __shared__ uint32_t oseg[kSegWords + 1];   // the same window aligned to the words of the stream
  // per block of the chunk: [21:0] raster index, [23:22] component, [24] real (not a dummy block)
  __shared__ uint32_t s_loc[kMaxChunk];
  __shared__ uint16_t s_nb[kMaxChunk];   // code bits
  __shared__ int16_t s_dc[kMaxChunk];    // DC difference
  __shared__ unsigned s_cta, s_predtail, s_ffrun, s_carry;
  const int j = threadIdx.x;
  if (j == 0) {
    if constexpr (BATCH) {
      const unsigned t = atomicAdd(ctl_arg, 1u);   // ticket order: within a scan, every predecessor is running or done
      const unsigned sc = batch_find(cta_end, nscan, t);
      batch_scan_slot() = sc;
      s_cta = t - (sc ? cta_end[sc - 1] : 0u);
    } else {
      s_cta = atomicAdd(ctl_arg + 5, 1u);  // ticket order: every predecessor is already running or done
    }
    s_ffrun = 0;
    s_predtail = 0;
  }
  for (int i = j; i < 1024; i += kEncThreads) s_books[i] = __ldg(books + i);
  __syncthreads();
  const HuffFrame* fp = &f_arg;
  unsigned long long *status = status_arg, *ffstatus = ffstatus_arg, *tails = tails_arg;
  uint8_t* __restrict__ out = out_arg;
  unsigned out_cap = out_cap_arg;
  unsigned* ctl = ctl_arg;
  if constexpr (BATCH) {   // the scan's descriptor into shared memory
    __shared__ uint4 s_desc[sizeof(HuffScanDesc) / 16];
    const uint4* d = reinterpret_cast<const uint4*>(scans + batch_scan_slot());
    for (int i = j; i < (int)(sizeof(HuffScanDesc) / 16); i += kEncThreads) s_desc[i] = __ldg(d + i);
    __syncthreads();
    const HuffScanDesc& D = *reinterpret_cast<const HuffScanDesc*>(s_desc);
    fp = &D.f;
    status = D.status;
    ffstatus = D.ffstatus;
    tails = D.tails;
    out = D.out;
    out_cap = D.out_cap;
    ctl = D.ctl;
  }
  const HuffFrame& f = *fp;
  const unsigned cta = s_cta;
  TRACE(0);
  const int bpt = f.bpt;
  const unsigned chunk = (unsigned)kEncThreads * bpt;
  const unsigned s0 = cta * chunk + j * bpt;   // this thread's first block of the scan

  // 1. the blocks, their code lengths
  unsigned tbits = 0;
  for (int b = 0; b < bpt; b++) {
    const unsigned s = s0 + b, i = j * bpt + b;
    unsigned nbits = 0, loc = 0;
    int dc_diff = 0;
    if (s < f.nblocks) {
      const Loc L = locate(f, s);
      const int c = L.c;
      const int pred = L.pred >= 0 ? (int)(short)(__ldg(&f.meta[c][L.pred].x) & 0xffffu) : 0;
      loc = (unsigned)c << 22;
      if (L.real) {
        const unsigned mx = __ldg(&f.meta[c][L.blk].x);  // AC code bits << 16 | DC
        loc |= L.blk | (1u << 24);
        dc_diff = (int)(short)(mx & 0xffffu) - pred;
        nbits = mx >> 16;
      } else {
        nbits = s_books[(c ? 768 : 256)] & 0xff;  // dummy block: DC difference 0, then EOB
      }
      const int mag = abs(dc_diff);
      const int nb = mag ? 32 - __clz(mag) : 0;
      nbits += (s_books[(c ? 512 : 0) + nb] & 0xff) + nb;
    }
    s_loc[i] = loc;
    s_nb[i] = (uint16_t)nbits;
    s_dc[i] = (int16_t)dc_diff;
    tbits += nbits;
  }

  // 2. bit offsets inside the CTA; the CTA's own total goes out at once, the look-back waits until
  //    the codes are in place (relative to the CTA's first bit)
  TRACE(1);
  unsigned total;
  const unsigned off = block_exclusive_scan(tbits, &total);
  chain_publish(status, cta, total);
  TRACE(2);
  const unsigned nrel = (total + 31) >> 5;       // words of the CTA-relative image
  const bool is_last = (cta + 1) * chunk >= f.nblocks;
  const int npass = nrel > kSegWords ? 2 : 1;  // several windows: count the 0xFF bytes first, write in a second sweep
  // known after the look-back:
  unsigned base = 0, sh = 0, first = 0, nwords = 0, tailbits = 0, lastw = 0, own_end = 0;
  unsigned ffbase = 0;  // stuffed zeros in front of this CTA's words

  for (int pass = 0; pass < npass; pass++) {
    const bool do_write = pass == npass - 1;
    for (unsigned win = 0; win < nrel; win += kSegWords) {
      const unsigned wn = min(kSegWords, nrel - win);
      if (j == 0) s_carry = win ? seg[kSegWords - 1] : 0u;  // last relative word of the previous window
      __syncthreads();
      for (unsigned i = j; i < wn; i += kEncThreads) seg[i] = 0;
      __syncthreads();
      // 3. codes of the blocks that reach into this window
      if (tbits && off + tbits > win * 32 && off < (win + wn) * 32) {
        unsigned pos = off;
        for (int b = 0; b < bpt; b++) {
          const unsigned i = j * bpt + b;
          const unsigned nb = s_nb[i];
          const unsigned pos_lo = pos, pos_hi = pos + nb;
          pos = pos_hi;
          if (!nb || pos_hi <= win * 32 || pos_lo >= (win + wn) * 32) continue;
          const unsigned loc = s_loc[i];
          const int c = (loc >> 22) & 3;
          const size_t blk = loc & 0x3fffffu;
          Emitter E;
          E.seg = seg; E.win = win; E.wn = wn;
          E.first_w = pos_lo >> 5; E.last_w = (pos_hi - 1) >> 5;
          E.acc = 0; E.fill = (int)(pos_lo & 31); E.widx = pos_lo >> 5;
          emit_block(E, (int)s_dc[i], nb, (loc >> 24) & 1, f.meta[c] + blk, reinterpret_cast<const uint4*>(f.slots[c] + blk * 64),
                     s_books + (c ? 512 : 0), s_books + (c ? 768 : 256));
        }
      }
      __syncthreads();
      TRACE(3);
      if (pass == 0 && win == 0) {  // now the predecessors' totals: where the segment starts in the stream
        base = chain_lookback(status, cta, total);
        sh = base & 31;
        first = base >> 5;
        const unsigned endbit = sh + total;      // relative to word `first`
        nwords = (endbit + 31) >> 5;             // words of the stream the segment touches
        tailbits = endbit & 31;
        lastw = endbit >> 5;                     // index of the word holding the trailing partial bits (if any)
        // words this CTA writes out: those whose last bit lies in its segment -- 0 .. lastw-1 -- and, for
        // the last CTA, the padded partial word.  Word 0 may start with bits of the predecessor (sh > 0).
        own_end = lastw + ((is_last && tailbits) ? 1u : 0u);
      }
      TRACE(4);
      // stream-aligned view of the window: stream word i (relative to `first`) = relative words i-1 and i
      // shifted by sh.  This window yields words win .. win+wn-1 and, at the very end, word nrel.
      const bool extra = win + wn == nrel && nwords > nrel;
      const unsigned on = wn + (extra ? 1u : 0u);
      for (unsigned r = j; r < on; r += kEncThreads) {
        const unsigned hi = r ? seg[r - 1] : s_carry, lo = r < wn ? seg[r] : 0u;
        oseg[r] = sh ? __funnelshift_r(lo, hi, sh) : lo;
      }
      __syncthreads();
      // 4. boundary words
      if (j == 0) {
        const bool tail_here = tailbits && lastw >= win && lastw < win + on;
        // a non-degenerate segment hands its trailing partial word on *before* waiting for the
        // predecessor's: otherwise every CTA would wait for the whole chain in front of it
        if (pass == 0 && tail_here && lastw > 0)
          *reinterpret_cast<volatile unsigned long long*>(tails + cta) = (1ull << 32) | oseg[lastw - win];
        if (win == 0 && sh > 0) {  // leading bits of word `first` belong to the predecessor
          if (pass == 0) {
            unsigned long long t;
            for (;;) {
              t = *reinterpret_cast<volatile unsigned long long*>(tails + cta - 1);
              if (t >> 32) break;
              __nanosleep(100);
            }
            s_predtail = (unsigned)t;
          }
          oseg[0] |= s_predtail;
        }
        // the whole segment lies inside word `first` (only a short last CTA can be this small): the
        // merged word is also our trailing partial word
        if (pass == 0 && tail_here && lastw == 0)
          *reinterpret_cast<volatile unsigned long long*>(tails + cta) = (1ull << 32) | oseg[0];
        if (is_last && tail_here) {  // jchuff.c flush_bits: fill the last byte with ones
          const unsigned pad = (8 - (tailbits & 7)) & 7;
          oseg[lastw - win] |= ((1u << pad) - 1u) << (32 - tailbits - pad);
        }
      }
      __syncthreads();
      TRACE(5);
      // 5. byte stuffing: thread j takes wpt consecutive stream words of the window (one in the common case)
      const unsigned wpt = (on + kEncThreads - 1) / kEncThreads;
      const unsigned r0 = j * wpt;
      unsigned cnt = 0;
      for (unsigned u = 0; u < wpt; u++) {
        const unsigned r = r0 + u, i = win + r;
        if (r < on && i < own_end) cnt += ff_count(oseg[r], (is_last && i == lastw) ? (int)((tailbits + 7) >> 3) : 4);
      }
      unsigned ffwin;
      const unsigned ffoff = block_exclusive_scan(cnt, &ffwin);
      TRACE(6);
      if (npass == 1) {
        chain_publish(ffstatus, cta, ffwin);
        ffbase = chain_lookback(ffstatus, cta, ffwin);
      }
      TRACE(7);
      if (do_write) {
        unsigned pos = 4u * (first + win + r0) + ffbase + s_ffrun + ffoff;
        bool ovf = false;
        for (unsigned u = 0; u < wpt; u++) {
          const unsigned r = r0 + u, i = win + r;
          if (r < on && i < own_end) {
            const unsigned v = oseg[r];
            const int nv = (is_last && i == lastw) ? (int)((tailbits + 7) >> 3) : 4;
#pragma unroll
            for (int b = 0; b < 4; b++) {
              if (b < nv) {
                const unsigned byte = (v >> (24 - 8 * b)) & 0xff;
                if (pos < out_cap) out[pos] = (uint8_t)byte; else ovf = true;
                pos++;
                if (byte == 0xff) {
                  if (pos < out_cap) out[pos] = 0; else ovf = true;
                  pos++;
                }
              }
            }
          }
        }
        if (ovf) ctl[4] = 1;
      }
      __syncthreads();
      if (j == 0) s_ffrun += ffwin;  // read again only after the barriers of the next window / by thread 0 itself
    }
    if (npass == 2 && pass == 0) {  // all windows counted: chain the stuffed-zero counts, then sweep again
      __syncthreads();
      const unsigned agg = s_ffrun;
      __syncthreads();
      chain_publish(ffstatus, cta, agg);
      ffbase = chain_lookback(ffstatus, cta, agg);
      if (j == 0) s_ffrun = 0;
      __syncthreads();
    }
  }
  TRACE(8);
  if (is_last && j == 0) {
    const unsigned total_bits = base + total;
    ctl[0] = total_bits;
    ctl[3] = ((total_bits + 7) >> 3) + ffbase + s_ffrun;
    if (ctl[3] > out_cap) ctl[4] = 1;
  }
#undef TRACE
}

__global__ void __launch_bounds__(kEncThreads, 6) k_huff_encode(const __grid_constant__ HuffFrame f, const uint32_t* __restrict__ books,
                                                             unsigned long long* status, unsigned long long* ffstatus,
                                                             unsigned long long* tails, uint8_t* __restrict__ out,
                                                             unsigned out_cap, unsigned* ctl, unsigned long long* trace) {
  huff_encode_cta<false>(f, books, status, ffstatus, tails, out, out_cap, ctl, trace, nullptr, nullptr, 0);
}

// Every scan of a batch in one launch.  A CTA takes a global ticket and maps it to (scan, CTA of that scan) by a binary
// search over cta_end (each scan's last ticket + 1).  Tickets are issued in order and a scan's CTAs hold consecutive
// tickets, so every predecessor a CTA waits for in its own scan is running or done, as in k_huff_encode; the look-backs
// and the boundary words stay inside the scan's own slices (CTA 0 of a scan starts at bit 0 and looks back at nothing).
// Five CTAs per SM: the scan's pointers come from its descriptor, and at six CTAs' 40 registers they would spill.
__global__ void __launch_bounds__(kEncThreads, 5) k_huff_encode_batch(const HuffScanDesc* __restrict__ scans,
                                                                   const unsigned* __restrict__ cta_end, unsigned nscan,
                                                                   const uint32_t* __restrict__ books, unsigned* ticket) {
  huff_encode_cta<true>(scans[0].f, books, nullptr, nullptr, nullptr, nullptr, 0, ticket, nullptr, scans, cta_end, nscan);
}

static FastDiv fast_div(unsigned d) {
  FastDiv f;
  f.d = d;
  f.m = d <= 1 ? 0u : (unsigned)((0x100000000ull + d - 1) / d);
  return f;
}

// the four standard code books, once per device; nullptr + last error on failure
static const uint32_t* device_books() {
  static PerDevice<const void*> books;
  return (const uint32_t*)device_table(books, 4 * 256 * sizeof(uint32_t), [](void* host) {
    for (int t = 0; t < 4; t++) jpeg_std_codebook(t, (uint32_t*)host + 256 * t);
  });
}

// what jpeg_entropy_dev planned: resident CTAs per wave, launches by bpt (index 1..8), launches beyond one wave
std::atomic<unsigned long long> g_enc_plan[10];

}  // namespace

void jpeg_encode_stats(unsigned long long out[10]) {
  for (int i = 0; i < 10; i++) out[i] = g_enc_plan[i].load(std::memory_order_relaxed);
}

namespace {

// the scan geometry k_huff_encode reads; *nblocks: blocks of the scan, dummy blocks included
void huff_frame(const JpegEncodeJob& job, HuffFrame* out, size_t* nblocks) {
  const JpegFrame& fr = job.frame;
  HuffFrame& f = *out;
  memset(&f, 0, sizeof f);
  f.ncomp = fr.ncomp;
  int k = 0;
  for (int c = 0; c < fr.ncomp; c++) {
    f.slots[c] = reinterpret_cast<const uint32_t*>(job.d_coefs[c]);
    f.meta[c] = job.d_meta[c];
    f.wblocks[c] = fr.comp[c].wblocks;
    f.hblocks[c] = fr.comp[c].hblocks;
    const int mw = fr.ncomp == 1 ? 1 : fr.comp[c].h_samp, mh = fr.ncomp == 1 ? 1 : fr.comp[c].v_samp;
    f.mw[c] = fast_div((unsigned)mw);
    f.per[c] = mw * mh;
    f.koff[c] = k;
    k += mw * mh;
  }
  f.bpm = fast_div((unsigned)k);
  f.mpr = fast_div((unsigned)fr.mcus_per_row);
  f.has_dummy = fr.has_dummy_blocks() ? 1 : 0;
  *nblocks = (size_t)fr.mcus_per_row * fr.mcu_rows * k;  // dummy blocks included
  f.nblocks = (unsigned)*nblocks;
}

// capacity of the entropy-coded segment: the reference's whole output buffer is w*h*6 bytes
// (ultrahdr_api.cpp:1294); a single scan can never need more than that in a valid encode
size_t scan_cap(const JpegFrame& fr) { return ((size_t)fr.width * fr.height * 6 + 4096 + 3) / 4 * 4; }

// blocks per thread: the smallest value for which the whole grid is resident at once
int blocks_per_thread(size_t nblocks, int resident) {
  const int bpt = (int)((nblocks + (size_t)kEncThreads * resident - 1) / ((size_t)kEncThreads * resident));
  return bpt < 1 ? 1 : (bpt > kMaxBpt ? kMaxBpt : bpt);
}

}  // namespace

int jpeg_entropy_dev(Workspace& ws, JpegEncodeJob* job) {
  if (!job->zigzag || !job->d_meta[0])
    return fail(E_ERROR, "internal: device entropy coder needs the zigzag forward stage and its block side information");
  const uint32_t* books = device_books();
  if (!books) return E_ERROR;
  HuffFrame f;
  size_t nblocks = 0;
  huff_frame(*job, &f, &nblocks);
  const size_t cap = scan_cap(job->frame);
  static PerDevice<int> wave;
  const int resident = wave_ctas(wave, (const void*)k_huff_encode, kEncThreads, 0);
  if (!resident) return E_ERROR;
  const int bpt = blocks_per_thread(nblocks, resident);
  f.bpt = bpt;
  const size_t chunk = (size_t)kEncThreads * bpt;
  const unsigned ncta = (unsigned)((nblocks + chunk - 1) / chunk);
  // [ctl 64 B][status ncta x 8][ffstatus ncta x 8][tails ncta x 8], zeroed together
  const size_t ctl_bytes = 64 + (size_t)ncta * 24;
  unsigned* ctl = (unsigned*)ws.dalloc(ctl_bytes);  // [0] total bits [3] out bytes [4] overflow [5] CTA tickets
  job->d_scan = (uint8_t*)ws.dalloc(cap + 64);
  job->h_scan_bytes = (unsigned*)ws.halloc(64);
  if (!ctl || !job->d_scan || !job->h_scan_bytes) return E_MEM;
  unsigned long long* status = reinterpret_cast<unsigned long long*>(ctl + 16);
  unsigned long long* ffstatus = status + ncta;
  unsigned long long* tails = ffstatus + ncta;
  job->d_scan_bytes = ctl + 3;
  job->scan_capacity = cap;
  cudaStream_t st = ws.stream();
  CUDA_TRY(cudaMemsetAsync(ctl, 0, ctl_bytes, st));
  count_launches(1);
  ws.t_begin("huff_encode");
  unsigned long long* trace = nullptr;
  static const bool want_trace = getenv("UHDR_B200_HUFF_TRACE") != nullptr;
  if (want_trace) {  // diagnostic: %globaltimer at the phase boundaries of every CTA, dumped to stderr
    trace = (unsigned long long*)ws.dalloc((size_t)ncta * 16 * 8);
    if (trace) cudaMemsetAsync(trace, 0, (size_t)ncta * 16 * 8, st);
  }
  k_huff_encode<<<ncta, kEncThreads, 0, st>>>(f, books, status, ffstatus, tails, job->d_scan, (unsigned)cap, ctl, trace);
  g_enc_plan[0].store((unsigned long long)resident, std::memory_order_relaxed);
  g_enc_plan[bpt].fetch_add(1, std::memory_order_relaxed);
  if (ncta > (unsigned)resident) g_enc_plan[9].fetch_add(1, std::memory_order_relaxed);
  if (trace) {
    std::vector<unsigned long long> h((size_t)ncta * 16);
    cudaMemcpyAsync(h.data(), trace, h.size() * 8, cudaMemcpyDeviceToHost, st);
    cudaStreamSynchronize(st);
    unsigned long long t0 = ~0ull, t1 = 0;
    for (unsigned c = 0; c < ncta; c++) { if (h[c * 16] && h[c * 16] < t0) t0 = h[c * 16]; if (h[c * 16 + 8] > t1) t1 = h[c * 16 + 8]; }
    double acc[9] = {0};
    for (unsigned c = 0; c < ncta; c++) for (int k = 1; k < 9; k++) acc[k] += (double)(h[c * 16 + k] - h[c * 16 + k - 1]);
    fprintf(stderr, "[huff trace] ncta %u bpt %d span %.1f us; first-start..last-start %.1f us; mean us per phase: phase1 %.2f scan %.2f emit %.2f bits-chain %.2f align+boundary %.2f ffscan %.2f ff-chain %.2f write %.2f\n",
            ncta, bpt, (t1 - t0) / 1e3, 0.0, acc[1] / ncta / 1e3, acc[2] / ncta / 1e3, acc[3] / ncta / 1e3, acc[4] / ncta / 1e3, acc[5] / ncta / 1e3, acc[6] / ncta / 1e3, acc[7] / ncta / 1e3, acc[8] / ncta / 1e3);
    unsigned long long smin = ~0ull, smax = 0;
    for (unsigned c = 0; c < ncta; c++) { if (h[c * 16] < smin) smin = h[c * 16]; if (h[c * 16] > smax) smax = h[c * 16]; }
    fprintf(stderr, "[huff trace] CTA start spread %.1f us; cta0 %.1f..%.1f, last cta %.1f..%.1f (us after first start)\n", (smax - smin) / 1e3,
            (h[0] - smin) / 1e3, (h[8] - smin) / 1e3, (h[(size_t)(ncta - 1) * 16] - smin) / 1e3, (h[(size_t)(ncta - 1) * 16 + 8] - smin) / 1e3);
  }
  ws.t_end();
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(job->h_scan_bytes, ctl, 32, cudaMemcpyDeviceToHost, st));
  return E_OK;
}

int jpeg_scan_check(const JpegEncodeJob& job) {
  if (job.h_scan_bytes[4]) return fail(E_MEM, "entropy-coded segment exceeds the %zu byte device buffer", job.scan_capacity);
  return E_OK;
}

// second phase after the sizes are on the host: fetch exactly the bytes produced
static int jpeg_entropy_fetch(Workspace& ws, JpegEncodeJob* job) {
  int rc = jpeg_scan_check(*job);
  if (rc) return rc;
  const unsigned n = job->h_scan_bytes[3];
  job->h_scan = (uint8_t*)ws.halloc(n + 64);
  if (!job->h_scan) return E_MEM;
  CUDA_TRY(cudaMemcpyAsync(job->h_scan, job->d_scan, n, cudaMemcpyDeviceToHost, ws.stream()));
  return E_OK;
}

int jpeg_entropy_collect(Workspace& ws, JpegEncodeJob* const* jobs, int n) {
  int rc = ws.sync();   // the scans' sizes
  for (int i = 0; !rc && i < n; i++) rc = jpeg_entropy_fetch(ws, jobs[i]);
  return rc ? rc : ws.sync();
}

namespace {

std::atomic<unsigned long long> g_enc_batch[2];   // k_huff_encode_batch launches, scans they coded

// one scan's bytes [0, n) for k_pack_scans, to offset `off` (a multiple of 16) of the packed buffer
struct PackSeg {
  const uint8_t* src;
  unsigned long long off;
  unsigned n, pad;
};
constexpr unsigned kPackBytes = kEncThreads * 16;   // bytes per CTA

// the entropy-coded segments of a batch, gathered into one buffer: a CTA copies 4 KiB of one segment, 16 bytes a thread
// (a segment's buffer has 64 spare bytes, so the last 16-byte word may read past its end)
__global__ void __launch_bounds__(kEncThreads) k_pack_scans(const PackSeg* __restrict__ segs, const unsigned* __restrict__ cta_end,
                                                        unsigned nseg, uint8_t* __restrict__ dst) {
  const unsigned si = batch_find(cta_end, nseg, blockIdx.x);
  const PackSeg s = segs[si];
  const unsigned o = (blockIdx.x - (si ? cta_end[si - 1] : 0u)) * kPackBytes + threadIdx.x * 16;
  if (o < s.n) *reinterpret_cast<uint4*>(dst + s.off + o) = __ldg(reinterpret_cast<const uint4*>(s.src + o));
}

size_t round_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace

void jpeg_encode_batch_stats(unsigned long long out[2]) {
  for (int i = 0; i < 2; i++) out[i] = g_enc_batch[i].load(std::memory_order_relaxed);
}

int jpeg_entropy_batch_dev(Workspace& ws, JpegEncodeJob* const* jobs, int n) {
  for (int i = 0; i < n; i++)
    if (!jobs[i]->zigzag || !jobs[i]->d_meta[0])
      return fail(E_ERROR, "internal: device entropy coder needs the zigzag forward stage and its block side information");
  const uint32_t* books = device_books();
  if (!books) return E_ERROR;
  static PerDevice<int> wave;
  const int resident = wave_ctas(wave, (const void*)k_huff_encode_batch, kEncThreads, 0);
  if (!resident) return E_ERROR;
  HuffScanDesc* h_desc = (HuffScanDesc*)ws.halloc(sizeof(HuffScanDesc) * n);
  unsigned* h_end = (unsigned*)ws.halloc(sizeof(unsigned) * n);
  unsigned* h_ctl = (unsigned*)ws.halloc((size_t)64 * n);
  if (!h_desc || !h_end || !h_ctl) return E_MEM;
  size_t total = 0;
  for (int i = 0; i < n; i++) {
    memset(&h_desc[i], 0, sizeof h_desc[i]);
    size_t nb = 0;
    huff_frame(*jobs[i], &h_desc[i].f, &nb);
    total += nb;
  }
  // one chunk size for the group: the existing rule over all its blocks
  const int bpt = blocks_per_thread(total, resident);
  const size_t chunk = (size_t)kEncThreads * bpt;
  unsigned ctas = 0;
  size_t scan_bytes = 0;
  for (int i = 0; i < n; i++) {
    h_desc[i].f.bpt = bpt;
    ctas += (unsigned)((h_desc[i].f.nblocks + chunk - 1) / chunk);
    h_end[i] = ctas;
    scan_bytes += round_up(scan_cap(jobs[i]->frame) + 64, 256);
  }
  // [ticket, 64 B][ctl 64 B per scan][status, ffstatus, tails: 8 B per CTA each], zeroed together
  const size_t ctl_bytes = 64 + (size_t)64 * n + (size_t)24 * ctas;
  unsigned* ctl = (unsigned*)ws.dalloc(ctl_bytes);
  uint8_t* scan = (uint8_t*)ws.dalloc(scan_bytes);
  HuffScanDesc* d_desc = (HuffScanDesc*)ws.dalloc(sizeof(HuffScanDesc) * n);
  unsigned* d_end = (unsigned*)ws.dalloc(sizeof(unsigned) * n);
  if (!ctl || !scan || !d_desc || !d_end) return E_MEM;
  unsigned long long* look = reinterpret_cast<unsigned long long*>(ctl + 16 + 16 * (size_t)n);
  unsigned c0 = 0;
  for (int i = 0; i < n; i++) {
    JpegEncodeJob& job = *jobs[i];
    HuffScanDesc& d = h_desc[i];
    const unsigned nc = h_end[i] - c0;
    d.status = look + c0;
    d.ffstatus = look + ctas + c0;
    d.tails = look + 2 * (size_t)ctas + c0;
    d.ctl = ctl + 16 * (size_t)(i + 1);
    job.scan_capacity = scan_cap(job.frame);
    d.out = job.d_scan = scan;
    d.out_cap = (unsigned)job.scan_capacity;
    job.d_scan_bytes = d.ctl + 3;
    job.h_scan_bytes = h_ctl + 16 * (size_t)i;
    job.h_scan = nullptr;
    scan += round_up(job.scan_capacity + 64, 256);
    c0 += nc;
  }
  cudaStream_t st = ws.stream();
  CUDA_TRY(cudaMemsetAsync(ctl, 0, ctl_bytes, st));
  CUDA_TRY(cudaMemcpyAsync(d_desc, h_desc, sizeof(HuffScanDesc) * n, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(d_end, h_end, sizeof(unsigned) * n, cudaMemcpyHostToDevice, st));
  count_launches(1);
  ws.t_begin("huff_encode_batch");
  k_huff_encode_batch<<<ctas, kEncThreads, 0, st>>>(d_desc, d_end, (unsigned)n, books, ctl);
  ws.t_end();
  CUDA_TRY(cudaGetLastError());
  g_enc_batch[0].fetch_add(1, std::memory_order_relaxed);
  g_enc_batch[1].fetch_add((unsigned long long)n, std::memory_order_relaxed);
  // every scan's control words in one copy
  CUDA_TRY(cudaMemcpyAsync(h_ctl, ctl + 16, (size_t)64 * n, cudaMemcpyDeviceToHost, st));
  return E_OK;
}

int jpeg_entropy_batch_fetch(Workspace& ws, JpegEncodeJob* const* jobs, int n) {
  PackSeg* h_seg = (PackSeg*)ws.halloc(sizeof(PackSeg) * n);
  unsigned* h_end = (unsigned*)ws.halloc(sizeof(unsigned) * n);
  if (!h_seg || !h_end) return E_MEM;
  size_t total = 0;
  unsigned ctas = 0;
  for (int i = 0; i < n; i++) {
    const unsigned* c = jobs[i]->h_scan_bytes;
    const unsigned nb = c[4] ? 0u : c[3];   // an overflowing scan is not fetched
    h_seg[i] = PackSeg{jobs[i]->d_scan, (unsigned long long)total, nb, 0};
    total += round_up(nb, 16);
    ctas += (nb + kPackBytes - 1) / kPackBytes;
    h_end[i] = ctas;
  }
  uint8_t* h_pack = (uint8_t*)ws.halloc(total + 64);
  if (!h_pack) return E_MEM;
  for (int i = 0; i < n; i++) jobs[i]->h_scan = jobs[i]->h_scan_bytes[4] ? nullptr : h_pack + h_seg[i].off;
  if (!ctas) return E_OK;
  PackSeg* d_seg = (PackSeg*)ws.dalloc(sizeof(PackSeg) * n);
  unsigned* d_end = (unsigned*)ws.dalloc(sizeof(unsigned) * n);
  uint8_t* d_pack = (uint8_t*)ws.dalloc(total + 64);
  if (!d_seg || !d_end || !d_pack) return E_MEM;
  cudaStream_t st = ws.stream();
  CUDA_TRY(cudaMemcpyAsync(d_seg, h_seg, sizeof(PackSeg) * n, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(d_end, h_end, sizeof(unsigned) * n, cudaMemcpyHostToDevice, st));
  count_launches(1);
  ws.t_begin("pack_scans");
  k_pack_scans<<<ctas, kEncThreads, 0, st>>>(d_seg, d_end, (unsigned)n, d_pack);
  ws.t_end();
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(h_pack, d_pack, total, cudaMemcpyDeviceToHost, st));
  return E_OK;
}

}  // namespace uhdr_b200
