// Baseline-JPEG entropy *decoding* on the device: the serial half of JpegDecoderHelper
// (jpegdecoderhelper.cpp:397-411 -> libjpeg-turbo jdhuff.c decode_mcu) restated as a
// data-parallel fixed-point iteration.
//
// A Huffman-coded scan has no block index: a decoder must know where the previous symbol ended.
// But a decoder started at a wrong place falls into step with the true symbol sequence after a
// few blocks (codes self-synchronise; an end-of-block resets the coefficient index; a wrong
// position inside the MCU meets the wrong table at the next luma/chroma change and is knocked
// out of step again until it lands on the right one).  So:
//   1. the host removes the FF00 stuffing while staging the scan in pinned memory
//   2. the scan is cut into restart intervals (the whole scan is one interval without a DRI
//      marker), and each interval into subsequences of at most kSeqBits bits, one thread each.
//      out[i] is the decoder state (bit position, coefficient index, block-in-MCU) at which
//      subsequence i+1 starts.  Every round each thread re-decodes its subsequence from out[i-1]
//      and replaces out[i]; the first subsequence of an interval always starts from the true
//      state (byte-aligned, DC symbol next, block 0 of an MCU), so the true states spread from
//      there at least one subsequence per round -- and in practice in a few rounds, because most
//      exit states are already right.  A round that changes nothing is a fixed point, and the
//      only fixed point is the sequential decoder's state sequence (induction over i).  When no
//      interval spans more than one subsequence every entry state is known and no round runs.
//   3. the per-subsequence block counts are prefix-summed, and a last pass decodes once more,
//      now writing coefficients ([block][64], natural order) and DC differences.  Interval k
//      owns blocks [k * Ri * bpm, (k + 1) * Ri * bpm): the up to 7 one-bits of padding before a
//      restart marker may decode as part of a symbol, so blocks past that quota are dropped, and
//      the counts of earlier intervals never move a later interval's blocks.
//   4. DC prediction (a running sum per component over the scan order, dummy edge blocks
//      included like jdhuff.c, restarting at every interval) is a prefix sum + scatter.
// Streams whose restart markers are irregular (see unstuff_scan), that do not reach a fixed point
// in kMaxRounds rounds, or whose intervals do not decode to exactly their quota of blocks return
// kHuffDecFallback and the caller uses the host decoder of jpeg_host.cpp.
#include <atomic>
#include <mutex>
#include <climits>
#include <cstring>

#include "jpeg.h"
#include "runtime.h"

namespace uhdr_b200 {

__constant__ uint8_t kZigzagDev[64];  // zigzag position -> natural index (copy of kZigzag)

namespace {

constexpr int kSeqBits = 1024;
constexpr int kLutBits = 9;
constexpr int kRoundsPerBatch = 16;  // settled rounds cost ~a launch each (CTAs without work exit at once): one host check usually suffices
constexpr int kMaxRounds = 512;

struct HdTables {  // 0 DC table 0, 1 DC table 1, 2 AC table 0, 3 AC table 1
  uint16_t lut[4][1 << kLutBits];  // (len << 8) | symbol; 0 = code longer than kLutBits bits
  int maxcode[4][18];              // canonical decode of the long codes; [17] = INT_MAX
  int valoff[4][17];               // index of a code's symbol = valoff[len] + code
  uint8_t vals[4][256];
};
struct HdFrame {
  int bpm;                       // blocks per MCU
  int comp_of[10], bi[10], bj[10], kin[10];  // per MCU position: component, block offset, index within component
  int dc_tab[3], ac_tab[3];      // indices into HdTables
  int h[3], v[3], hv[3], wblocks[3], hblocks[3];
  int mcus_per_row;
  unsigned total_bits, nseq, total_blocks;
  unsigned iv_blocks;            // blocks per restart interval (all of them without a DRI marker)
};
struct HdShared {
  HdTables t;
  HdFrame f;
};

__device__ __forceinline__ unsigned peek32(const uint32_t* __restrict__ bits, unsigned p) {
  const unsigned k = p >> 5;
  const uint32_t w0 = __byte_perm(__ldg(bits + k), 0, 0x0123), w1 = __byte_perm(__ldg(bits + k + 1), 0, 0x0123);
  return __funnelshift_l(w1, w0, p & 31);
}
__device__ __forceinline__ int extend(unsigned v, unsigned s) {  // jdhuff.c HUFF_EXTEND
  return v < (1u << (s - 1)) ? (int)v - (int)(1u << s) + 1 : (int)v;
}

struct HdOut {  // WRITE pass destinations
  int16_t* coefs[3];
  int* dcd[3];
  unsigned* err;
};

// Subsequence layout (k_hd_layout): subsequence i covers clean bits [lo[i], lo[i + 1]) of restart
// interval iv[i]; interval k is subsequences [first[k], first[k + 1]).
struct HdSeqs {
  const unsigned* lo;     // nseq + 1 entries, lo[nseq] = total_bits
  const unsigned* iv;     // nseq
  const unsigned* first;  // intervals + 1, first[intervals] = nseq
};

// Decodes the symbols that start in [p, end_bit).  State in/out: p, z (0 = DC symbol next), c.
// WRITE: b is the index of the block being decoded; blocks from b_end on (what the padding before a
// restart marker and the next interval's first bits decode to) are neither stored nor checked, and
// the block that reaches b_end must have ended by bit p_end.
template <bool WRITE>
__device__ __forceinline__ unsigned decode_seq(const HdShared& S, const uint32_t* __restrict__ bits, unsigned& p, unsigned& z,
                                               unsigned& c, const unsigned end_bit, unsigned b, const unsigned b_end,
                                               const unsigned p_end, const HdOut& o) {
  const HdFrame& f = S.f;
  unsigned nblk = 0;
  int16_t* blk = nullptr;
  unsigned mcu = 0;
  auto locate = [&]() {  // block b at MCU position c -> coefficient block (or nullptr for dummy / surplus blocks)
    const int comp = f.comp_of[c];
    const unsigned mx = mcu % (unsigned)f.mcus_per_row, my = mcu / (unsigned)f.mcus_per_row;
    const int bx = (int)mx * f.h[comp] + f.bi[c], by = (int)my * f.v[comp] + f.bj[c];
    blk = (b < b_end && bx < f.wblocks[comp] && by < f.hblocks[comp]) ? o.coefs[comp] + ((size_t)by * f.wblocks[comp] + bx) * 64 : nullptr;
  };
  if (WRITE) {
    mcu = b / (unsigned)f.bpm;
    locate();
  }
  while (p < end_bit) {
    const unsigned w = peek32(bits, p);
    const int comp = f.comp_of[c];
    const int t = z == 0 ? f.dc_tab[comp] : f.ac_tab[comp];
    const unsigned e = S.t.lut[t][w >> (32 - kLutBits)];
    unsigned len = e >> 8, sym = e & 0xff;
    if (len == 0) {  // long code: canonical search, like jdhuff.c's slow path
      len = kLutBits + 1;
      int code = (int)(w >> (32 - len));
      while (code > S.t.maxcode[t][len]) {
        len++;
        code = (int)(w >> (32 - len));
      }
      if (len > 16) {  // not a code of this table (possible only while out of step, past the quota, or corrupt data)
        len = 16;
        sym = 0;
        if (WRITE && b < b_end) *o.err = 1;
      } else {
        sym = S.t.vals[t][(S.t.valoff[t][len] + code) & 255];
      }
    }
    const unsigned s = sym & 15;
    const unsigned v = s ? (w << len) >> (32 - s) : 0;
    p += len + s;
    if (z == 0) {
      if (WRITE && b < b_end) o.dcd[comp][(size_t)mcu * f.hv[comp] + f.kin[c]] = s ? extend(v, s) : 0;
      z = 1;
    } else {
      const unsigned r = sym >> 4;
      if (s) {
        z += r;
        if (WRITE) {
          if (z > 63) {
            if (b < b_end) *o.err = 1;
          } else if (blk) {
            blk[kZigzagDev[z]] = (int16_t)extend(v, s);
          }
        }
        z++;
      } else {
        z = r == 15 ? z + 16 : 64;
      }
    }
    if (z >= 64) {
      z = 0;
      nblk++;
      c = c + 1 == (unsigned)f.bpm ? 0 : c + 1;
      if (WRITE) {
        b++;
        if (b == b_end && p > p_end) *o.err = 1;  // the interval's last block reads into the next interval
        if (c == 0) mcu++;
        locate();
      }
    }
  }
  return nblk;
}

__device__ __forceinline__ void stage_shared(HdShared& S, const HdShared* __restrict__ g) {
  const uint32_t* src = reinterpret_cast<const uint32_t*>(g);
  uint32_t* dst = reinterpret_cast<uint32_t*>(&S);
  for (unsigned i = threadIdx.x; i < sizeof(HdShared) / 4; i += blockDim.x) dst[i] = __ldg(src + i);
  __syncthreads();
}

// one relaxation round, in place (64-bit states are read and written atomically)
__global__ void __launch_bounds__(128) k_hd_sync(const uint32_t* __restrict__ bits, unsigned long long* out, unsigned long long* used, unsigned* cnt,
                                                 unsigned* changed, const HdShared* __restrict__ gs, const HdSeqs q) {
  __shared__ HdShared S;
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned nseq = gs->f.nseq;
  // state word: bit position | (z | c << 8) << 32; an interval's first subsequence starts at its true state
  const unsigned long long entry = i >= nseq ? 0ull
                                   : q.first[q.iv[i]] == i ? (unsigned long long)q.lo[i]
                                                           : *reinterpret_cast<volatile unsigned long long*>(out + i - 1);
  const bool todo = i < nseq && entry != used[i];  // same start as last time: same result
  // after the second round nearly every subsequence is settled: a CTA without work leaves before it
  // stages the 6 KB of tables, so the later rounds cost little more than their launch
  if (!__syncthreads_or(todo ? 1 : 0)) return;
  stage_shared(S, gs);
  if (!todo) return;
  unsigned p = (unsigned)entry, z = (unsigned)(entry >> 32) & 0xff, c = (unsigned)(entry >> 40);
  const HdOut none = {};
  const unsigned n = decode_seq<false>(S, bits, p, z, c, q.lo[i + 1], 0, 0, 0, none);
  const unsigned long long now = (unsigned long long)p | ((unsigned long long)(z | (c << 8)) << 32);
  used[i] = entry;
  cnt[i] = n;
  if (now != out[i]) {
    *reinterpret_cast<volatile unsigned long long*>(out + i) = now;
    *changed = 1;
  }
}

// expands the per-interval layout built on the host (start bit and first subsequence of each interval)
// into the per-subsequence one
__global__ void k_hd_layout(const unsigned* __restrict__ start, const unsigned* __restrict__ first, unsigned nint, unsigned nseq,
                            unsigned total_bits, unsigned* lo, unsigned* iv) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) lo[nseq] = total_bits;
  if (i >= nseq) return;
  unsigned a = 0, b = nint - 1;  // last interval whose first subsequence is <= i
  while (a < b) {
    const unsigned m = (a + b + 1) / 2;
    if (first[m] <= i) a = m;
    else b = m - 1;
  }
  lo[i] = start[a] + (i - first[a]) * (unsigned)kSeqBits;
  iv[i] = a;
}

__global__ void k_hd_init(unsigned long long* out, unsigned long long* used, unsigned* cnt, unsigned nseq, const unsigned* __restrict__ lo) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nseq) return;
  out[i] = (unsigned long long)lo[i + 1];
  used[i] = ~0ull;
  cnt[i] = 0;
}

// exclusive prefix sum of cnt (one CTA; nseq is at most a few hundred thousand)
__global__ void __launch_bounds__(1024) k_hd_scan(const unsigned* __restrict__ cnt, unsigned* __restrict__ base, unsigned n) {
  __shared__ unsigned warp_sums[32];
  __shared__ unsigned carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (unsigned start = 0; start < n; start += 1024) {
    const unsigned i = start + threadIdx.x;
    const unsigned v = i < n ? cnt[i] : 0;
    unsigned x = v;
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned y = __shfl_up_sync(0xffffffffu, x, o);
      if ((threadIdx.x & 31) >= o) x += y;
    }
    if ((threadIdx.x & 31) == 31) warp_sums[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
      unsigned s = warp_sums[threadIdx.x];
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned y = __shfl_up_sync(0xffffffffu, s, o);
        if (threadIdx.x >= o) s += y;
      }
      warp_sums[threadIdx.x] = s;
    }
    __syncthreads();
    const unsigned wbase = (threadIdx.x >> 5) ? warp_sums[(threadIdx.x >> 5) - 1] : 0;
    if (i < n) base[i] = carry + wbase + x - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry += wbase + x;
    __syncthreads();
  }
}

// out and base are read only for subsequences that do not start an interval
__global__ void __launch_bounds__(128) k_hd_write(const uint32_t* __restrict__ bits, const unsigned long long* __restrict__ out, const unsigned* __restrict__ base,
                                                  const HdShared* __restrict__ gs, const HdSeqs q, HdOut o) {
  __shared__ HdShared S;
  stage_shared(S, gs);
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= S.f.nseq) return;
  const unsigned k = q.iv[i], head = q.first[k], next = q.first[k + 1];
  const unsigned long long entry = head == i ? (unsigned long long)q.lo[i] : out[i - 1];
  unsigned p = (unsigned)entry, z = (unsigned)(entry >> 32) & 0xff, c = (unsigned)(entry >> 40);
  const unsigned b0 = k * S.f.iv_blocks;
  const unsigned b = b0 + (head == i ? 0u : base[i] - base[head]);
  const unsigned b_end = min(b0 + S.f.iv_blocks, S.f.total_blocks);
  if (b % (unsigned)S.f.bpm != c) *o.err = 2;  // the states and the block counts must agree
  const unsigned n = decode_seq<true>(S, bits, p, z, c, q.lo[i + 1], b, b_end, q.lo[next], o);
  if (next == i + 1 && b + n < b_end) *o.err = 1;  // the interval holds fewer blocks than it must
}

// ---- DC prediction: inclusive scan of the differences per component, scatter into the blocks ----
struct DcPlan {
  int* dcd;
  int16_t* coefs;
  unsigned n;  // blocks of this component in scan order (dummy blocks included)
  unsigned seg;  // blocks of this component per restart interval: the prediction restarts from 0 at multiples of seg
  int h, v, hv, wblocks, hblocks, mcus_per_row;
  int* sums;   // per-CTA totals
};
constexpr int kDcCta = 1024;
__device__ __forceinline__ int cta_inclusive_scan(int v, int* warp_sums /* [32] */) {
  int x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if ((threadIdx.x & 31) >= o) x += y;
  }
  if ((threadIdx.x & 31) == 31) warp_sums[threadIdx.x >> 5] = x;
  __syncthreads();
  if (threadIdx.x < 32) {
    int s = warp_sums[threadIdx.x];
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, o);
      if (threadIdx.x >= o) s += y;
    }
    warp_sums[threadIdx.x] = s;
  }
  __syncthreads();
  return x + ((threadIdx.x >> 5) ? warp_sums[(threadIdx.x >> 5) - 1] : 0);
}
__global__ void __launch_bounds__(kDcCta) k_dc_local(DcPlan d) {
  __shared__ int ws[32];
  const unsigned i = blockIdx.x * kDcCta + threadIdx.x;
  const int x = cta_inclusive_scan(i < d.n ? d.dcd[i] : 0, ws);
  if (i < d.n) d.dcd[i] = x;
  if (threadIdx.x == kDcCta - 1) d.sums[blockIdx.x] = x;
}
__global__ void __launch_bounds__(kDcCta) k_dc_sums(int* sums, unsigned n) {  // in place, exclusive, one CTA
  __shared__ int ws[32];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (unsigned start = 0; start < n; start += kDcCta) {
    const unsigned i = start + threadIdx.x;
    const int v = i < n ? sums[i] : 0;
    const int x = cta_inclusive_scan(v, ws);
    if (i < n) sums[i] = carry + x - v;
    __syncthreads();
    if (threadIdx.x == kDcCta - 1) carry += x;
    __syncthreads();
  }
}
__global__ void __launch_bounds__(256) k_dc_apply(DcPlan d) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= d.n) return;
  // running sum within the interval = prefix sum to i minus prefix sum before the interval's first block;
  // exact in wrapping 32-bit arithmetic, which is how jpeg_host_decode_coefs accumulates too
  const unsigned s = i - i % d.seg;
  unsigned dc = (unsigned)d.dcd[i] + (unsigned)d.sums[i / kDcCta];
  if (s) dc -= (unsigned)d.dcd[s - 1] + (unsigned)d.sums[(s - 1) / kDcCta];
  const unsigned mcu = i / (unsigned)d.hv, k = i % (unsigned)d.hv;
  const int bx = (int)(mcu % (unsigned)d.mcus_per_row) * d.h + (int)(k % (unsigned)d.h);
  const int by = (int)(mcu / (unsigned)d.mcus_per_row) * d.v + (int)(k / (unsigned)d.h);
  if (bx < d.wblocks && by < d.hblocks) d.coefs[((size_t)by * d.wblocks + bx) * 64] = (int16_t)dc;
}

void build_tables(const JpegHeader& h, HdTables* t) {
  memset(t, 0, sizeof *t);
  for (int cls = 0; cls < 2; cls++)
    for (int id = 0; id < 2; id++) {
      const int ti = cls * 2 + id;
      for (int l = 0; l < 18; l++) t->maxcode[ti][l] = -1;
      t->maxcode[ti][17] = INT_MAX;
      if (!h.have_tbl[cls][id]) {  // absent table: every lookup is a 16-bit "invalid" (never selected by a valid header)
        for (int l = 0; l < 17; l++) t->maxcode[ti][l] = -1;
        continue;
      }
      const uint8_t* bits = h.bits[cls][id];
      memcpy(t->vals[ti], h.vals[cls][id], 256);
      int code = 0, k = 0;
      for (int len = 1; len <= 16; len++) {
        t->valoff[ti][len] = k - code;
        for (int i = 0; i < bits[len]; i++, k++, code++)
          if (len <= kLutBits && code < (1 << len))  // guard: never index past `lut` whatever the lengths say
            for (int r = 0; r < (1 << (kLutBits - len)); r++)
              t->lut[ti][(code << (kLutBits - len)) | r] = (uint16_t)((len << 8) | h.vals[cls][id][k & 255]);
        t->maxcode[ti][len] = bits[len] ? code - 1 : -1;
        code <<= 1;
      }
    }
}

}  // namespace

namespace {
std::atomic<unsigned long long> g_hd_done{0}, g_hd_declined{0}, g_hd_rounds{0};
int declined() {
  g_hd_declined.fetch_add(1);
  return kHuffDecFallback;
}
}  // namespace
void jpeg_entropy_decoder_stats(unsigned long long out[3]) {
  out[0] = g_hd_done.load();
  out[1] = g_hd_declined.load();
  out[2] = g_hd_rounds.load();
}

// Removes byte stuffing from the entropy-coded segment that starts at data[from] and records in
// starts[k] the clean byte offset at which restart interval k begins.  Returns the clean length, or
// -1 unless the segment is regular: exactly nint - 1 restart markers, RST0, RST1, ... modulo 8 in
// that order, and (with a DRI marker) nothing but EOI or the end of the data after the last interval.
static long unstuff_scan(const uint8_t* data, size_t size, size_t from, uint8_t* dst, bool dri, unsigned* starts, unsigned nint) {
  size_t p = from;
  uint8_t* o = dst;
  unsigned k = 1;  // intervals seen
  starts[0] = 0;
  while (p < size) {
    const uint8_t* ff = (const uint8_t*)memchr(data + p, 0xFF, size - p);
    const size_t run = ff ? (size_t)(ff - (data + p)) : size - p;
    memcpy(o, data + p, run);
    o += run;
    p += run;
    if (!ff) break;
    if (p + 1 >= size) break;  // FF at the very end: treat as end of data
    const uint8_t nx = data[p + 1];
    if (nx == 0x00) {
      *o++ = 0xFF;
      p += 2;
    } else if (nx == 0xFF) {
      p += 1;  // fill byte before a marker
    } else if (nx >= 0xD0 && nx <= 0xD7) {
      if (!dri || k == nint || nx != 0xD0 + ((k - 1) & 7)) return -1;
      starts[k++] = (unsigned)(o - dst);
      p += 2;
    } else {
      if (dri && nx != 0xD9) return -1;
      break;  // EOI or any other marker ends the segment
    }
  }
  return k == nint ? (long)(o - dst) : -1;
}

int jpeg_entropy_decode_dev(Workspace& ws, const uint8_t* data, size_t size, const JpegHeader& h, int16_t* d_coefs[3]) {
  const JpegFrame& f = h.frame;
  HdShared hs;
  memset(&hs, 0, sizeof hs);
  HdFrame& hf = hs.f;
  int bpm = 0;
  for (int c = 0; c < f.ncomp; c++) {
    const JpegComp& k = f.comp[c];
    const int mw = f.ncomp == 1 ? 1 : k.h_samp, mh = f.ncomp == 1 ? 1 : k.v_samp;
    hf.h[c] = mw;
    hf.v[c] = mh;
    hf.hv[c] = mw * mh;
    hf.wblocks[c] = k.wblocks;
    hf.hblocks[c] = k.hblocks;
    if (h.dc_sel[c] < 0 || h.dc_sel[c] > 1 || h.ac_sel[c] < 0 || h.ac_sel[c] > 1) return declined();
    if (!h.have_tbl[0][h.dc_sel[c]] || !h.have_tbl[1][h.ac_sel[c]]) return declined();
    hf.dc_tab[c] = h.dc_sel[c];
    hf.ac_tab[c] = 2 + h.ac_sel[c];
    for (int j = 0; j < mh; j++)
      for (int i = 0; i < mw; i++) {
        if (bpm >= 10) return declined();
        hf.comp_of[bpm] = c;
        hf.bi[bpm] = i;
        hf.bj[bpm] = j;
        hf.kin[bpm] = j * mw + i;
        bpm++;
      }
  }
  hf.bpm = bpm;
  hf.mcus_per_row = f.mcus_per_row;
  const size_t mcus = (size_t)f.mcus_per_row * f.mcu_rows;
  if (mcus * bpm > 0xfffffff0u) return declined();
  hf.total_blocks = (unsigned)(mcus * bpm);
  // restart intervals: Ri MCUs each, the last one possibly shorter; no DRI marker = one interval
  const size_t ri = h.restart_interval && (size_t)h.restart_interval < mcus ? (size_t)h.restart_interval : mcus;
  if (ri == 0) return declined();
  const unsigned nint = (unsigned)((mcus + ri - 1) / ri);
  hf.iv_blocks = (unsigned)(ri * bpm);
  build_tables(h, &hs.t);

  // 1. clean bit stream in pinned memory, then on the device (8 zero bytes of slack for the reader)
  if (size <= h.scan_offset) return fail(E_ERROR, "Corrupt JPEG data: no entropy-coded segment");
  const size_t cap = size - h.scan_offset + 16;
  uint8_t* h_bits = (uint8_t*)ws.halloc(cap);
  unsigned* h_starts = (unsigned*)ws.halloc(sizeof(unsigned) * nint);
  if (!h_bits || !h_starts) return E_MEM;
  PhaseTrace tr;
  const long clean = unstuff_scan(data, size, h.scan_offset, h_bits, h.restart_interval != 0, h_starts, nint);
  tr.mark("  unstuff");
  if (clean < 0) return declined();
  if ((size_t)clean * 8 > 0xfffffff0u - kSeqBits) return declined();
  memset(h_bits + clean, 0, 16);
  const size_t padded = ((size_t)clean + 16 + 3) & ~(size_t)3;
  hf.total_bits = (unsigned)(clean * 8);
  if (hf.total_bits == 0) return fail(E_ERROR, "Corrupt JPEG data: empty entropy-coded segment");

  // subsequences: every interval is cut into pieces of at most kSeqBits bits (an empty interval
  // gets one empty piece, whose missing blocks the writing pass reports).  The host numbers them per
  // interval; k_hd_layout expands that on the device.
  unsigned* h_first = (unsigned*)ws.halloc(sizeof(unsigned) * (nint + 1));
  if (!h_first) return E_MEM;
  size_t nseq_total = 0;
  for (unsigned k = 0; k < nint; k++) {
    const unsigned lo = h_starts[k] * 8u, hi = k + 1 < nint ? h_starts[k + 1] * 8u : hf.total_bits;
    h_starts[k] = lo;
    h_first[k] = (unsigned)nseq_total;
    nseq_total += hi > lo ? (hi - lo + kSeqBits - 1) / kSeqBits : 1;
  }
  const unsigned nseq = (unsigned)nseq_total;
  h_first[nint] = nseq;
  hf.nseq = nseq;
  tr.mark("  interval layout");

  uint32_t* d_bits = (uint32_t*)ws.dalloc(padded);
  HdShared* d_hs = (HdShared*)ws.dalloc(sizeof(HdShared));
  HdShared* h_hs = (HdShared*)ws.halloc(sizeof(HdShared));
  unsigned long long* d_out = (unsigned long long*)ws.dalloc(sizeof(unsigned long long) * nseq);
  unsigned long long* d_used = (unsigned long long*)ws.dalloc(sizeof(unsigned long long) * nseq);
  unsigned* d_cnt = (unsigned*)ws.dalloc(sizeof(unsigned) * nseq);
  unsigned* d_base = (unsigned*)ws.dalloc(sizeof(unsigned) * nseq);
  unsigned* d_flags = (unsigned*)ws.dalloc(sizeof(unsigned) * (kMaxRounds + 8));
  unsigned* h_flags = (unsigned*)ws.halloc(sizeof(unsigned) * (kMaxRounds + 8));
  unsigned* d_start = (unsigned*)ws.dalloc(sizeof(unsigned) * nint);
  unsigned* d_first = (unsigned*)ws.dalloc(sizeof(unsigned) * (nint + 1));
  unsigned* d_lo = (unsigned*)ws.dalloc(sizeof(unsigned) * (nseq + 1));
  unsigned* d_iv = (unsigned*)ws.dalloc(sizeof(unsigned) * nseq);
  if (!d_bits || !d_hs || !h_hs || !d_out || !d_used || !d_cnt || !d_base || !d_flags || !h_flags || !d_start || !d_first || !d_lo || !d_iv)
    return E_MEM;
  const HdSeqs q = {d_lo, d_iv, d_first};
  memcpy(h_hs, &hs, sizeof hs);
  cudaStream_t s = ws.stream();
  CUDA_TRY(cudaMemcpyAsync(d_bits, h_bits, padded, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_hs, h_hs, sizeof hs, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_start, h_starts, sizeof(unsigned) * nint, cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(d_first, h_first, sizeof(unsigned) * (nint + 1), cudaMemcpyHostToDevice, s));
  k_hd_layout<<<(nseq + 255) / 256, 256, 0, s>>>(d_start, d_first, nint, nseq, hf.total_bits, d_lo, d_iv);
  count_launches(1);
  CUDA_TRY(cudaMemsetAsync(d_flags, 0, sizeof(unsigned) * (kMaxRounds + 8), s));
  {  // once per device, synchronously and under a lock: decodes run concurrently on several streams / threads
    static std::mutex zig_mu;
    static bool zig_done[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> lk(zig_mu);
    if (dev < 0 || dev >= 64 || !zig_done[dev]) {
      void* zig = nullptr;
      CUDA_TRY(cudaGetSymbolAddress(&zig, kZigzagDev));
      if (int rc = copy_sync(zig, kZigzag, 64, cudaMemcpyHostToDevice)) return rc;
      if (dev >= 0 && dev < 64) zig_done[dev] = true;
    }
  }
  // coefficient blocks start as zeros; only non-zero coefficients are written
  int* d_dcd[3] = {nullptr, nullptr, nullptr};
  for (int c = 0; c < f.ncomp; c++) {
    d_coefs[c] = (int16_t*)ws.dalloc(f.blocks(c) * 128);
    d_dcd[c] = (int*)ws.dalloc(sizeof(int) * mcus * hf.hv[c]);
    if (!d_coefs[c] || !d_dcd[c]) return E_MEM;
    CUDA_TRY(cudaMemsetAsync(d_coefs[c], 0, f.blocks(c) * 128, s));
  }

  // 2. relaxation rounds until one of them changes nothing; none when every subsequence starts an
  // interval, since all entry states are then known
  const unsigned grid = (nseq + 127) / 128;
  const bool relax = nseq > nint;
  int rounds = 0, first_quiet = 0;
  if (relax) {
    ws.t_begin("huffdec_sync");
    k_hd_init<<<(nseq + 255) / 256, 256, 0, s>>>(d_out, d_used, d_cnt, nseq, q.lo);
    count_launches(1);
    bool converged = false;
    while (!converged && rounds < kMaxRounds) {
      count_launches(kRoundsPerBatch);
      for (int r = 0; r < kRoundsPerBatch; r++) k_hd_sync<<<grid, 128, 0, s>>>(d_bits, d_out, d_used, d_cnt, d_flags + rounds + r, d_hs, q);
      CUDA_TRY(cudaGetLastError());
      CUDA_TRY(cudaMemcpyAsync(h_flags + rounds, d_flags + rounds, sizeof(unsigned) * kRoundsPerBatch, cudaMemcpyDeviceToHost, s));
      CUDA_TRY(cudaStreamSynchronize(s));
      for (int r = 0; r < kRoundsPerBatch && !converged; r++)
        if (!h_flags[rounds + r]) {
          converged = true;
          first_quiet = rounds + r + 1;
        }
      rounds += kRoundsPerBatch;
    }
    ws.t_end();
    tr.mark("  relaxation rounds");
    if (!converged) return declined();
  }

  // 3. block offsets within each interval, then the writing pass
  unsigned* d_err = d_flags + kMaxRounds;
  HdOut o;
  memset(&o, 0, sizeof o);
  for (int c = 0; c < f.ncomp; c++) { o.coefs[c] = d_coefs[c]; o.dcd[c] = d_dcd[c]; }
  o.err = d_err;
  ws.t_begin("huffdec_write");
  count_launches((relax ? 2 : 1) + 3 * f.ncomp);
  if (relax) k_hd_scan<<<1, 1024, 0, s>>>(d_cnt, d_base, nseq);
  k_hd_write<<<grid, 128, 0, s>>>(d_bits, d_out, d_base, d_hs, q, o);
  ws.t_end();
  CUDA_TRY(cudaGetLastError());
  // 4. DC prediction
  ws.t_begin("huffdec_dc");
  for (int c = 0; c < f.ncomp; c++) {
    DcPlan d;
    d.dcd = d_dcd[c];
    d.coefs = d_coefs[c];
    d.n = (unsigned)(mcus * hf.hv[c]);
    d.seg = (unsigned)(ri * hf.hv[c]);
    d.h = hf.h[c]; d.v = hf.v[c]; d.hv = hf.hv[c];
    d.wblocks = hf.wblocks[c]; d.hblocks = hf.hblocks[c];
    d.mcus_per_row = hf.mcus_per_row;
    const unsigned nct = (d.n + kDcCta - 1) / kDcCta;
    d.sums = (int*)ws.dalloc(sizeof(int) * nct);
    if (!d.sums) return E_MEM;
    k_dc_local<<<nct, kDcCta, 0, s>>>(d);
    k_dc_sums<<<1, kDcCta, 0, s>>>(d.sums, nct);
    k_dc_apply<<<(d.n + 255) / 256, 256, 0, s>>>(d);
  }
  ws.t_end();
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(h_flags, d_err, sizeof(unsigned), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  tr.mark("  write + dc");
  if (h_flags[0]) return declined();  // let the host decoder produce the diagnosis
  g_hd_done.fetch_add(1);
  g_hd_rounds.store((unsigned long long)first_quiet);
  return E_OK;
}

}  // namespace uhdr_b200
