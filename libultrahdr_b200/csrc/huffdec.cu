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
// in kMaxRounds rounds, or whose intervals do not decode to exactly their quota of blocks go to the
// host decoder of jpeg_host.cpp.
#include <atomic>
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

// start bit of subsequence i < nseq and its interval *iv
__device__ __forceinline__ unsigned hd_seq_lo(const unsigned* __restrict__ start, const unsigned* __restrict__ first, unsigned nint,
                                              unsigned i, unsigned* iv) {
  unsigned a = 0, b = nint - 1;  // last interval whose first subsequence is <= i
  while (a < b) {
    const unsigned m = (a + b + 1) / 2;
    if (first[m] <= i) a = m;
    else b = m - 1;
  }
  *iv = a;
  return start[a] + (i - first[a]) * (unsigned)kSeqBits;
}

// A batch of scans.  Scan s owns subsequence slots [seq0, seq0 + nseq + 1) of the per-subsequence arrays, seq0 a
// multiple of 128, so that every CTA of the relaxation and writing passes works on one scan and stages one scan's
// tables; and intervals [iv0, iv0 + nint + 1) of the per-interval arrays.  Within its slice a scan is laid out as alone.
struct HdScan {
  const uint32_t* bits;
  unsigned seq0, iv0, nint;
  HdOut o;
};
struct HdBatch {
  const HdShared* gs;     // per scan
  const HdScan* scans;
  const uint2* ctas;      // per CTA of a launch: {scan, first slot}
  const unsigned* start;  // per interval: start bit (local to the scan)
  HdSeqs q;               // lo / iv / first of every scan, values local to the scan
};
__device__ __forceinline__ HdSeqs hd_local(const HdBatch& B, const HdScan& sc) {
  return HdSeqs{B.q.lo + sc.seq0, B.q.iv + sc.seq0, B.q.first + sc.iv0};
}

// expands the per-interval layout built on the host (start bit and first subsequence of each interval) into the
// per-subsequence one, and sets the initial states; one thread per slot
__global__ void __launch_bounds__(128) k_hd_layout(const HdBatch B, unsigned* lo, unsigned* iv, unsigned long long* out,
                                                   unsigned long long* used, unsigned* cnt) {
  const uint2 cta = B.ctas[blockIdx.x];
  const HdScan& sc = B.scans[cta.x];
  const unsigned nseq = B.gs[cta.x].f.nseq, total_bits = B.gs[cta.x].f.total_bits;
  const unsigned i = cta.y - sc.seq0 + threadIdx.x;
  const HdSeqs q = hd_local(B, sc);
  const unsigned* start = B.start + sc.iv0;
  if (i == 0) lo[sc.seq0 + nseq] = total_bits;
  if (i >= nseq) return;
  unsigned iv1;
  lo[sc.seq0 + i] = hd_seq_lo(start, q.first, sc.nint, i, iv + sc.seq0 + i);
  out[sc.seq0 + i] = i + 1 < nseq ? (unsigned long long)hd_seq_lo(start, q.first, sc.nint, i + 1, &iv1) : (unsigned long long)total_bits;
  used[sc.seq0 + i] = ~0ull;
  cnt[sc.seq0 + i] = 0;
}

// one relaxation round over the CTAs of the scans that still need rounds, in place (64-bit states are read and
// written atomically); a scan's change stores round + 1 into last[scan]
__global__ void __launch_bounds__(128) k_hd_sync(const HdBatch B, unsigned long long* out, unsigned long long* used, unsigned* cnt,
                                                 unsigned* last, const unsigned round) {
  __shared__ HdShared S;
  const uint2 cta = B.ctas[blockIdx.x];
  const HdScan& sc = B.scans[cta.x];
  const unsigned seq0 = sc.seq0;
  const unsigned i = cta.y - seq0 + threadIdx.x;
  const HdShared* __restrict__ gs = B.gs + cta.x;
  const HdSeqs q = hd_local(B, sc);
  out += seq0;
  used += seq0;
  cnt += seq0;
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
  const unsigned n = decode_seq<false>(S, sc.bits, p, z, c, q.lo[i + 1], 0, 0, 0, none);
  const unsigned long long now = (unsigned long long)p | ((unsigned long long)(z | (c << 8)) << 32);
  used[i] = entry;
  cnt[i] = n;
  if (now != out[i]) {
    *reinterpret_cast<volatile unsigned long long*>(out + i) = now;
    last[cta.x] = round + 1;
  }
}

// exclusive prefix sum of the block counts of each scan that had rounds: one CTA per scan (nseq is at most a few
// hundred thousand)
__global__ void __launch_bounds__(1024) k_hd_scan(const HdBatch B, const unsigned* __restrict__ which, const unsigned* __restrict__ cnt,
                                                  unsigned* __restrict__ base) {
  const unsigned scan = which[blockIdx.x];
  const unsigned seq0 = B.scans[scan].seq0;
  const unsigned n = B.gs[scan].f.nseq;
  cnt += seq0;
  base += seq0;
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

// the writing pass: each subsequence decoded once more from its entry state, tables staged in S.  out and base are read
// only for subsequences that do not start an interval
__global__ void __launch_bounds__(128) k_hd_write(const HdBatch B, const unsigned long long* __restrict__ out,
                                                  const unsigned* __restrict__ base) {
  __shared__ HdShared S;
  const uint2 cta = B.ctas[blockIdx.x];
  stage_shared(S, B.gs + cta.x);
  const HdScan& sc = B.scans[cta.x];
  const unsigned seq0 = sc.seq0;
  const unsigned i = cta.y - seq0 + threadIdx.x;
  const HdSeqs q = hd_local(B, sc);
  const HdOut& o = sc.o;
  out += seq0;
  base += seq0;
  if (i >= S.f.nseq) return;
  const unsigned k = q.iv[i], head = q.first[k], next = q.first[k + 1];
  const unsigned long long entry = head == i ? (unsigned long long)q.lo[i] : out[i - 1];
  unsigned p = (unsigned)entry, z = (unsigned)(entry >> 32) & 0xff, c = (unsigned)(entry >> 40);
  const unsigned b0 = k * S.f.iv_blocks;
  const unsigned b = b0 + (head == i ? 0u : base[i] - base[head]);
  const unsigned b_end = min(b0 + S.f.iv_blocks, S.f.total_blocks);
  if (b % (unsigned)S.f.bpm != c) *o.err = 2;  // the states and the block counts must agree
  const unsigned n = decode_seq<true>(S, sc.bits, p, z, c, q.lo[i + 1], b, b_end, q.lo[next], o);
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

// The three DC passes over many plans (every component of every scan of a batch), one launch each.  cta_end[j]: the
// CTAs of plans 0..j in the launch's numbering (inclusive prefix), kDcCta-thread CTAs for the local pass, 256-thread
// ones for the scatter; the sums pass runs one CTA per plan.
__global__ void __launch_bounds__(kDcCta) k_dc_local(const DcPlan* __restrict__ plans, const unsigned* __restrict__ cta_end, unsigned n) {
  __shared__ int ws[32];
  const unsigned j = batch_find(cta_end, n, blockIdx.x);
  const DcPlan& d = plans[j];
  const unsigned cta = blockIdx.x - (j ? cta_end[j - 1] : 0);
  const unsigned i = cta * kDcCta + threadIdx.x;
  const int x = cta_inclusive_scan(i < d.n ? d.dcd[i] : 0, ws);
  if (i < d.n) d.dcd[i] = x;
  if (threadIdx.x == kDcCta - 1) d.sums[cta] = x;
}
// each plan's per-CTA totals, in place, exclusive
__global__ void __launch_bounds__(kDcCta) k_dc_sums(const DcPlan* __restrict__ plans) {
  __shared__ int ws[32];
  __shared__ int carry;
  const DcPlan& d = plans[blockIdx.x];
  int* sums = d.sums;
  const unsigned n = (d.n + kDcCta - 1) / kDcCta;
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
__global__ void __launch_bounds__(256) k_dc_apply(const DcPlan* __restrict__ plans, const unsigned* __restrict__ cta_end, unsigned n) {
  const unsigned j = batch_find(cta_end, n, blockIdx.x);
  const DcPlan& d = plans[j];
  const unsigned i = (blockIdx.x - (j ? cta_end[j - 1] : 0)) * 256 + threadIdx.x;
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
bool declined() {
  g_hd_declined.fetch_add(1);
  return false;
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

// The frame description and tables of a scan (all of hs but total_bits and nseq), its MCUs per restart interval and
// its intervals; false for a scan the device decoder does not take
static bool hd_prepare(const JpegHeader& h, HdShared& hs, size_t* ri_out, unsigned* nint_out) {
  const JpegFrame& f = h.frame;
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
  *ri_out = ri;
  *nint_out = nint;
  return true;
}

// subsequences: every interval is cut into pieces of at most kSeqBits bits (an empty interval gets one empty piece,
// whose missing blocks the writing pass reports).  The host numbers them per interval (starts: clean byte offsets in,
// bit offsets out; first[k]: the interval's first subsequence); k_hd_layout expands that on the device.  Returns nseq.
static unsigned hd_intervals(unsigned* starts, unsigned* first, unsigned nint, unsigned total_bits) {
  size_t nseq_total = 0;
  for (unsigned k = 0; k < nint; k++) {
    const unsigned lo = starts[k] * 8u, hi = k + 1 < nint ? starts[k + 1] * 8u : total_bits;
    starts[k] = lo;
    first[k] = (unsigned)nseq_total;
    nseq_total += hi > lo ? (hi - lo + kSeqBits - 1) / kSeqBits : 1;
  }
  first[nint] = (unsigned)nseq_total;
  return (unsigned)nseq_total;
}

// kZigzagDev, once per device
static int upload_zigzag() {
  static PerDevice<const void*> zigzag;
  return device_table(zigzag, 64, [](void* host) { memcpy(host, kZigzag, 64); }, &kZigzagDev) ? E_OK : E_ERROR;
}

namespace {
template <typename T>
T* dalloc_n(Workspace& ws, size_t n) { return (T*)ws.dalloc(sizeof(T) * (n ? n : 1)); }
template <typename T>
T* halloc_n(Workspace& ws, size_t n) { return (T*)ws.halloc(sizeof(T) * (n ? n : 1)); }
void scan_error(JpegScanJob& sc, int rc) {
  sc.rc = rc;
  snprintf(sc.err, sizeof sc.err, "%s", last_error());
}
}  // namespace

int jpeg_entropy_decode_dev(Workspace& ws, JpegScanJob* scans, int n) {
  cudaStream_t s = ws.stream();
  struct Plan {
    bool dev;              // on the device (else the host decoder)
    bool relax;            // has relaxation rounds
    unsigned nint, nseq, seq0, iv0;
    size_t ri, bits_off;   // bits_off: clean bytes before this scan's in the staging buffer (multiple of 4)
  };
  Plan* pl = halloc_n<Plan>(ws, n);
  HdShared* h_hs = halloc_n<HdShared>(ws, n);
  if (!pl || !h_hs) return E_MEM;
  PhaseTrace tr;
  // 1. per scan, on the host: tables, intervals, and the staging size of its clean bits.  With the host decoder
  // selected (jpeg_set_entropy_decoder(1)) every scan goes to it, and the device decoder's counts do not move.
  const bool host_only = jpeg_get_entropy_decoder() == 1;
  size_t bits_cap = 0, niv = 0;
  for (int i = 0; i < n; i++) {
    JpegScanJob& sc = scans[i];
    const JpegHeader& h = *sc.h;
    Plan& p = pl[i];
    memset(&p, 0, sizeof p);
    sc.rc = E_OK;
    for (int c = 0; c < 3; c++) sc.d_coefs[c] = nullptr;
    p.dev = !host_only && hd_prepare(h, h_hs[i], &p.ri, &p.nint);
    if (!p.dev) continue;
    if (sc.size <= h.scan_offset) {
      scan_error(sc, fail(E_ERROR, "Corrupt JPEG data: no entropy-coded segment"));
      continue;
    }
    p.bits_off = bits_cap;
    p.iv0 = (unsigned)niv;
    bits_cap += (sc.size - h.scan_offset + 16 + 3) & ~(size_t)3;
    niv += p.nint + 1;
  }
  uint8_t* h_bits = halloc_n<uint8_t>(ws, bits_cap);
  unsigned* h_start = halloc_n<unsigned>(ws, niv);
  unsigned* h_first = halloc_n<unsigned>(ws, niv);
  if (!h_bits || !h_start || !h_first) return E_MEM;
  // 2. every scan unstuffed into one pinned buffer; a scan with irregular restart markers goes to the host decoder
  size_t nslots = 0, nrelax = 0, cta_all = 0, cta_sync = 0;
  for (int i = 0; i < n; i++) {
    JpegScanJob& sc = scans[i];
    Plan& p = pl[i];
    if (!p.dev || sc.rc) continue;
    uint8_t* dst = h_bits + p.bits_off;
    const long clean = unstuff_scan(sc.data, sc.size, sc.h->scan_offset, dst, sc.h->restart_interval != 0, h_start + p.iv0, p.nint);
    if (clean < 0 || (size_t)clean * 8 > 0xfffffff0u - kSeqBits) {
      p.dev = false;
      declined();
      continue;
    }
    memset(dst + clean, 0, 16);
    HdFrame& hf = h_hs[i].f;
    hf.total_bits = (unsigned)(clean * 8);
    if (hf.total_bits == 0) {
      scan_error(sc, fail(E_ERROR, "Corrupt JPEG data: empty entropy-coded segment"));
      continue;
    }
    p.nseq = hf.nseq = hd_intervals(h_start + p.iv0, h_first + p.iv0, p.nint, hf.total_bits);
    p.relax = p.nseq > p.nint;
    p.seq0 = (unsigned)nslots;
    nslots += (p.nseq + 1 + 127) / 128 * 128;  // + 1: lo[nseq]
    const unsigned ctas = (p.nseq + 127) / 128;
    cta_all += ctas;
    if (p.relax) {
      cta_sync += ctas;
      nrelax++;
    }
  }
  tr.mark("  unstuff");
  if (nslots > 0xffffff00u) return fail(E_ERROR, "internal: entropy-decoder batch of %zu subsequences", nslots);
  // the CTA lists (all scans, then those with rounds), the scans with rounds, the per-scan slices, the DC plans
  uint2* h_ctas = halloc_n<uint2>(ws, cta_all + cta_sync);
  unsigned* h_which = halloc_n<unsigned>(ws, nrelax);
  HdScan* h_scans = halloc_n<HdScan>(ws, n);
  unsigned* h_last = halloc_n<unsigned>(ws, 2 * (size_t)n);  // [0, n): last changing round, [n, 2n): write-pass errors
  DcPlan* h_dc = halloc_n<DcPlan>(ws, 3 * (size_t)n);
  unsigned* h_dc_end = halloc_n<unsigned>(ws, 6 * (size_t)n);  // [0, 3n): local-pass CTAs, [3n, 6n): scatter CTAs
  if (!h_ctas || !h_which || !h_scans || !h_last || !h_dc || !h_dc_end) return E_MEM;
  uint32_t* d_bits = dalloc_n<uint32_t>(ws, bits_cap / 4);
  HdShared* d_hs = dalloc_n<HdShared>(ws, n);
  HdScan* d_scans = dalloc_n<HdScan>(ws, n);
  uint2* d_ctas = dalloc_n<uint2>(ws, cta_all + cta_sync);
  unsigned* d_which = dalloc_n<unsigned>(ws, nrelax);
  unsigned* d_start = dalloc_n<unsigned>(ws, niv);
  unsigned* d_first = dalloc_n<unsigned>(ws, niv);
  unsigned* d_lo = dalloc_n<unsigned>(ws, nslots);
  unsigned* d_iv = dalloc_n<unsigned>(ws, nslots);
  unsigned long long* d_out = dalloc_n<unsigned long long>(ws, nslots);
  unsigned long long* d_used = dalloc_n<unsigned long long>(ws, nslots);
  unsigned* d_cnt = dalloc_n<unsigned>(ws, nslots);
  unsigned* d_base = dalloc_n<unsigned>(ws, nslots);
  unsigned* d_last = dalloc_n<unsigned>(ws, 2 * (size_t)n);
  DcPlan* d_dc = dalloc_n<DcPlan>(ws, 3 * (size_t)n);
  unsigned* d_dc_end = dalloc_n<unsigned>(ws, 6 * (size_t)n);
  if (!d_bits || !d_hs || !d_scans || !d_ctas || !d_which || !d_start || !d_first || !d_lo || !d_iv || !d_out || !d_used || !d_cnt ||
      !d_base || !d_last || !d_dc || !d_dc_end)
    return E_MEM;
  // coefficient blocks start as zeros (the device decoder writes only non-zero coefficients; the host decoder's
  // blocks are copied over them)
  size_t a = 0, b = 0, nw = 0, ndc = 0, n_local = 0, n_apply = 0;
  for (int i = 0; i < n; i++) {
    JpegScanJob& sc = scans[i];
    const Plan& p = pl[i];
    if (sc.rc) continue;
    const JpegFrame& f = sc.h->frame;
    const HdFrame& hf = h_hs[i].f;
    HdScan& hs = h_scans[i];
    memset(&hs, 0, sizeof hs);
    for (int c = 0; c < f.ncomp; c++) {
      sc.d_coefs[c] = (int16_t*)ws.dalloc(f.blocks(c) * 128);
      if (!sc.d_coefs[c]) return E_MEM;
      CUDA_TRY(cudaMemsetAsync(sc.d_coefs[c], 0, f.blocks(c) * 128, s));
    }
    if (!p.dev) continue;
    hs.bits = d_bits + p.bits_off / 4;
    hs.seq0 = p.seq0;
    hs.iv0 = p.iv0;
    hs.nint = p.nint;
    hs.o.err = d_last + n + i;
    const size_t mcus = (size_t)f.mcus_per_row * f.mcu_rows;
    for (int c = 0; c < f.ncomp; c++) {
      hs.o.coefs[c] = sc.d_coefs[c];
      hs.o.dcd[c] = (int*)ws.dalloc(sizeof(int) * mcus * hf.hv[c]);
      if (!hs.o.dcd[c]) return E_MEM;
      DcPlan& d = h_dc[ndc];
      d.dcd = hs.o.dcd[c];
      d.coefs = sc.d_coefs[c];
      d.n = (unsigned)(mcus * hf.hv[c]);
      d.seg = (unsigned)(p.ri * hf.hv[c]);
      d.h = hf.h[c]; d.v = hf.v[c]; d.hv = hf.hv[c];
      d.wblocks = hf.wblocks[c]; d.hblocks = hf.hblocks[c];
      d.mcus_per_row = hf.mcus_per_row;
      const unsigned nct = (d.n + kDcCta - 1) / kDcCta;
      d.sums = (int*)ws.dalloc(sizeof(int) * nct);
      if (!d.sums) return E_MEM;
      n_local += nct;
      n_apply += (d.n + 255) / 256;
      h_dc_end[ndc] = (unsigned)n_local;
      h_dc_end[3 * n + ndc] = (unsigned)n_apply;
      ndc++;
    }
    const unsigned ctas = (p.nseq + 127) / 128;
    for (unsigned c = 0; c < ctas; c++) {
      h_ctas[a++] = make_uint2((unsigned)i, p.seq0 + c * 128);
      if (p.relax) h_ctas[cta_all + b++] = make_uint2((unsigned)i, p.seq0 + c * 128);
    }
    if (p.relax) h_which[nw++] = (unsigned)i;
  }
  if (cta_all) {
    CUDA_TRY(cudaMemcpyAsync(d_bits, h_bits, bits_cap, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(d_hs, h_hs, sizeof(HdShared) * n, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(d_scans, h_scans, sizeof(HdScan) * n, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(d_ctas, h_ctas, sizeof(uint2) * (cta_all + cta_sync), cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(d_which, h_which, sizeof(unsigned) * (nrelax ? nrelax : 1), cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(d_start, h_start, sizeof(unsigned) * niv, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(d_first, h_first, sizeof(unsigned) * niv, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(d_dc, h_dc, sizeof(DcPlan) * ndc, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(d_dc_end, h_dc_end, sizeof(unsigned) * 6 * n, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemsetAsync(d_last, 0, sizeof(unsigned) * 2 * n, s));
    if (int rc = upload_zigzag()) return rc;
    HdBatch B = {d_hs, d_scans, d_ctas, d_start, HdSeqs{d_lo, d_iv, d_first}};
    k_hd_layout<<<(unsigned)cta_all, 128, 0, s>>>(B, d_lo, d_iv, d_out, d_used, d_cnt);
    count_launches(1);
    CUDA_TRY(cudaGetLastError());
    tr.mark("  interval layout");
    // 3. relaxation rounds over every scan that has them, one host check per kRoundsPerBatch rounds for the whole
    // batch, until each of them has had a round that changed nothing
    int rounds = 0;
    bool pending = cta_sync > 0;
    HdBatch Bs = B;
    Bs.ctas = d_ctas + cta_all;
    if (pending) ws.t_begin("huffdec_sync");
    while (pending && rounds < kMaxRounds) {
      count_launches(kRoundsPerBatch);
      for (int r = 0; r < kRoundsPerBatch; r++)
        k_hd_sync<<<(unsigned)cta_sync, 128, 0, s>>>(Bs, d_out, d_used, d_cnt, d_last, (unsigned)(rounds + r));
      CUDA_TRY(cudaGetLastError());
      CUDA_TRY(cudaMemcpyAsync(h_last, d_last, sizeof(unsigned) * n, cudaMemcpyDeviceToHost, s));
      CUDA_TRY(cudaStreamSynchronize(s));
      rounds += kRoundsPerBatch;
      pending = false;
      for (size_t j = 0; j < nrelax; j++) pending = pending || h_last[h_which[j]] == (unsigned)rounds;  // changed in the last round
    }
    if (cta_sync) {
      ws.t_end();
      tr.mark("  relaxation rounds");
    }
    for (size_t j = 0; j < nrelax; j++) {
      const unsigned i = h_which[j];
      if (h_last[i] == (unsigned)rounds) {  // no quiet round in kMaxRounds: the host decoder takes it
        pl[i].dev = false;
        declined();
      }
    }
    // 4. block offsets within each interval, the writing pass, DC prediction: one launch each for the batch
    ws.t_begin("huffdec_write");
    if (nrelax) k_hd_scan<<<(unsigned)nrelax, 1024, 0, s>>>(B, d_which, d_cnt, d_base);
    k_hd_write<<<(unsigned)cta_all, 128, 0, s>>>(B, d_out, d_base);
    ws.t_end();
    ws.t_begin("huffdec_dc");
    k_dc_local<<<(unsigned)n_local, kDcCta, 0, s>>>(d_dc, d_dc_end, (unsigned)ndc);
    k_dc_sums<<<(unsigned)ndc, kDcCta, 0, s>>>(d_dc);
    k_dc_apply<<<(unsigned)n_apply, 256, 0, s>>>(d_dc, d_dc_end + 3 * n, (unsigned)ndc);
    ws.t_end();
    count_launches((nrelax ? 1 : 0) + 4);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(h_last + n, d_last + n, sizeof(unsigned) * n, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    tr.mark("  write + dc");
    for (int i = 0; i < n; i++) {
      if (!pl[i].dev || scans[i].rc) continue;
      if (h_last[n + i]) {  // let the host decoder produce the diagnosis
        pl[i].dev = false;
        declined();
      } else {
        g_hd_done.fetch_add(1);
        g_hd_rounds.store(pl[i].relax ? (unsigned long long)h_last[i] + 1 : 0ull);  // the first quiet round
      }
    }
  }
  // 5. the scans the device decoder did not take, on the host; their blocks replace the device's
  for (int i = 0; i < n; i++) {
    JpegScanJob& sc = scans[i];
    if (pl[i].dev || sc.rc) continue;
    const JpegFrame& f = sc.h->frame;
    int16_t* h_coefs[3] = {nullptr, nullptr, nullptr};
    for (int c = 0; c < f.ncomp; c++) {
      h_coefs[c] = (int16_t*)ws.halloc(f.blocks(c) * 128);
      if (!h_coefs[c]) return E_MEM;
    }
    if (int rc = jpeg_host_decode_coefs(sc.data, sc.size, *sc.h, h_coefs)) {
      scan_error(sc, rc);
      continue;
    }
    for (int c = 0; c < f.ncomp; c++)
      CUDA_TRY(cudaMemcpyAsync(sc.d_coefs[c], h_coefs[c], f.blocks(c) * 128, cudaMemcpyHostToDevice, s));
  }
  return E_OK;
}

}  // namespace uhdr_b200
