"""A model of the encoder's entropy-coded scan, computed on the CPU from a finished baseline stream.

The stream's quantised coefficients come from the checker (oracle/jpeg_oracle.c jo_read_header + jo_decode_coefs),
its code lengths from the stream's own DHT tables.  From them, with numpy (3 M blocks take seconds):

  * the scan order: MCU-interleaved with libjpeg's dummy blocks (Y400: one block per MCU, no dummies);
  * the code bits of every scan block: DC code + magnitude against the last real block of the component (a dummy
    block codes difference 0), run/size codes, one ZRL per 16 zeros, EOB unless coefficient 63 is non-zero;
  * the CTA plan of k_huff_encode (csrc/huffman.cu) for a given bpt: 256 * bpt scan blocks per CTA, each CTA's
    total bits, start bit, shift sh = start % 32, words nrel = ceil(total / 32), windows = ceil(nrel / 2048);
  * the bytes of the unstuffed scan: which are 0xFF, which of those take bits from two CTAs or lie in the first or
    last word of a window, whether the padded final byte is 0xFF;
  * per-block case counts: AC string lengths, coefficient 63 non-zero, ZRLs per zero run, DC category 11.

`block_codes` gives the codes of single blocks, so a plain bit writer can rebuild the scan from the model
(tests/test_jpeg_scan_model_cpu.py pins it that way against libjpeg-turbo's bytes).
"""
import ctypes as C

import numpy as np

import uhdr_testlib as T

THREADS = 256        # k_huff_encode: threads per CTA
SEG_WORDS = 2048     # k_huff_encode: words of one shared-memory window
# zigzag position -> natural index (jutils.c jpeg_natural_order)
NATURAL = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                    6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38,
                    31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])
SIZE = np.array([int(v).bit_length() for v in range(1 << 12)], np.int64)   # magnitude category of |v| < 4096
_CHUNK = 1 << 17


def _oracle():
    T.ensure_oracle_built()
    return C.CDLL(T.ORACLE_SO)


def huff_codes(bits, vals):
    """canonical Huffman code of a DHT table -> (code[256], length[256]); length 0: symbol absent"""
    code = np.zeros(256, np.int64)
    length = np.zeros(256, np.int64)
    c, k = 0, 0
    for ln in range(1, 17):
        for _ in range(bits[ln]):
            code[vals[k]], length[vals[k]] = c, ln
            c += 1
            k += 1
        c <<= 1
    return code, length


def unstuff(scan):
    """stuffed scan bytes -> the coded bytes (the 0x00 after every 0xFF removed)"""
    s = np.frombuffer(scan, np.uint8)
    ff = np.nonzero(s[:-1] == 0xFF)[0]
    assert (s[ff + 1] == 0).all(), "marker inside the scan"
    keep = np.ones(len(s), bool)
    keep[ff + 1] = False
    return s[keep]


def _ac_stats(z, acode_len, zrl_len, eob_len):
    """zigzag blocks (n, 64) -> AC string bits (EOB included), coefficient 63 non-zero, most ZRLs in one run"""
    ac = z[:, 1:].astype(np.int32)
    nz = ac != 0
    pos = np.arange(1, 64, dtype=np.int32)
    last = np.maximum.accumulate(np.where(nz, pos, 0), axis=1)
    prev = np.concatenate([np.zeros((len(z), 1), np.int32), last[:, :-1]], 1)
    run = pos - prev - 1
    size = SIZE[np.abs(ac)]
    nzrl = np.where(nz, run >> 4, 0)
    sym = ((run & 15) << 4) | size
    bits = np.where(nz, acode_len[sym] + size, 0).sum(1) + nzrl.sum(1) * zrl_len
    c63 = nz[:, -1]
    bits = bits + np.where(c63, 0, eob_len)
    return bits, c63, nzrl.max(1), c63 & (nz.sum(1) == 1)


class ScanModel:
    """The scan of one baseline JPEG (one interleaved scan, no restart markers), as the device coder sees it."""

    def __init__(self, data, lib=None):
        lib = lib or _oracle()
        self.data = bytes(data)
        h = T.JoHeader()
        buf = (C.c_uint8 * len(data)).from_buffer_copy(data)
        assert lib.jo_read_header(buf, C.c_size_t(len(data)), C.byref(h)) == 0
        assert h.restart_interval == 0
        f = h.frame
        self.ncomp = f.ncomp
        self.geom = [(f.comp[c].h_samp, f.comp[c].v_samp, f.comp[c].wblocks, f.comp[c].hblocks) for c in range(f.ncomp)]
        nat = [np.zeros((f.comp[c].wblocks * f.comp[c].hblocks, 64), np.int16) for c in range(f.ncomp)]
        cp = (C.c_void_p * 3)(*([a.ctypes.data for a in nat] + [None] * (3 - f.ncomp)))
        assert lib.jo_decode_coefs(buf, C.c_size_t(len(data)), C.byref(h), cp) == 0
        self.z = [a[:, NATURAL] for a in nat]   # zigzag order
        del nat
        # code books of the stream: [component] -> (dc code, dc length), (ac code, ac length)
        self.dcb = [huff_codes(list(h.bits[0][h.dc_sel[c]]), list(h.vals[0][h.dc_sel[c]])) for c in range(f.ncomp)]
        self.acb = [huff_codes(list(h.bits[1][h.ac_sel[c]]), list(h.vals[1][h.ac_sel[c]])) for c in range(f.ncomp)]
        self.scan_offset = h.scan_offset
        assert self.data[-2:] == b"\xff\xd9"
        self.raw = unstuff(self.data[h.scan_offset:-2])
        # per real block of each component
        self.acbits, self.c63, self.maxzrl, self.c63_alone, self.dc = [], [], [], [], []
        for c in range(f.ncomp):
            aclen = self.acb[c][1]
            parts = [_ac_stats(self.z[c][i:i + _CHUNK], aclen, aclen[0xF0], aclen[0]) for i in range(0, len(self.z[c]), _CHUNK)]
            self.acbits.append(np.concatenate([p[0] for p in parts]))
            self.c63.append(np.concatenate([p[1] for p in parts]))
            self.maxzrl.append(np.concatenate([p[2] for p in parts]))
            self.c63_alone.append(np.concatenate([p[3] for p in parts]))
            self.dc.append(self.z[c][:, 0].astype(np.int64))
        self._scan_order(f.mcus_per_row, f.mcu_rows)
        self._block_bits()

    # -- scan order and block bits -----------------------------------------------------------------------
    def _scan_order(self, mpr, mrows):
        if self.ncomp == 1:   # non-interleaved: raster order of the component's blocks
            n = len(self.z[0])
            self.scan_c = np.zeros(n, np.int8)
            self.scan_blk = np.arange(n, dtype=np.int64)
            return
        cs, bs = [], []
        my, mx = np.mgrid[0:mrows, 0:mpr]
        for c, (hs, vs, wb, hb) in enumerate(self.geom):
            ky, kx = np.mgrid[0:vs, 0:hs]
            by = my.reshape(-1, 1) * vs + ky.reshape(1, -1)
            bx = mx.reshape(-1, 1) * hs + kx.reshape(1, -1)
            bs.append(np.where((bx < wb) & (by < hb), by.astype(np.int64) * wb + bx, -1))
            cs.append(np.full(by.shape, c, np.int8))
        self.scan_c = np.concatenate(cs, 1).ravel()
        self.scan_blk = np.concatenate(bs, 1).ravel()

    def _block_bits(self):
        n = len(self.scan_c)
        self.dc_diff = np.zeros(n, np.int64)
        self.bits = np.zeros(n, np.int64)
        for c in range(self.ncomp):
            sel = np.nonzero(self.scan_c == c)[0]
            blk = self.scan_blk[sel]
            real = blk >= 0
            rs, rb = sel[real], blk[real]
            dcs = self.dc[c][rb]
            self.dc_diff[rs] = np.diff(dcs, prepend=0)
            dclen = self.dcb[c][1]
            cat = SIZE[np.abs(self.dc_diff[rs])]
            self.bits[rs] = dclen[cat] + cat + self.acbits[c][rb]
            self.bits[sel[~real]] = dclen[0] + self.acb[c][1][0]
        self.starts = np.concatenate([[0], np.cumsum(self.bits)[:-1]])
        self.total_bits = int(self.bits.sum())
        assert (self.total_bits + 7) // 8 == len(self.raw), "block bits do not add up to the scan"

    @property
    def nblocks(self):
        return len(self.bits)

    # -- codes of single blocks (for a plain bit writer) -----------------------------------------------
    def block_codes(self, s):
        """[(code, length), ...] of scan block s, as jchuff.c encode_one_block emits them"""
        c, blk = int(self.scan_c[s]), int(self.scan_blk[s])
        dcode, dlen = self.dcb[c]
        acode, alen = self.acb[c]
        out = []
        d = int(self.dc_diff[s])
        cat = abs(d).bit_length()
        out.append((int(dcode[cat]), int(dlen[cat])))
        if cat:
            out.append(((d if d > 0 else d - 1) & ((1 << cat) - 1), cat))
        if blk < 0:
            out.append((int(acode[0]), int(alen[0])))
            return out
        z = self.z[c][blk]
        run = 0
        for k in range(1, 64):
            v = int(z[k])
            if v == 0:
                run += 1
                continue
            while run >= 16:
                out.append((int(acode[0xF0]), int(alen[0xF0])))
                run -= 16
            sz = abs(v).bit_length()
            out.append((int(acode[(run << 4) | sz]), int(alen[(run << 4) | sz])))
            out.append(((v if v > 0 else v - 1) & ((1 << sz) - 1), sz))
            run = 0
        if run:
            out.append((int(acode[0]), int(alen[0])))
        return out

    # -- the CTA plan of k_huff_encode ---------------------------------------------------------------------
    def plan(self, bpt):
        chunk = THREADS * bpt
        cstart = np.arange(0, self.nblocks, chunk)
        total = np.add.reduceat(self.bits, cstart)
        start = self.starts[cstart]
        sh = start % 32
        nrel = (total + 31) // 32
        endbit = sh + total
        return dict(bpt=bpt, ncta=len(cstart), first_block=cstart, total=total, start=start, sh=sh, nrel=nrel,
                    first=start // 32, windows=(nrel + SEG_WORDS - 1) // SEG_WORDS,
                    one_word=(endbit >> 5) == 0,               # the whole segment inside stream word `first` (lastw == 0)
                    ends_aligned=(start + total) % 32 == 0)    # the segment ends on a word boundary

    def ff_bytes(self, P):
        """0xFF bytes of the unstuffed scan under plan P -> dict of boolean arrays over them, and their positions"""
        pos = np.nonzero(self.raw == 0xFF)[0]
        lo = pos * 8
        hi = np.minimum(lo + 8, self.total_bits) - 1      # last coded bit of the byte (the rest is padding)
        cta_lo = np.searchsorted(P["start"], lo, "right") - 1
        cta_hi = np.searchsorted(P["start"], hi, "right") - 1
        word = pos // 4
        # the CTA that writes a stream word: the one holding the word's last bit (the last CTA: the padded word)
        owner = np.searchsorted(P["start"], np.minimum(word * 32 + 31, self.total_bits - 1), "right") - 1
        i = word - P["first"][owner]
        nrel, nwin = P["nrel"][owner], P["windows"][owner]
        win = np.minimum(i // SEG_WORDS, nwin - 1)
        wlast = np.minimum((win + 1) * SEG_WORDS, nrel) - 1
        edge = (i == win * SEG_WORDS) | (i >= wlast)
        return dict(pos=pos, two_ctas=cta_lo != cta_hi, window_edge=edge & (nwin > 1),
                    padded_last=(pos == len(self.raw) - 1) & (self.total_bits % 8 != 0))

    # -- case counts -------------------------------------------------------------------------------------
    def ac_lengths(self):
        return np.concatenate(self.acbits)

    def cases(self):
        ac = self.ac_lengths()
        zrl = np.concatenate(self.maxzrl)
        cat11 = [int((SIZE[np.abs(self.dc_diff[self.scan_c == c])] == 11).sum()) for c in range(self.ncomp)]
        return {"ac96": int((ac == 96).sum()), "ac97": int((ac == 97).sum()), "ac128": int((ac == 128).sum()),
                "ac129": int((ac == 129).sum()), "ac_gt96": int((ac > 96).sum()), "ac_max": int(ac.max()),
                "c63": int(sum(int(a.sum()) for a in self.c63)),
                "c63_alone": int(sum(int(a.sum()) for a in self.c63_alone)),
                "zrl1": int((zrl == 1).sum()), "zrl2": int((zrl == 2).sum()), "zrl3": int((zrl == 3).sum()),
                "dc11_luma": cat11[0], "dc11_chroma": sum(cat11[1:])}

    def locate(self, offset, bpt):
        """byte `offset` of the whole stream -> 'CTA c window w block s (component, raster index)' under bpt"""
        if offset < self.scan_offset:
            return f"byte {offset}: headers"
        st = np.frombuffer(self.data[self.scan_offset:offset], np.uint8)
        u = len(st) - int(((st[:-1] == 0xFF) & (st[1:] == 0)).sum())   # unstuffed index
        bit = min(8 * u, self.total_bits - 1)
        P = self.plan(bpt)
        c = int(np.searchsorted(P["start"], bit, "right") - 1)
        s = int(np.searchsorted(self.starts, bit, "right") - 1)
        w = ((bit >> 5) - int(P["first"][c])) // SEG_WORDS
        return (f"byte {offset} (scan byte {u}): CTA {c} of {P['ncta']}, window {w} of {int(P['windows'][c])}, "
                f"scan block {s} (component {int(self.scan_c[s])}, block {int(self.scan_blk[s])}) at bpt {bpt}")


def write_scan(model):
    """a plain bit writer over model.block_codes: the stuffed scan bytes (jchuff.c emit_bits / flush_bits)"""
    acc, n, out = 0, 0, bytearray()
    for s in range(model.nblocks):
        for code, ln in model.block_codes(s):
            acc = (acc << ln) | code
            n += ln
            while n >= 8:
                n -= 8
                b = (acc >> n) & 0xFF
                out.append(b)
                if b == 0xFF:
                    out.append(0)
            acc &= (1 << n) - 1
    if n:
        b = ((acc << (8 - n)) | ((1 << (8 - n)) - 1)) & 0xFF
        out.append(b)
        if b == 0xFF:
            out.append(0)
    return bytes(out)
