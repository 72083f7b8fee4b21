"""A baseline JPEG writer for decoder tests, and a model of the device entropy decoder's relaxation (huffdec.cu).

Writer: quantised coefficient blocks (natural order, absolute DC) -> a complete baseline stream with any DHT
content (Annex K, optimal tables built from the blocks' own symbol counts, hand-made ones), any DC / AC table
selector per component, 8- or 16-bit DQT, any sampling factors (h, v <= 4, at most 10 blocks per MCU) with
libjpeg's dummy edge blocks, and DRI / RSTn markers with optional 0xFF fill bytes before a marker.  `Stream.syms`
gives the clean (unstuffed) bit offset, kind and scan block of every symbol, so a case can put a subsequence
boundary exactly where it wants.

Model: `Decoder.decode` is decode_seq of huffdec.cu over the clean bits (same tables, same handling of codes that are
not in the table), `relax_rounds` replays k_hd_layout + k_hd_sync rounds in lock step (each round reads only the
states of the round before), and `flat_phases` lists the bit phases of a repeating flat MCU from which a decoder
started in the first-guess state (DC symbol of block 0 next) never falls back into step.
"""
import io
import struct

import numpy as np

from jpeg_scan_model import NATURAL, huff_codes

SEQ_BITS = 1024      # huffdec.cu kSeqBits
MAX_ROUNDS = 512     # huffdec.cu kMaxRounds


# ---- tables ---------------------------------------------------------------------------------------------------------
def read_markers(data):
    """-> list of (marker, payload bytes) up to SOS (included), and the offset of the entropy-coded segment"""
    out, p = [], 2
    assert data[:2] == b"\xff\xd8"
    while True:
        while data[p + 1] == 0xFF:
            p += 1
        m = data[p + 1]
        n = (data[p + 2] << 8) | data[p + 3]
        out.append((m, data[p + 4:p + 2 + n]))
        p += 2 + n
        if m == 0xDA:
            return out, p


def read_tables(data):
    """DHT tables of a stream -> {(cls, id): (bits[17], vals)}"""
    tabs = {}
    for m, s in read_markers(data)[0]:
        i = 0
        while m == 0xC4 and i < len(s):
            cls, tid = s[i] >> 4, s[i] & 15
            bits = [0] + list(s[i + 1:i + 17])
            n = sum(bits)
            tabs[(cls, tid)] = (bits, list(s[i + 17:i + 17 + n]))
            i += 17 + n
    return tabs


def annex_k():
    """the Annex K tables (K.3), as libjpeg writes them by default: {(cls, id): (bits, vals)}"""
    from PIL import Image
    b = io.BytesIO()
    Image.new("YCbCr", (8, 8)).save(b, "JPEG", quality=90)
    return read_tables(b.getvalue())


def optimal_table(freq, maxlen=16):
    """Huffman code lengths from symbol counts by the procedure of Annex K.2 (one reserved code point so that no
    code is all ones; lengths limited to maxlen by K.3's adjustment) -> (bits[17], vals)"""
    freq = [int(x) for x in freq] + [0] * (257 - len(freq))
    freq[256] = 1
    size = [0] * 257
    others = [-1] * 257
    while True:
        c1 = c2 = -1
        v = 1 << 60
        for i in range(257):
            if freq[i] and freq[i] <= v:
                v, c1 = freq[i], i
        v = 1 << 60
        for i in range(257):
            if freq[i] and freq[i] <= v and i != c1:
                v, c2 = freq[i], i
        if c2 < 0:
            break
        freq[c1] += freq[c2]
        freq[c2] = 0
        size[c1] += 1
        while others[c1] >= 0:
            c1 = others[c1]
            size[c1] += 1
        others[c1] = c2
        size[c2] += 1
        while others[c2] >= 0:
            c2 = others[c2]
            size[c2] += 1
    bits = [0] * 64
    for i in range(257):
        if size[i]:
            bits[size[i]] += 1
    for i in range(63, maxlen, -1):
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = maxlen
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1   # the reserved code point
    vals = [s for ln in range(1, 33) for s in range(256) if size[s] == ln]
    return [0] + bits[1:17], vals


def table_from_lengths(order, lengths):
    """symbols in `order` get code lengths `lengths` (ascending, a prefix code without the all-ones code)"""
    assert list(lengths) == sorted(lengths) and sum(2.0 ** -ln for ln in lengths) < 1.0
    bits = [0] * 17
    for ln in lengths:
        bits[ln] += 1
    return bits, list(order)


def chain_table(order):
    """lengths 1, 2, ..., n for the n symbols of `order` (n <= 16)"""
    return table_from_lengths(order, range(1, len(order) + 1))


def reversed_table(freq):
    """the optimal code lengths handed out in reverse: the most common symbol gets the longest code"""
    bits, vals = optimal_table(freq)
    lens = [ln for ln in range(1, 17) for _ in range(bits[ln])]
    f = np.asarray(list(freq) + [0] * (256 - len(freq)))
    order = sorted(vals, key=lambda s: (int(f[s]), -s))   # rarest first
    return table_from_lengths(order, lens)


# ---- frame geometry -------------------------------------------------------------------------------------------------
def _cdiv(a, b):
    return -(-a // b)


class Frame:
    """libjpeg's geometry of a baseline frame: comps = [(h, v), ...]"""

    def __init__(self, width, height, samp):
        self.width, self.height = width, height
        self.samp = [(1, 1)] if len(samp) == 1 else list(samp)
        self.ncomp = len(samp)
        self.max_h = max(h for h, v in self.samp)
        self.max_v = max(v for h, v in self.samp)
        if self.ncomp == 1:
            self.mpr, self.mrows = _cdiv(width, 8), _cdiv(height, 8)
        else:
            self.mpr, self.mrows = _cdiv(width, 8 * self.max_h), _cdiv(height, 8 * self.max_v)
        # per component: downsampled size, real blocks, blocks of the MCU grid
        self.dw = [_cdiv(width * h, self.max_h) for h, v in samp]
        self.dh = [_cdiv(height * v, self.max_v) for h, v in samp]
        self.wb = [_cdiv(w, 8) for w in self.dw]
        self.hb = [_cdiv(h, 8) for h in self.dh]
        self.bpm = sum(h * v for h, v in self.samp)
        assert self.bpm <= 10
        # scan order: (component, block row, block column) of every MCU position
        self.mcu_pos = [(c, j, i) for c, (h, v) in enumerate(self.samp) for j in range(v) for i in range(h)]

    @property
    def mcus(self):
        return self.mpr * self.mrows

    def blocks(self, c):
        return self.wb[c] * self.hb[c]

    def scan_blocks(self):
        """scan order -> list of (component, raster index or -1 for a dummy block), MCU by MCU"""
        out = []
        for my in range(self.mrows):
            for mx in range(self.mpr):
                for c, j, i in self.mcu_pos:
                    bx, by = mx * self.samp[c][0] + i, my * self.samp[c][1] + j
                    out.append((c, by * self.wb[c] + bx if bx < self.wb[c] and by < self.hb[c] else -1))
        return out


# ---- symbols of a scan ----------------------------------------------------------------------------------------------
def _cat(v):
    return abs(int(v)).bit_length()


def _mag(v, s):
    return (v if v >= 0 else v - 1) & ((1 << s) - 1)


def block_symbols(zz, dc_diff):
    """one block (zigzag order) -> [(kind, symbol, magnitude value, magnitude bits)], kinds 'dc', 'ac', 'zrl', 'eob'"""
    s = _cat(dc_diff)
    out = [("dc", s, _mag(dc_diff, s), s)]
    run = 0
    for k in range(1, 64):
        v = int(zz[k])
        if v == 0:
            run += 1
            continue
        while run >= 16:
            out.append(("zrl", 0xF0, 0, 0))
            run -= 16
        sz = _cat(v)
        out.append(("ac", (run << 4) | sz, _mag(v, sz), sz))
        run = 0
    if run:
        out.append(("eob", 0x00, 0, 0))
    return out


class Stream:
    """A written stream: .data, and per symbol (clean bit offset, kind, scan block, code bits, magnitude bits)"""


def scan_symbols(frame, coefs, restart=0):
    """[(interval, scan block, component, block symbols)] in scan order; DC prediction restarts every interval"""
    order = frame.scan_blocks()
    zz = [np.asarray(c)[:, NATURAL] if len(c) else np.zeros((0, 64), np.int64) for c in coefs]
    per_iv = restart * frame.bpm if restart else len(order)
    pred = [0] * frame.ncomp
    empty = np.zeros(64, np.int64)
    out = []
    for s, (c, b) in enumerate(order):
        if s % per_iv == 0:
            pred = [0] * frame.ncomp
        z = zz[c][b] if b >= 0 else empty
        dc = int(z[0]) if b >= 0 else pred[c]   # a dummy block codes difference 0 (jccoefct.c)
        out.append((s // per_iv, s, c, block_symbols(z, dc - pred[c])))
        pred[c] = dc
    return out


def symbol_counts(frame, coefs, sel, restart=0):
    """symbol counts per (cls, table id) under selectors sel = [(dc id, ac id), ...]"""
    cnt = {}
    for _iv, _s, c, syms in scan_symbols(frame, coefs, restart):
        for kind, sym, _v, _n in syms:
            key = (0, sel[c][0]) if kind == "dc" else (1, sel[c][1])
            cnt.setdefault(key, np.zeros(256, np.int64))[sym] += 1
    return cnt


def optimal_tables(frame, coefs, sel, restart=0, maxlen=16):
    return {k: optimal_table(v, maxlen) for k, v in symbol_counts(frame, coefs, sel, restart).items()}


# ---- the writer -----------------------------------------------------------------------------------------------------
def _seg(marker, payload):
    return bytes([0xFF, marker]) + struct.pack(">H", len(payload) + 2) + bytes(payload)


def write_jpeg(width, height, samp, coefs, tables, sel=None, qt=None, tq=None, dqt16=False, restart=0, fill=0,
               extra_dht=()):
    """samp: [(h, v)] per component; coefs: per component (wb * hb, 64) ints, natural order, absolute DC;
    tables: {(cls, id): (bits, vals)}; sel: [(dc id, ac id)] per component (default luma 0, chroma 1);
    qt: {id: 64 values in natural order} (default all ones); tq: quantiser id per component;
    restart: DRI interval in MCUs (0: none); fill: 0xFF fill bytes before every RSTn;
    extra_dht: more (cls, id, bits, vals) written in a DHT after the others (a later definition replaces an earlier).
    -> Stream"""
    fr = Frame(width, height, samp)
    n = fr.ncomp
    sel = sel or [(0, 0)] + [(1, 1)] * (n - 1)
    tq = tq or [0] + [1] * (n - 1)
    qt = qt or {0: [1] * 64, 1: [1] * 64}
    for c in range(n):
        assert np.asarray(coefs[c]).shape == (fr.blocks(c), 64), (c, np.asarray(coefs[c]).shape)
    books = {k: huff_codes(b, v) for k, v in tables.items() for b, v in [v]}
    hdr = bytearray(b"\xff\xd8") + _seg(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for tid in sorted(set(tq)):
        q = np.asarray(qt[tid])[NATURAL]
        if dqt16:
            hdr += _seg(0xDB, bytes([0x10 | tid]) + b"".join(struct.pack(">H", int(x)) for x in q))
        else:
            assert q.max() <= 255
            hdr += _seg(0xDB, bytes([tid]) + bytes(int(x) for x in q))
    sof = bytearray([8]) + struct.pack(">HH", height, width) + bytes([n])
    for c in range(n):
        h, v = samp[c]
        sof += bytes([c + 1, (h << 4) | v, tq[c]])
    hdr += _seg(0xC0, sof)
    dht = bytearray()
    for (cls, tid), (bits, vals) in sorted(tables.items()):
        dht += bytes([(cls << 4) | tid]) + bytes(bits[1:17]) + bytes(vals)
    hdr += _seg(0xC4, dht)
    if extra_dht:
        hdr += _seg(0xC4, b"".join(bytes([(cls << 4) | tid]) + bytes(bits[1:17]) + bytes(vals)
                                   for cls, tid, bits, vals in extra_dht))
    if restart:
        hdr += _seg(0xDD, struct.pack(">H", restart))
    sos = bytearray([n])
    for c in range(n):
        sos += bytes([c + 1, (sel[c][0] << 4) | sel[c][1]])
    hdr += _seg(0xDA, sos + b"\x00\x3f\x00")

    # symbols -> bit strings per interval
    ivs, syms, clean_off = [], [], 0
    cur, cur_iv, pos = [], 0, 0

    def close():
        nonlocal cur, pos, clean_off
        s = "".join(cur)
        pad = (-len(s)) % 8
        ivs.append((clean_off, s + "1" * pad))
        clean_off += len(s) + pad
        cur, pos = [], 0

    for iv, s, c, bs in scan_symbols(fr, coefs, restart):
        if iv != cur_iv:
            close()
            cur_iv = iv
        for kind, sym, val, nb in bs:
            cls, tid = (0, sel[c][0]) if kind == "dc" else (1, sel[c][1])
            code, length = books[(cls, tid)]
            ln = int(length[sym])
            assert ln, ("symbol not in table", cls, tid, hex(sym))
            syms.append((clean_off + pos, kind, s, ln, nb))
            cur.append(format(int(code[sym]), "0%db" % ln))
            if nb:
                cur.append(format(val, "0%db" % nb))
            pos += ln + nb
    close()
    body = bytearray()
    starts = []
    for k, (off, bitstr) in enumerate(ivs):
        if k:
            body += b"\xff" * fill + bytes([0xFF, 0xD0 + (k - 1) % 8])
        starts.append(off)
        raw = int(bitstr, 2).to_bytes(len(bitstr) // 8, "big") if bitstr else b""
        body += raw.replace(b"\xff", b"\xff\x00")
    st = Stream()
    st.frame, st.sel, st.tables, st.restart = fr, sel, tables, restart
    st.coefs = [np.asarray(c) for c in coefs]
    st.data = bytes(hdr + body + b"\xff\xd9")
    st.clean = b"".join(int(b, 2).to_bytes(len(b) // 8, "big") if b else b"" for _o, b in ivs)
    st.starts = starts               # clean bit offset of every restart interval
    st.total_bits = clean_off
    st.syms = syms                   # (clean bit offset, kind, scan block, code bits, magnitude bits)
    st.scan_data = bytes(body)
    return st


# ---- model of the device decoder (huffdec.cu) -----------------------------------------------------------------------
class DecTables:
    """16-bit peek -> (code length, symbol) of decode_seq: the 9-bit LUT, then the canonical long-code search;
    a code of no length <= 16 decodes as (16, 0)"""

    def __init__(self, bits, vals):
        lut = np.zeros((1 << 16, 2), np.int64)
        lut[:, 0] = 16
        filled = np.zeros(1 << 16, bool)
        code = k = 0
        for ln in range(1, 17):
            for _ in range(bits[ln]):
                lo, hi = code << (16 - ln), (code + 1) << (16 - ln)
                sel = ~filled[lo:hi]
                lut[lo:hi][sel] = (ln, vals[k])
                filled[lo:hi] = True
                code += 1
                k += 1
            code <<= 1
        self.lut = [tuple(x) for x in lut.tolist()]


class Decoder:
    """decode_seq<false> of huffdec.cu over a stream's clean bits"""

    def __init__(self, st):
        f = st.frame
        self.comp_of = [c for c, j, i in f.mcu_pos] if f.ncomp > 1 else [0]
        self.bpm = len(self.comp_of)
        t = {k: DecTables(*v) for k, v in st.tables.items()}
        self.dc = [t[(0, st.sel[c][0])].lut for c in range(f.ncomp)]
        self.ac = [t[(1, st.sel[c][1])].lut for c in range(f.ncomp)]
        self.bits = st.clean + bytes(16)

    def peek(self, p, n):
        """n <= 32 bits from bit p (the clean bits are followed by 16 zero bytes, like the device's copy)"""
        k = p >> 3
        return (int.from_bytes(self.bits[k:k + 5], "big") >> (40 - (p & 7) - n)) & ((1 << n) - 1)

    def decode(self, p, z, c, end):
        """state (p, z, c) -> state after the symbols that start before `end`, and the blocks finished"""
        nblk = 0
        while p < end:
            w = self.peek(p, 16)
            comp = self.comp_of[c]
            ln, sym = (self.dc if z == 0 else self.ac)[comp][w]
            s = sym & 15
            p += ln + s
            if z == 0:
                z = 1
            elif s:
                z += (sym >> 4) + 1
            else:
                z = z + 16 if sym >> 4 == 15 else 64
            if z >= 64:
                z = 0
                nblk += 1
                c = 0 if c + 1 == self.bpm else c + 1
        return (p, z, c), nblk


def subsequences(st):
    """[(lo, hi, first of its interval)] as jpeg_entropy_decode_dev cuts the clean bits"""
    out = []
    for k, lo in enumerate(st.starts):
        hi = st.starts[k + 1] if k + 1 < len(st.starts) else st.total_bits
        n = max(1, _cdiv(hi - lo, SEQ_BITS))
        out += [(lo + i * SEQ_BITS, min(lo + (i + 1) * SEQ_BITS, hi) if hi > lo else hi, i == 0) for i in range(n)]
    return out


def relax_rounds(st, max_rounds=MAX_ROUNDS):
    """k_hd_layout + k_hd_sync in lock step -> (first round that changes nothing, or None if none within
    max_rounds; 0 when every subsequence starts an interval; subsequences; per round the subsequences it changed)"""
    seqs = subsequences(st)
    n = len(seqs)
    if n == len(st.starts):
        return 0, seqs, []
    d = Decoder(st)
    out = [(seqs[i][1], 0, 0) for i in range(n)]
    used = [None] * n
    changed = []
    for r in range(1, max_rounds + 1):
        entry = [(seqs[i][0], 0, 0) if seqs[i][2] else out[i - 1] for i in range(n)]
        new, ch = list(out), []
        for i in range(n):
            if entry[i] == used[i]:
                continue
            used[i] = entry[i]
            now, _nb = d.decode(*entry[i], seqs[i][1])
            if now != out[i]:
                new[i] = now
                ch.append(i)
        out = new
        changed.append(ch)
        if not ch:
            return r, seqs, changed
    return None, seqs, changed


def flat_phases(samp, tables, sel=None, mcus=64):
    """Phases of a flat MCU pattern (every block "DC difference 0, EOB") from which a decoder started in the
    first-guess state (DC symbol of block 0 next) never falls back into step -> (MCU bits, sorted phases)"""
    fr_w = 8 * max(h for h, v in samp) * mcus
    fr_h = 8 * max(v for h, v in samp)
    fr = Frame(fr_w, fr_h, samp)
    coefs = [np.zeros((fr.blocks(c), 64), np.int64) for c in range(fr.ncomp)]
    st = write_jpeg(fr_w, fr_h, samp, coefs, tables, sel)
    d = Decoder(st)
    starts =[o for o, kind, s, _l, _n in st.syms if kind == "dc" and s % fr.bpm == 0]
    period = starts[1] - starts[0]
    true_states = {}   # phase -> (z, c) of the true decoder at every symbol start within one MCU
    for o, kind, s, _l, _n in st.syms[:2 * fr.bpm]:
        true_states[o % period] = (0 if kind == "dc" else 1, s % fr.bpm)
    bad = []
    for ph in range(period):
        state, seen = (period * 2 + ph, 0, 0), set()
        synced = False
        while state[0] < st.total_bits - 2 * period:
            key = (state[0] % period, state[1], state[2])
            if key in seen:
                break
            seen.add(key)
            if true_states.get(key[0]) == (1 if key[1] else 0, key[2]) and key[1] <= 1:
                synced = True
                break
            state, _ = d.decode(state[0], state[1], state[2], state[0] + 1)
        if not synced:
            bad.append(ph)
    return period, bad
