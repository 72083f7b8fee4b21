"""The streams of tests/test_gpu_jpeg_decode_routes.py, built on the CPU with tests/jpeg_stream_writer.py.

Every builder returns (name, Stream or bytes, expect): expect["rounds"] is the relaxation round count the lock-step
model predicts (None: more than kMaxRounds, so the device decoder hands the stream back), and expect["why"] says,
from the writer's symbol offsets or the model, why the stream reaches its case.  tests/test_jpeg_stream_writer_cpu.py
decodes every stream with libjpeg-turbo and requires zero warnings.
"""
import numpy as np

import jpeg_stream_writer as W

S420, S422, S444, S440 = [(2, 2), (1, 1), (1, 1)], [(2, 1), (1, 1), (1, 1)], [(1, 1)] * 3, [(1, 2), (1, 1), (1, 1)]
S411, S410, GRAY = [(4, 1), (1, 1), (1, 1)], [(4, 2), (1, 1), (1, 1)], [(1, 1)]
K = W.annex_k()
FLAT_BAD = {"420": W.flat_phases(S420, K)[1], "gray": W.flat_phases(GRAY, K)[1], "444": W.flat_phases(S444, K)[1]}


def _zeros(fr):
    return [np.zeros((fr.blocks(c), 64), np.int64) for c in range(fr.ncomp)]


def random_blocks(rs, n, amp, density, dc_amp=40):
    """n blocks, natural order: DC uniform in +-dc_amp, AC Laplacian-ish of scale amp on a random `density` share"""
    b = np.zeros((n, 64), np.int64)
    b[:, 0] = rs.randint(-dc_amp, dc_amp + 1, n)
    mask = rs.rand(n, 63) < density * np.exp(-np.arange(63) / 20.0)
    vals = np.round(rs.laplace(0, amp, (n, 63))).astype(np.int64)
    b[:, 1:] = np.where(mask, np.clip(vals, -1023, 1023), 0)
    return b


def alphabet_blocks(rs, n, ac_syms, dc_amp=20):
    """n blocks whose AC symbols all come from ac_syms (EOB, ZRL and (run, size) symbols)"""
    real = [s for s in ac_syms if s not in (0x00, 0xF0)]
    b = np.zeros((n, 64), np.int64)
    b[:, 0] = rs.randint(-dc_amp, dc_amp + 1, n)
    zz = W.NATURAL
    for i in range(n):
        pos = 1
        for _ in range(rs.randint(0, 12)):
            zrl = 0xF0 in ac_syms and rs.rand() < 0.2
            sym = real[rs.randint(len(real))]
            r, s = sym >> 4, sym & 15
            p = pos + (16 if zrl else 0) + r
            if p > 63:
                break
            mag = rs.randint(1 << (s - 1), 1 << s)
            b[i, zz[p]] = mag if rs.rand() < 0.5 else -mag
            pos = p + 1
    return b


def pil_coefs(w, h, layout, q, kind, seed):
    """coefficients of a Pillow stream (natural order), read back with the C restatement"""
    import scaled_testlib as S
    data = S.pil_jpeg(S.image(w, h, kind, seed=seed), q, layout)
    return pil_coefs_of(data), data


def _header(data):
    import ctypes as C
    import uhdr_testlib as T
    hd = T.JoHeader()
    buf = (C.c_uint8 * len(data)).from_buffer_copy(data)
    assert C.CDLL(T.ORACLE_SO).jo_read_header(buf, C.c_size_t(len(data)), C.byref(hd)) == 0
    return hd


def pil_coefs_of(data):
    import ctypes as C
    import uhdr_testlib as T
    lib = C.CDLL(T.ORACLE_SO)
    hd = T.JoHeader()
    buf = (C.c_uint8 * len(data)).from_buffer_copy(data)
    assert lib.jo_read_header(buf, C.c_size_t(len(data)), C.byref(hd)) == 0
    f = hd.frame
    co = [np.zeros((f.comp[c].wblocks * f.comp[c].hblocks, 64), np.int16) for c in range(f.ncomp)]
    cp = (C.c_void_p * 3)(*([a.ctypes.data for a in co] + [None] * (3 - f.ncomp)))
    assert lib.jo_decode_coefs(buf, C.c_size_t(len(data)), C.byref(hd), cp) == 0
    return [a.astype(np.int64) for a in co]


def _lens(tab):
    return W.huff_codes(*tab)[1]


def pillow_stream(data):
    """a Pillow stream as a Stream (the writer's scan from its coefficients and tables is byte-identical), so that the
    model can predict its rounds"""
    co = pil_coefs_of(data)
    hd = _header(data)
    f = hd.frame
    samp = [(f.comp[c].h_samp, f.comp[c].v_samp) for c in range(f.ncomp)]
    st = W.write_jpeg(f.width, f.height, samp, co, W.read_tables(data), [(hd.dc_sel[c], hd.ac_sel[c]) for c in range(f.ncomp)])
    assert st.scan_data + b"\xff\xd9" == data[W.read_markers(data)[1]:]
    st.data = data
    return st


def frontier_only(st, rounds=6):
    """the lock-step model's first rounds: when only the frontier settles (the changed subsequences drop by at most 2
    a round) and more of them are left than the remaining rounds plus the CTA boundaries the device may cross a round
    early, no fixed point comes within kMaxRounds -> (changed counts, verdict)"""
    _r, seqs, changed = W.relax_rounds(st, rounds)
    n = [len(c) for c in changed]
    return n, all(a - b <= 2 for a, b in zip(n, n[1:])) and n[-1] > W.MAX_ROUNDS - rounds + len(seqs) // 128 + 2


def _case(name, st, why, rounds="model"):
    if rounds == "model" and not isinstance(st, bytes) and st.total_bits > 600000:
        n, never = frontier_only(st)
        if never:
            return name, st, {"rounds": None, "why": why + "; subsequences each lock-step round changes: %s" % n}
    if rounds == "model":
        rounds = W.relax_rounds(st)[0] if not isinstance(st, bytes) else "any"
    return name, st, {"rounds": rounds, "why": why}


# ---- lead blocks: one block whose coded length exceeds an empty block's by any chosen number of bits ----------------
def _lead_map(tab_ac):
    """delta (bits over "DC 0, EOB") -> zigzag AC content of one block, from (0, s) symbols of categories <= 5 only (a
    block of larger values can leave the 16-bit range of libjpeg-turbo's SIMD IDCT, where it and the exact IDCT part)"""
    ln = _lens(tab_ac)
    out = {}
    for nbig in range(0, 63):
        for n1 in range(0, 63 - nbig):
            for extra in (0, 2, 3, 4):
                k = nbig + n1 + (1 if extra else 0)
                if k > 62:
                    continue
                d = nbig * (ln[0x05] + 5) + n1 * (ln[0x01] + 1) + (ln[extra] + extra if extra else 0)   # EOB in both
                if d not in out:
                    z = [(-1) ** i * 31 for i in range(nbig)] + [1] * n1 + ([(1 << extra) - 1] if extra else [])
                    out[d] = z
    return out


_LEAD = {}


def lead_deltas():
    if not _LEAD:
        _LEAD.update(_lead_map(K[(1, 0)]))
    return _LEAD


def lead_block(delta, dc=0):
    """a luma block (Annex K tables) whose code is `delta` bits longer than "DC difference 0, EOB"'s"""
    z = lead_deltas()[delta]
    b = np.zeros(64, np.int64)
    b[0] = dc
    b[W.NATURAL[1:1 + len(z)]] = z
    return b


# ---- A: table shapes ------------------------------------------------------------------------------------------------
def cases_tables():
    out = []
    import scaled_testlib as S
    for kind, q in (("noise", 20), ("noise", 100), ("smooth", 60), ("smooth", 100)):
        data = S.pil_jpeg(S.image(328, 200, kind, seed=q), q, "420", optimize=True)
        out.append(_case("A_pillow_optimal_%s_q%d" % (kind, q), pillow_stream(data),
                         "Pillow optimize=True: tables from the image's counts"))
    for kind, q, layout, samp in (("noise", 30, "420", S420), ("smooth", 95, "444", S444), ("noise", 90, "gray", GRAY)):
        co, _d = pil_coefs(264, 136, layout, q, kind, 5)
        sel = [(0, 0)] + [(1, 1)] * (len(samp) - 1)
        fr = W.Frame(264, 136, samp)
        tabs = W.optimal_tables(fr, co, sel)
        st = W.write_jpeg(264, 136, samp, co, tabs, sel)
        out.append(_case("A_writer_optimal_%s_%s_q%d" % (layout, kind, q), st, "optimal tables from the blocks' counts"))
    # DC: the common category on a 1-bit code, then on a 12-bit code; AC: every code <= 9 bits; EOB and (0,1) long
    co, _d = pil_coefs(200, 152, "420", 50, "smooth", 7)
    fr = W.Frame(200, 152, S420)
    sel = [(0, 0), (1, 1), (1, 1)]
    cnt = W.symbol_counts(fr, co, sel)
    common = int(np.argmax(cnt[(0, 0)]))
    order = [common] + [c for c in range(12) if c != common]
    for tag, dc0 in (("dc_1bit", W.chain_table(order)), ("dc_12bit", W.chain_table(order[::-1]))):
        tabs = dict(K)
        tabs[(0, 0)] = dc0
        st = W.write_jpeg(200, 152, S420, co, tabs, sel)
        out.append(_case("A_" + tag, st, "luma DC category %d has a %d-bit code" % (common, _lens(dc0)[common])))
    co, _d = pil_coefs(264, 200, "420", 92, "noise", 8)
    fr = W.Frame(264, 200, S420)
    cnt = W.symbol_counts(fr, co, sel)
    tabs = dict(K)
    tabs[(1, 0)] = W.optimal_table(cnt[(1, 0)], maxlen=9)
    st = W.write_jpeg(264, 200, S420, co, tabs, sel)
    out.append(_case("A_ac_all_lut", st, "luma AC codes are at most %d bits" % max(l for l in range(17) if tabs[(1, 0)][0][l])))
    tabs = dict(K)
    bits, vals = W.reversed_table(cnt[(1, 0)])
    tabs[(1, 0)] = (bits, [v for v in vals if v not in (0x00, 0x01)] + [0x00, 0x01])   # the two longest codes
    ln = _lens(tabs[(1, 0)])
    st = W.write_jpeg(264, 200, S420, co, tabs, sel)
    out.append(_case("A_ac_long_common", st, "luma EOB %d bits, (0,1) %d bits" % (ln[0], ln[1])))
    # one-symbol tables: every block "DC difference 0, EOB", 1-bit codes
    one = {(0, 0): ([0, 1] + [0] * 15, [0]), (1, 0): ([0, 1] + [0] * 15, [0])}
    fr = W.Frame(512, 256, S420)
    st = W.write_jpeg(512, 256, S420, _zeros(fr), one, [(0, 0)] * 3)
    out.append(_case("A_one_symbol", st, "1-bit DC and AC tables of one symbol"))
    # an AC table that uses every length 1..16 (16 symbols, one of each length)
    rs = np.random.RandomState(11)
    alpha = [0x00, 0x01, 0x02, 0x11, 0x03, 0x21, 0x12, 0x04, 0x31, 0x05, 0x13, 0x41, 0x06, 0x22, 0x51, 0xF0]
    fr = W.Frame(120, 88, S420)
    co = [alphabet_blocks(rs, fr.blocks(c), alpha) for c in range(3)]
    tabs = dict(K)
    tabs[(1, 0)] = tabs[(1, 1)] = W.chain_table(alpha)
    st = W.write_jpeg(120, 88, S420, co, tabs, sel)
    out.append(_case("A_every_length", st, "AC code lengths 1..16, one symbol each"))
    return out


# ---- B: table selectors ---------------------------------------------------------------------------------------------
def cases_selectors():
    out = []
    co, _d = pil_coefs(264, 136, "420", 80, "smooth", 9)
    fr = W.Frame(264, 136, S420)
    for tag, sel in (("all_tables_0", [(0, 0)] * 3), ("chroma_dc0_ac1", [(0, 0), (0, 1), (0, 1)]),
                     ("chroma_dc1_ac0", [(0, 0), (1, 0), (1, 0)]), ("luma_tables_1", [(1, 1), (0, 0), (0, 0)])):
        tabs = W.optimal_tables(fr, co, sel)
        for k in [(0, 0), (0, 1), (1, 0), (1, 1)]:
            tabs.setdefault(k, K[k])   # a defined table the scan never selects
        st = W.write_jpeg(264, 136, S420, co, tabs, sel)
        out.append(_case("B_" + tag, st, "SOS selectors %s" % sel))
    tabs = W.optimal_tables(fr, co, [(0, 0)] * 3)
    bad = (1, 1, [0, 3] + [0] * 15, [1, 2, 3])   # three 1-bit codes: not a prefix code, and never selected
    st = W.write_jpeg(264, 136, S420, co, tabs, [(0, 0)] * 3, extra_dht=[bad])
    out.append(_case("B_unused_bogus_table", st, "AC table 1 has three 1-bit codes and no scan selects it"))
    return out


# ---- C: samplings ---------------------------------------------------------------------------------------------------
SAMPLINGS = {"440": S440, "411": S411, "410": S410, "422": S422}


def cases_samplings():
    out = []
    rs = np.random.RandomState(12)
    for tag, samp in SAMPLINGS.items():
        for w, h in ((37, 29), (101, 67)):
            for ri in (0, 3):
                fr = W.Frame(w, h, samp)
                co = [random_blocks(rs, fr.blocks(c), 6, 0.3) for c in range(3)]
                tabs = W.optimal_tables(fr, co, [(0, 0), (1, 1), (1, 1)], ri)
                st = W.write_jpeg(w, h, samp, co, tabs, restart=ri)
                dummies = sum(1 for _c, b in fr.scan_blocks() if b < 0)
                out.append(_case("C_%s_%dx%d_ri%d" % (tag, w, h, ri), st,
                                 "%d blocks per MCU, %d dummy blocks" % (fr.bpm, dummies)))
    return out


# ---- D: subsequence boundaries --------------------------------------------------------------------------------------
def split_lead(need, n):
    """need bits over n lead blocks -> n deltas that lead_block accepts"""
    reach, out = lead_deltas(), []
    for i in range(n):
        d = need if i == n - 1 else min(need, 600)
        while d not in reach or (i < n - 1 and need - d not in reach and need - d > 600 * (n - 1 - i)):
            d -= 1
        out.append(d)
        need -= d
    assert need == 0 and all(d in reach for d in out)
    return out


def _lead_420(co, fr, mcu, need):
    """spread `need` extra bits over the four luma blocks of MCU `mcu` (4:2:0)"""
    for i, d in enumerate(split_lead(need, 4)):
        by, bx = (mcu // fr.mpr) * 2 + i // 2, (mcu % fr.mpr) * 2 + i % 2
        co[0][by * fr.wb[0] + bx] = lead_block(d, co[0][by * fr.wb[0] + bx][0])


def _shifted(base_co, fr, delta):
    co = [c.copy() for c in base_co]
    _lead_420(co, fr, 0, delta)
    return W.write_jpeg(fr.width, fr.height, fr.samp, co, K)


def cases_boundaries():
    """a boundary (bit 1024 k) on every bit of one instance of each part of a symbol, and on an MCU's last bit"""
    out = []
    rs = np.random.RandomState(13)
    fr = W.Frame(96, 64, S420)
    co = [random_blocks(rs, fr.blocks(c), 30, 0.25, dc_amp=400) for c in range(3)]
    for c in range(3):   # a few zero runs of 16+ for ZRLs
        co[c][1::7, W.NATURAL[1:40]] = 0
        co[c][1::7, W.NATURAL[41]] = 3
    for b in (0, 1, fr.wb[0], fr.wb[0] + 1):   # MCU 0's luma blocks carry the lead
        co[0][b, 1:] = 0
    base = W.write_jpeg(96, 64, S420, co, K)
    first = [o for o, kind, s, _l, _n in base.syms if s == 4][0]   # symbols after the lead blocks move by delta
    targets = []
    for want in ("dc:code", "dc:mag", "ac:code", "ac:mag", "eob:code", "zrl:code", "mcu:last"):
        kind, part = want.split(":")
        for o, k, s, ln, nb in base.syms:
            if o < first + 64:
                continue
            if kind == "mcu" and k == "dc" and s % fr.bpm == 0 and s > 6:
                targets += [(want, 0, o - 1)]
                break
            if k == kind and (part == "code" or nb >= 5):
                span = range(ln) if part == "code" else range(ln, ln + nb)
                targets += [(want, j, o + j) for j in span]
                break
    for want, j, bit in targets:
        delta = (-bit) % W.SEQ_BITS
        st = _shifted(co, fr, delta)
        moved = bit + st.syms[[s for _o, _k, s, _l, _n in st.syms].index(4)][0] - first
        assert moved % W.SEQ_BITS == 0, (want, j)
        out.append(_case("D_%s_bit%d" % (want.replace(":", "_"), j), st,
                         "a subsequence boundary at bit %d of %s (clean bit %d)" % (j, want, moved)))
    return out


def cases_interval_lengths():
    """restart intervals whose coded length is n 1024 - 1, n 1024 and n 1024 + 1 bits, next to intervals that fit one
    subsequence; and a stream whose every interval fits one (no round runs)"""
    out = []
    fr = W.Frame(256, 64, S420)   # 16 x 4 MCUs
    ri = 8
    empty = W.write_jpeg(256, 64, S420, _zeros(fr), K, restart=ri)
    base_len = [max(o + l + n for o, k, s, l, n in empty.syms if s // (ri * 6) == iv) - empty.starts[iv] for iv in range(8)]
    for n in (1, 2):
        want = [n * 1024 - 1, 300, n * 1024, 500, n * 1024 + 1, n * 1024 + 7, n * 1024 + 8, 260]
        co = _zeros(fr)
        for iv in range(8):
            _lead_420(co, fr, iv * ri, want[iv] - base_len[iv])   # the interval's first MCU carries the extra bits
        st = W.write_jpeg(256, 64, S420, co, K, restart=ri)
        got = [max(o + l + nb for o, k, s, l, nb in st.syms if s // (ri * 6) == iv) - st.starts[iv] for iv in range(8)]
        assert got == want, (got, want)
        out.append(_case("D_interval_bits_n%d" % n, st, "interval coded lengths %s" % got))
    co = _zeros(fr)
    st = W.write_jpeg(256, 64, S420, co, K, restart=ri, fill=3)
    out.append(_case("D_every_interval_one_subsequence", st, "intervals of %s bits, 3 fill bytes before every RSTn"
                     % [st.starts[i + 1] - st.starts[i] for i in range(3)]))
    return out


# ---- E: convergence on flat frames ----------------------------------------------------------------------------------
def flat_frame(w, h, samp, lead, dc=-40, bars=None, seed=21):
    """a flat frame (every block "DC difference 0, EOB" after the first, whose AC content is lead_block(lead)); bars:
    (top, bottom) MCU rows of flat letterbox bars around noise content"""
    fr = W.Frame(w, h, samp)
    co = _zeros(fr)
    for c in range(fr.ncomp):
        co[c][:, 0] = dc if c == 0 else 0
    co[0][0] = lead_block(lead, dc)
    if bars:
        rs = np.random.RandomState(seed)
        for c in range(fr.ncomp):
            v, wb = fr.samp[c][1], fr.wb[c]
            r0, r1 = bars[0] * v, min(fr.hb[c], (fr.mrows - bars[1]) * v)
            co[c][r0 * wb:r1 * wb] = random_blocks(rs, (r1 - r0) * wb, 3, 0.1)
    return W.write_jpeg(w, h, samp, co, K)


def run_start(st, block):
    return [o for o, k, s, _l, _n in st.syms if s == block][0]


def orbit(ph, period):
    """the phases of the flat run at its successive subsequence boundaries (each 1024 bits on from the last)"""
    return sorted({int(ph + k * W.SEQ_BITS) % period for k in range(period)})


def lead_for_phase(samp, bad, period, dc=-40):
    """the smallest lead that makes the flat run (from MCU 1 on) meet a phase that never falls back into step at
    some subsequence boundary (bad), or at none of them -> (lead, phases at the boundaries)"""
    layout = "gray" if len(samp) == 1 else "444" if samp == S444 else "420"
    o0 = run_start(flat_frame(64, 64, samp, 0, dc), W.Frame(64, 64, samp).bpm)
    for lead in sorted(lead_deltas()):
        phases = orbit((W.SEQ_BITS - o0 - lead) % period, period)
        if any(p in FLAT_BAD[layout] for p in phases) == bad:
            return lead, phases


def cases_convergence(big=True):
    out = []
    for layout, samp, period in (("420", S420, 32), ("gray", GRAY, 6), ("444", S444, 14)):
        for bad in (False, True):
            if bad and not FLAT_BAD[layout]:
                continue
            lead, ph = lead_for_phase(samp, bad, period)
            st = flat_frame(1920, 1080, samp, lead)
            out.append(_case("E_flat_%s_1920x1080_%s" % (layout, "bad" if bad else "good"), st,
                             "flat run at boundary phases %s of %d; phases that never fall back into step: %s"
                             % (ph, period, FLAT_BAD[layout])))
    if big:
        for bad in (False, True):
            lead, ph = lead_for_phase(S420, bad, 32, dc=-128)
            st = flat_frame(3840, 2160, S420, lead, dc=-128)
            out.append(_case("E_black_420_3840x2160_%s" % ("bad" if bad else "good"), st,
                             "black frame, flat run at boundary phases %s" % ph))
    # letterbox: flat bars, content between them (the bars' phases are reported; the model gives the rounds)
    bars = (13, 14)
    st = flat_frame(1920, 1080, S420, 0, bars=bars)
    o_top = run_start(st, 6)
    o_bot = run_start(st, (st.frame.mrows - bars[1]) * st.frame.mpr * 6)
    lead = next(d for d in sorted(lead_deltas()) if (-o_top - d) % 32 in FLAT_BAD["420"] and (-o_bot - d) % 32 in FLAT_BAD["420"])
    st = flat_frame(1920, 1080, S420, lead, bars=bars)
    top, bottom = (-run_start(st, 6)) % 32, (-o_bot - lead) % 32
    out.append(_case("E_letterbox_420_1920x1080", st, "bars at phases %d and %d" % (top, bottom)))
    return out


# ---- F: large scans -------------------------------------------------------------------------------------------------
def cases_large():
    out = []
    rs = np.random.RandomState(31)
    fr = W.Frame(1000, 700, S420)
    co = [random_blocks(rs, fr.blocks(c), 4, 0.1) for c in range(3)]
    for c in range(3):
        co[c][:, 0] = np.where(np.arange(fr.blocks(c)) % 2, 1023, -1023)
    st = W.write_jpeg(1000, 700, S420, co, K)
    cats = [W._cat(int(d)) for d in np.diff(co[0][:, 0])]
    out.append(_case("F_dc_category11_1000x700", st, "%d luma blocks (not a multiple of 1024), DC differences of category %d"
                     % (fr.blocks(0), max(cats))))
    return out


# ---- G: IDCT --------------------------------------------------------------------------------------------------------
QUANTISERS = {"q1": ([1] * 64, False), "q255": ([255] * 64, False),
              "q16bit": ([int(v) for v in np.linspace(1, 1200, 64)], True)}


def idct_blocks(q, wide=False):
    """single-coefficient blocks: every position x both signs x magnitudes up to the category-10/11 limit, with
    |coefficient x quantiser| <= 2047, the most an encoder of 8-bit samples produces (beyond it libjpeg-turbo's SIMD
    IDCT, which scales the dequantised values by 4 in 16-bit lanes, wraps where the exact IDCT does not); then
    checkerboards of all 64 coefficients at the largest magnitude that stays inside those lanes.
    wide: the products libjpeg-turbo's SIMD IDCT cannot take, up to the 16-bit limit for single coefficients and
    2047 for checkerboards (checked against the C restatement's exact islow instead)"""
    cap, board = (32767, 2047) if wide else (2047, 256)
    q = np.asarray(q)
    blocks = []
    for pos in range(64):
        lim = min(2047 if pos == 0 else 1023, cap // int(q[pos]))
        for m in sorted({1, 2, max(1, lim // 7), max(1, lim // 2), lim}):
            for sgn in (1, -1):
                b = np.zeros(64, np.int64)
                b[pos] = sgn * m
                if pos == 0:
                    b[pos] = sgn * min(m, 1023)   # an absolute DC; the differences stay within category 11
                blocks.append(b)
    # all 64 products at once: kept at <= 256 (the q = 1 checkerboard), which libjpeg-turbo's 16-bit SIMD lanes hold
    lim = np.minimum(1023 if wide else 255, board // q)
    y, x = np.divmod(np.arange(64), 8)
    for sgn in (1, -1) if lim.min() > 0 else ():
        blocks.append(np.where((x + y) % 2 == 0, 1, -1) * lim * sgn)
    return np.array(blocks, np.int64)


def cases_idct(wide=False):
    out = []
    for i, (tag, (q, dqt16)) in enumerate(QUANTISERS.items()):
        b = idct_blocks(q, wide)
        for layout, samp in (("gray", GRAY), ("444", S444)):
            nb = len(b)
            wb = 40
            hb = -(-nb // wb)
            w, h = wb * 8 - (1 + i * 2 + (layout == "444")), hb * 8 - (3 + i * 2 + (layout == "444")) % 8
            fr = W.Frame(w, h, samp)
            co = []
            for c in range(fr.ncomp):
                a = np.zeros((fr.blocks(c), 64), np.int64)
                src = np.roll(b, c * 17, axis=0)
                k = min(len(src), len(a))
                a[:k] = src[:k]
                co.append(a)
            st = W.write_jpeg(w, h, samp, co, W.optimal_tables(fr, co, [(0, 0)] + [(1, 1)] * (fr.ncomp - 1)),
                              qt={0: q, 1: q}, dqt16=dqt16)
            out.append(_case("G_idct%s_%s_%s_%dx%d" % ("_wide" if wide else "", tag, layout, w, h), st,
                             "%d test blocks, quantiser max %d, widths %% 8 = %d, heights %% 8 = %d"
                             % (nb, max(q), w % 8, h % 8)))
    return out


# ---- H: colour conversion at tiny sizes -----------------------------------------------------------------------------
def cases_colour():
    out = []
    for tag, samp in (("422", S422), ("420", S420)):
        for w in (1, 2, 3, 4, 5):
            for h in (1, 2, 3):
                fr = W.Frame(w, h, samp)
                co = _zeros(fr)
                # luma and chroma blocks of the highest frequency at full scale with opposite DCs: every sample is
                # 0 or 255 in a checkerboard, so r, g and b saturate both ways
                chk = np.zeros(64, np.int64)
                chk[63] = 1023
                chk[0] = 0
                for c in range(3):
                    for b in range(fr.blocks(c)):
                        co[c][b] = chk * (1 if (b + c) % 2 == 0 else -1)
                        co[c][b][0] = [300, -300, 300][c]
                st = W.write_jpeg(w, h, samp, co, K)
                cw = -(-w // samp[0][0])
                out.append(_case("H_colour_%s_%dx%d" % (tag, w, h), st, "chroma width %d: %s" %
                                 (cw, "replicated" if cw <= 2 else "fancy upsampling")))
    return out


def all_cases(big=True):
    return (cases_tables() + cases_selectors() + cases_samplings() + cases_boundaries() + cases_interval_lengths()
            + cases_convergence(big) + cases_large() + cases_idct() + cases_colour())


# ---- I: a whole JPEG/R ----------------------------------------------------------------------------------------------
def jpegr_parts(lib, w, h, primary=None, map_lead=None):
    """the parts of a JPEG/R for API-4: a writer-made 4:2:0 primary (smooth Pillow coefficients under optimal tables,
    or `primary`), a flat single-channel gain map of w/4 x h/4 at a boundary phase that falls back into step (or at
    lead `map_lead`), and metadata from a library-encoded file -> (primary Stream, map Stream, metadata)"""
    import ctypes as C
    import uhdr_testlib as T
    from libultrahdr_b200 import ctypes_api as A
    from test_probe_cpu import _probe
    if primary is None:
        co, _d = pil_coefs(w, h, "420", 90, "smooth", 17)
        fr = W.Frame(w, h, S420)
        sel = [(0, 0), (1, 1), (1, 1)]
        primary = W.write_jpeg(w, h, S420, co, W.optimal_tables(fr, co, sel), sel)
    lead = lead_for_phase(GRAY, False, 6)[0] if map_lead is None else map_lead
    gm = flat_frame(w // 4, h // 4, GRAY, lead, dc=20)
    api = T.UhdrApi(lib)
    hb, sb = T.make_p010(64, 64, "smooth"), T.make_yuv420(64, 64, "smooth")
    hdr, _k1 = A.p010_image(hb, 64, 64, A.CG_BT2100, A.CT_HLG, A.CR_LIMITED)
    sdr, _k2 = A.yuv420_image(sb, 64, 64, A.CG_BT709)
    md = _probe(lib, api.encode(hdr, sdr, scale=4, multichannel=0))["md"]
    assert md is not None
    md.use_base_cg = 1   # the map is applied in the base image's space: a writer-made map carries no ICC profile
    return primary, gm, md

