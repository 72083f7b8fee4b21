"""The test stream writer (tests/jpeg_stream_writer.py) pinned on the CPU: byte-identical scans to Pillow's
libjpeg-turbo, every stream of the decoder routes file accepted by libjpeg-turbo without a warning, coefficients read
back by the C restatement, and the flat-frame phase table of the relaxation model."""
import ctypes as C

import numpy as np
import pytest

import jpeg_decode_cases as D
import jpeg_stream_writer as W
import scaled_testlib as S
import uhdr_testlib as T


def _coefs(data):
    lib = C.CDLL(T.ORACLE_SO)
    hd = T.JoHeader()
    buf = (C.c_uint8 * len(data)).from_buffer_copy(data)
    if lib.jo_read_header(buf, C.c_size_t(len(data)), C.byref(hd)) != 0:
        return None, None
    f = hd.frame
    co = [np.zeros((f.comp[c].wblocks * f.comp[c].hblocks, 64), np.int16) for c in range(f.ncomp)]
    cp = (C.c_void_p * 3)(*([a.ctypes.data for a in co] + [None] * (3 - f.ncomp)))
    assert lib.jo_decode_coefs(buf, C.c_size_t(len(data)), C.byref(hd), cp) == 0
    return hd, [a.astype(np.int64) for a in co]


@pytest.mark.parametrize("restart", [0, 5])
@pytest.mark.parametrize("optimize", [False, True])
@pytest.mark.parametrize("layout", ["gray", "444", "422", "420"])
def test_scan_identical_to_pillow(oracle_libs, layout, optimize, restart):
    """Pillow's stream -> its coefficients and tables -> the writer's scan is the same bytes"""
    for w, h, kind, q in ((67, 45, "noise", 90), (200, 121, "smooth", 40)):
        kw = {"optimize": optimize}
        if restart:
            kw["restart_marker_blocks"] = restart
        data = S.pil_jpeg(S.image(w, h, kind, seed=w), q, layout, **kw)
        hd, co = _coefs(data)
        f = hd.frame
        samp = [(f.comp[c].h_samp, f.comp[c].v_samp) for c in range(f.ncomp)]
        sel = [(hd.dc_sel[c], hd.ac_sel[c]) for c in range(f.ncomp)]
        st = W.write_jpeg(w, h, samp, co, W.read_tables(data), sel, restart=hd.restart_interval)
        _m, off = W.read_markers(data)
        assert hd.restart_interval == restart
        assert st.scan_data + b"\xff\xd9" == data[off:], (layout, optimize, restart, w, h)


@pytest.mark.parametrize("layout", ["gray", "444", "420"])
def test_optimal_tables_equal_libjpeg_turbos(oracle_libs, layout):
    """the tables the writer builds from a Pillow optimize=True stream's coefficients are that stream's own DHT"""
    for w, h, kind, q in ((67, 45, "noise", 90), (200, 121, "smooth", 40), (120, 88, "noise", 100)):
        data = S.pil_jpeg(S.image(w, h, kind, seed=w), q, layout, optimize=True)
        hd, co = _coefs(data)
        f = hd.frame
        samp = [(f.comp[c].h_samp, f.comp[c].v_samp) for c in range(f.ncomp)]
        sel = [(hd.dc_sel[c], hd.ac_sel[c]) for c in range(f.ncomp)]
        got = W.optimal_tables(W.Frame(w, h, samp), co, sel)
        assert got == W.read_tables(data), (layout, w, h)


def test_optimal_table_is_a_prefix_code_within_16_bits():
    rs = np.random.RandomState(1)
    for n in (1, 2, 12, 162, 256):
        freq = np.zeros(256, np.int64)
        freq[:n] = rs.zipf(1.3, n).clip(1, 10 ** 9)
        bits, vals = W.optimal_table(freq)
        assert sorted(vals) == list(range(n)) and sum(bits) == n
        assert sum(bits[ln] * 2.0 ** -ln for ln in range(1, 17)) < 1.0
        bits9, _v = W.optimal_table(freq, maxlen=9)
        assert not any(bits9[10:]) or n > 511


def test_flat_phase_table():
    """phases of a flat MCU ("DC difference 0, EOB" in every block, Annex K tables) from which a decoder started in the
    first-guess state never falls back into step"""
    k = W.annex_k()
    assert W.flat_phases(D.S420, k) == (32, [1, 2, 6, 9, 11, 13, 18, 20, 25, 28, 31])
    assert W.flat_phases(D.GRAY, k) == (6, [4])
    assert W.flat_phases(D.S444, k) == (14, [])


def test_relaxation_model_on_flat_frames():
    """lock-step rounds: a flat 4:2:0 run at a bad phase advances the true states one subsequence per round"""
    good = D.flat_frame(1920, 1080, D.S420, D.lead_for_phase(D.S420, False, 32)[0])
    bad = D.flat_frame(1920, 1080, D.S420, D.lead_for_phase(D.S420, True, 32)[0])
    rg, seqs, _c = W.relax_rounds(good)
    rb, _s, changed = W.relax_rounds(bad)
    assert rg <= 4 and len(seqs) == 256
    assert rb == 257 and all(len(c) == 1 for c in changed[2:-1])


@pytest.fixture(scope="module")
def all_cases(oracle_libs):
    if not S.have_harness():
        pytest.skip("no libjpeg-turbo harness")
    return D.all_cases()


def test_warning_count_reaches_the_tests(oracle_libs):
    """positive control of the check below: streams libjpeg-turbo decodes with a warning report it in info[15]"""
    if not S.have_harness():
        pytest.skip("no libjpeg-turbo harness")
    good = S.pil_jpeg(S.image(64, 48, "noise", seed=2), 90, "420")
    assert S.harness_decode(good, 1)[0][15] == 0
    _m, off = W.read_markers(good)
    cut = good[:off + (len(good) - off) // 2]   # entropy-coded data cut in half, no EOI: "premature end"
    for mode in (0, 1):
        assert S.harness_decode(cut, 1, mode)[0][15] >= 1, mode
    i = good.index(b"JFIF\x00")
    jfif3 = good[:i + 5] + b"\x03" + good[i + 6:]   # JFIF major version 3: "unknown JFIF revision"
    assert S.harness_decode(jfif3, 1)[0][15] >= 1


def test_libjpeg_turbo_decodes_every_stream_without_warnings(all_cases):
    for name, st, _e in all_cases:
        data = st if isinstance(st, bytes) else st.data
        for mode in ((0, 1) if name.startswith(("H_", "A_", "B_")) else (0,)):
            info, _p = S.harness_decode(data, 1, mode)
            assert info[15] == 0, (name, mode, info[15])


def test_coefficients_read_back(all_cases):
    """where the C restatement parses the layout, it returns exactly the coefficients written"""
    n = 0
    for name, st, _e in all_cases:
        assert not isinstance(st, bytes), name
        if name.startswith(("C_440", "C_411", "C_410")):
            continue   # samplings the restatement does not parse
        hd, co = _coefs(st.data)
        assert hd is not None, name
        want = st.coefs
        for c in range(len(co)):
            assert (co[c] == want[c]).all(), (name, c)
        n += 1
    assert n > 50
