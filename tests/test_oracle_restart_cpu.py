"""Pins the restart-interval handling of the CPU checker (oracle/jpeg_oracle.c jo_decode_coefs) to
libjpeg-turbo: streams that Pillow writes with a DRI marker and RSTn markers must decode to exactly
the planes Pillow's libjpeg-turbo decodes them to.  The GPU tests of restart-interval decoding
compare against this checker."""
import io

import numpy as np
import pytest

import uhdr_testlib as T

Image = pytest.importorskip("PIL.Image")

SUBSAMPLING = {"444": 0, "422": 1, "420": 2}


def pil_jpeg(a, quality, layout, **restart):
    b = io.BytesIO()
    if layout == "gray":
        Image.fromarray(a[:, :, 0]).save(b, "JPEG", quality=quality, **restart)
    else:
        Image.fromarray(a).save(b, "JPEG", quality=quality, subsampling=SUBSAMPLING[layout], **restart)
    return b.getvalue()


def image(w, h, kind, seed=7):
    if kind == "noise":
        return np.random.RandomState(seed).randint(0, 256, (h, w, 3)).astype(np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    return np.stack([(128 + 100 * np.sin(xx / 23.0 + k) * np.cos(yy / 17.0)) for k in range(3)], -1).astype(np.uint8)


def rst_count(data):
    s = data.index(b"\xff\xda")
    return sum(1 for i in range(s, len(data) - 1) if data[i] == 0xFF and 0xD0 <= data[i + 1] <= 0xD7)


@pytest.mark.parametrize("layout", ["gray", "420", "422", "444"])
@pytest.mark.parametrize("w,h", [(72, 34), (200, 97)])
def test_oracle_restart_decode_equals_libjpeg_turbo(oracle_libs, layout, w, h):
    o = oracle_libs.Oracle().lib
    for kind, q in (("noise", 100), ("smooth", 20)):
        a = image(w, h, kind)
        for restart in ({"restart_marker_blocks": 1}, {"restart_marker_blocks": 3}, {"restart_marker_rows": 1},
                        {"restart_marker_blocks": 5000}):
            data = pil_jpeg(a, q, layout, **restart)
            hd, planes = T.oracle_decode(o, data)
            assert hd.restart_interval > 0
            if "restart_marker_blocks" in restart and restart["restart_marker_blocks"] < 5000:
                assert rst_count(data) > 0
            im = Image.open(io.BytesIO(data))
            if layout != "gray":
                im.draft("YCbCr", None)
            px = np.asarray(im)
            if px.ndim == 2:
                px = px[:, :, None]
            assert (planes[0][:h, :w] == px[:, :, 0]).all(), (layout, kind, restart)
            if layout == "444":  # no chroma upsampling: every plane is comparable as it stands
                for c in (1, 2):
                    assert (planes[c][:h, :w] == px[:, :, c]).all(), (layout, kind, restart, c)
            # the same image without restart markers has the same coefficients
            _hd, plain = T.oracle_decode(o, pil_jpeg(a, q, layout))
            assert all((p == r).all() for p, r in zip(plain, planes)), (layout, kind, restart)
