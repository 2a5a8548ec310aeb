"""The JPEG syntax other encoders write, on the host (no GPU): tests/jpeg_writer.py writes what it claims (Pillow opens
every valid case, encoded images lie within a stated PSNR of their source), dirb200_jpeg_parse's descriptor equals
what was written, and the accept / refuse table of tests/jpeg_syntax_cases.py holds.
tests/test_gpu_jpeg_syntax.py checks the device's pixels on the same cases."""
import io
import math

import numpy as np
import pytest

import jpeg_syntax_cases as S
import jpeg_writer as W

NAMES = [c.name for c in S.CASES]


def _desc(raw):
    import datasets as D
    rc, desc, intervals = D.parse_jpeg(raw)
    return rc, (desc.view(D.JPEG_DESC_DTYPE)[0] if rc == 0 else None), intervals


@pytest.mark.parametrize("name", NAMES)
def test_parse_result_is_the_tables(name):
    case = S.BY_NAME[name]
    rc, _, _ = _desc(case.raw)
    assert rc == case.rc, (name, rc, case.rc)
    assert case.features, name
    if case.rc == 0:
        assert case.device in ("exact", "flag")


def test_table_names_every_feature():
    """Every syntax feature the decoder's accept / refuse line depends on has at least one case."""
    text = " | ".join(f for c in S.CASES for f in c.features)
    for feature in ["colour: no JFIF", "Adobe transform 0", "Adobe transform 1", "IDs 'R' 'G' 'B'", "SOF1",
                    "16-bit DQT", "slots 2 and 3", "12-bit", "slow path", "DC category 11", "AC category 10", "ZRL",
                    "coefficient 63 without EOB", "DC predictor wrap-around", "outside int16",
                    "outside the range-limit", "DRI 1 MCU", "DRI not dividing", "DRI larger than the image",
                    "RSTn wraps", "fill 0xFF before RSTn", "pad bits 0", "RSTn out of sequence", "APP1 EXIF",
                    "COM", "APP2", "fill 0xFF before markers", "between SOF and SOS", "several tables in one",
                    "one table per segment", "redefined", "after the scan", "bytes after EOI", "4:4:0", "4:1:1",
                    "Y 2x2 with chroma 2x2", "non-interleaved multi-scan", "chroma width 1", "noise in MCU padding",
                    "16 x 4000", "1000 px"]:
        assert feature in text, feature
    # a >= 1000 px case for colour space, SOF1, long codes, restart intervals and marker walking
    big = [c.name for c in S.CASES if c.rc == 0 and max(c.written.frame.height, c.written.frame.width) >= 1000]
    assert len(big) >= 6, big
    # chroma widths 1, 2 and 3 in both subsamplings
    widths = {(c.written.frame.vmax, (c.written.frame.width + 1) // 2) for c in S.CASES
              if c.rc == 0 and c.name.startswith("edge_4")}
    assert {(v, cw) for v in (1, 2) for cw in (1, 2, 3)} <= widths


@pytest.mark.parametrize("name", [c.name for c in S.CASES if c.pillow_opens])
def test_pillow_opens_what_the_writer_wrote(name):
    case = S.BY_NAME[name]
    got = S.pillow_rgb(case.raw)
    if case.source is None:
        return
    src = case.source()
    assert got.shape[:2] == src.shape[:2]
    if case.psnr:
        src = np.repeat(src[..., None], 3, -1) if src.ndim == 2 else src
        mse = ((got.astype(np.float64) - src) ** 2).mean()
        assert 10 * math.log10(255 ** 2 / max(mse, 1e-12)) >= case.psnr, name


def test_pillow_refuses_what_no_decoder_accepts():
    for c in S.CASES:
        if not c.pillow_opens:
            with pytest.raises(Exception):
                S.pillow_rgb(c.raw)


@pytest.mark.parametrize("name", [c.name for c in S.CASES if c.rc == 0])
def test_descriptor_equals_what_was_written(name):
    from PIL import Image
    case = S.BY_NAME[name]
    written, frame = case.written, case.written.frame
    rc, d, intervals = _desc(case.raw)
    assert rc == 0
    im = Image.open(io.BytesIO(case.raw))
    assert [(c.id, c.h, c.v, c.tq) for c in frame.comps] == [tuple(layer) for layer in im.layer]
    assert (int(d["height"]), int(d["width"]), int(d["ncomp"])) == (frame.height, frame.width, len(frame.comps))
    assert (int(d["hmax"]), int(d["vmax"])) == (frame.hmax, frame.vmax)
    mx, my = frame.mcus(frame.comps)
    assert (int(d["mcus_x"]), int(d["mcus_y"])) == (mx, my)
    for i, c in enumerate(frame.comps):
        got = tuple(int(d[k][i]) for k in ("comp_h", "comp_v", "comp_tq", "comp_td", "comp_ta"))
        assert got == (c.h, c.v, c.tq, c.td, c.ta), (i, got)
        # the table in force in the component's slot, natural order (Pillow reads the same one)
        assert list(d["qt"][c.tq]) == list(written.qtables[c.tq]) == list(im.quantization[c.tq])
        for cls, slot in ((0, c.td), (1, c.ta)):
            bits, vals = written.huff[(cls, slot)]
            assert list(d["huff_bits"][cls][slot]) == list(bits)
            assert list(d["huff_vals"][cls][slot][:len(vals)]) == list(vals)
            assert not d["huff_vals"][cls][slot][len(vals):].any()
    ri = int(d["restart_interval"])
    assert ri == written.restart
    assert int(d["n_intervals"]) == (math.ceil(mx * my / ri) if ri else 1) == len(written.interval_starts)
    assert intervals.tolist() == written.interval_starts
    assert (int(d["scan_begin"]), int(d["scan_end"])) == (written.scan_begin, written.scan_end)


def test_writer_huffman_tables_reach_16_bits_and_limit_lengths():
    """table_from_frequencies: a prefix code (Kraft sum below 1, no all-ones code) whose lengths reach max_len for
    skewed frequencies and never pass it."""
    freq = {s: 2 ** (s % 20) for s in range(40)}
    for max_len in (9, 12, 16):
        bits, vals = W.table_from_frequencies(freq, max_len)
        assert sorted(vals) == list(range(40)) and sum(bits) == 40
        assert max(l + 1 for l in range(16) if bits[l]) == max_len
        assert sum(b * 2.0 ** -(l + 1) for l, b in enumerate(bits)) < 1
    codes = W.code_table(*W.table_from_frequencies(freq, 16))
    words = sorted(format(c, f"0{n}b") for c, n in codes.values())
    assert not any(b.startswith(a) for a, b in zip(words, words[1:]))
