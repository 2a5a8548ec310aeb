"""The JPEG syntax case table of the device decoder's tests: files that tests/jpeg_writer.py writes, each with what
dirb200_jpeg_parse must return for it and what the device decode must do with it.

rc: 0 (in the supported set), UNSUPPORTED (decoded on the host) or MALFORMED.
device (rc 0 only): "exact" -- status 0 and byte for byte Pillow's image; "flag" -- a status bit set, so that the
host decodes it.
features: the T.81 / libjpeg features the case exercises (the table names each at least once).
"""
import functools
import io
from dataclasses import dataclass

import numpy as np

import jpeg_cases as J
import jpeg_writer as W

UNSUPPORTED, MALFORMED = 1, -4


@dataclass
class Case:
    name: str
    build: object                       # () -> jpeg_writer.Written
    rc: int = 0
    device: str = "exact"
    features: tuple = ()
    source: object = None               # () -> the 8-bit image the file encodes, for the PSNR check
    psnr: float = 0.0                   # Pillow's decode lies within this PSNR (dB) of `source`
    pillow_opens: bool = True

    @functools.cached_property
    def written(self):
        return self.build()

    @property
    def raw(self):
        return self.written.raw


def ycc(h, w, sampling=(1, 1), ids=(1, 2, 3), tq=(0, 1, 1), td=(0, 1, 1), ta=(0, 1, 1), chroma=(1, 1)):
    hy, vy = sampling
    comps = [W.Comp(ids[0], hy, vy, tq[0], td[0], ta[0])]
    comps += [W.Comp(ids[i], chroma[0], chroma[1], tq[i], td[i], ta[i]) for i in (1, 2)]
    return W.Frame(h, w, comps)


def gray(h, w, id=1, tq=0, td=0, ta=0, hv=(1, 1)):
    return W.Frame(h, w, [W.Comp(id, hv[0], hv[1], tq, td, ta)])


QT = {0: W.scaled_qtable(90), 1: W.scaled_qtable(90, chroma=True)}


def image(kind, h, w, seed, is_gray=False):
    return J.content(kind, h, w, seed, gray=is_gray)


def from_image(frame, kind="smooth", seed=0, qtables=QT, pad="edge", multiscan=False, **kw):
    """(build, source) of a file encoding a seeded image with the given frame and encode() options."""
    is_gray = len(frame.comps) == 1
    src = functools.partial(image, kind, frame.height, frame.width, seed, is_gray)

    def build():
        coefs = W.quantise(src(), frame, qtables, pad=pad, seed=seed, multiscan=multiscan)
        return W.encode(frame, coefs, qtables, **kw)
    return build, src


# psnr=0: the file's samples are YCbCr but its markers say RGB, so Pillow's image is not the source
def image_case(name, frame, features, kind="smooth", seed=0, psnr=30.0, rc=0, device="exact", qtables=QT,
               pad="edge", multiscan=False, pillow_opens=True, **kw):
    build, src = from_image(frame, kind, seed, qtables, pad, multiscan, **kw)
    return Case(name, build, rc, device if rc == 0 else None, tuple(features), src,
                psnr if kind == "smooth" and pillow_opens else 0.0, pillow_opens)


def _blocks(frame, fn):
    """Raw coefficient blocks: fn(component index, block y, block x) -> 64 natural-order values."""
    out = []
    for i, c in enumerate(frame.comps):
        bw, bh = frame.comp_blocks(c)
        out.append(np.array([[fn(i, y, x) for x in range(bw)] for y in range(bh)], np.int64).reshape(bh, bw, 64))
    return out


def raw_case(name, frame, fn, qtables, features, rc=0, device="exact", **kw):
    return Case(name, lambda: W.encode(frame, _blocks(frame, fn), qtables, **kw), rc, device, tuple(features))


def _syntax_block(i, y, x):
    """DC differences of +-2047 (category 11), AC +-1023 (category 10), a 20-zero run (ZRL), and a non-zero
    coefficient 63 (no EOB); the samples stay within what the range limit reproduces."""
    b = np.zeros(64, np.int64)
    b[0] = -1024 if (x + y + i) % 2 == 0 else 1023
    zz = W.ZIGZAG
    b[zz[1 + (x % 3)]] = 1023 if y % 2 else -1023
    b[zz[25]] = -200 + 13 * x
    b[zz[63]] = 1 + (x % 2)
    return b


def _dc_wrap(bw, restart=0):
    """Every block's DC difference +2047 (grayscale, bw blocks per row): the predictor passes 32767, and the
    coefficient it gives wraps in JCOEF (int16).  The written values are the unwrapped sums."""
    def fn(i, y, x):
        m = y * bw + x
        b = np.zeros(64, np.int64)
        b[0] = 2047 * (1 + (m % restart if restart else m))
        return b
    return fn


def _overflow_block(i, y, x):
    """Dequantised values outside int16 (coefficient x 16-bit quantiser)."""
    b = np.zeros(64, np.int64)
    b[0] = 3 - (x % 7)
    b[W.ZIGZAG[1 + x % 5]] = (x % 3) - 1
    return b


def _range_block(i, y, x):
    """In int16 after dequantisation, but samples far outside what the range-limit table reproduces: the C IDCT wraps
    them (index & 0x3FF), SIMD saturates."""
    b = np.zeros(64, np.int64)
    b[0] = 1016 if x % 2 else -1024
    for k in range(1, 6):
        b[W.ZIGZAG[k]] = 1023 if (x + k) % 2 else -1023
    return b


def _thumbnail():
    return J.case("noise", 12, 10, "420", seed=7)


def _rgb_ids_frame(h, w):
    return ycc(h, w, ids=(ord("R"), ord("G"), ord("B")))


def _redefinition(h, w):
    """DQT and DHT segments that define slot 0 / 1 twice: the last definition before SOS is the one in force."""
    frame = ycc(h, w, sampling=(2, 2))
    src = functools.partial(image, "smooth", h, w, 4)
    decoy_q = W.flat_qtable(77)

    def build():
        coefs = W.quantise(src(), frame, QT)
        first = W.encode(frame, coefs, QT)
        huff = first.huff
        decoy_h = W.table_from_frequencies({s: 1 for s in range(12)}, 16)
        dqts = [W.dqt((0, decoy_q, 0), (1, decoy_q, 0)), W.dqt((0, QT[0], 0)), W.dqt((1, QT[1], 0))]
        dhts = [W.dht((0, 0, *decoy_h), (0, 1, *decoy_h)),
                W.dht(*[(c, s, b, v) for (c, s), (b, v) in sorted(huff.items())])]
        return W.encode(frame, coefs, QT, huff, dqt_segments=dqts, dht_segments=dhts)
    return build, src


def _split_tables(h, w):
    """Every table in its own DQT / DHT segment, the DHT segments between SOF and SOS after a DRI-less COM."""
    frame = ycc(h, w, sampling=(2, 1))
    src = functools.partial(image, "smooth", h, w, 5)

    def build():
        coefs = W.quantise(src(), frame, QT)
        huff = W.encode(frame, coefs, QT).huff
        return W.encode(frame, coefs, QT, huff, dqt_segments=[W.dqt((s, q, 0)) for s, q in sorted(QT.items())],
                        dht_segments=[W.dht((c, s, b, v)) for (c, s), (b, v) in sorted(huff.items())])
    return build, src


def _sof1_slots(h, w, q16):
    """SOF1 with every table in slots 2 and 3, optionally 16-bit DQT with values above 255."""
    frame = ycc(h, w, sampling=(2, 2), tq=(2, 3, 3), td=(3, 2, 2), ta=(2, 3, 3))
    qt = {2: W.scaled_qtable(70) * (3 if q16 else 1), 3: W.scaled_qtable(70, chroma=True) * (5 if q16 else 1)}
    src = functools.partial(image, "smooth", h, w, 6)

    def build():
        return W.encode(frame, W.quantise(src(), frame, qt), qt, sof_marker=0xC1, q16=q16)
    return build, src


def _nonint_multiscan(h, w):
    frame = ycc(h, w, sampling=(2, 2))
    src = functools.partial(image, "smooth", h, w, 8)

    def build():
        coefs = W.quantise(src(), frame, QT, multiscan=True)
        return W.encode(frame, coefs, QT, scans=[[c] for c in frame.comps])
    return build, src


def _rst_out_of_sequence(h, w):
    build, _ = from_image(ycc(h, w), restart=2)

    def bad():
        wr = build()
        p = wr.interval_starts[2] - 1                  # the second RSTn's code: D1 -> D3
        raw = bytearray(wr.raw)
        assert raw[p] == 0xD1
        raw[p] = 0xD3
        wr.raw = bytes(raw)
        return wr
    return bad


def _case_list():
    C = []
    add = C.append
    # ---------------------------------------------------------------- colour space (default_decompress_parms)
    add(image_case("no_jfif_ids_123", ycc(37, 45, (2, 2)), ["colour: no JFIF, IDs 1 2 3 -> YCbCr"], head=[]))
    add(image_case("no_jfif_ids_012", ycc(40, 33, (2, 1), ids=(0, 1, 2)), ["colour: no JFIF, other IDs -> YCbCr"],
                   head=[]))
    add(image_case("no_jfif_ids_abc", ycc(19, 26, ids=(ord("a"), ord("b"), ord("c"))),
                   ["colour: no JFIF, other IDs -> YCbCr"], head=[]))
    add(image_case("adobe_transform1", ycc(33, 35, (2, 2)), ["colour: Adobe transform 1 -> YCbCr"],
                   head=[W.adobe(1)]))
    add(image_case("adobe_transform2_3comp", ycc(24, 30), ["colour: Adobe transform 2 on 3 components -> YCbCr"],
                   head=[W.adobe(2)]))
    add(image_case("jfif_and_adobe0", ycc(30, 24, (2, 1)), ["colour: JFIF wins over Adobe transform 0"],
                   head=[W.jfif(), W.adobe(0)]))
    add(image_case("jfif_rgb_ids", _rgb_ids_frame(21, 27), ["colour: JFIF wins over IDs 'R' 'G' 'B'"]))
    add(image_case("adobe1_rgb_ids", _rgb_ids_frame(21, 27), ["colour: Adobe transform 1 wins over IDs 'R' 'G' 'B'"],
                   head=[W.adobe(1)]))
    add(image_case("adobe_transform0", ycc(20, 20), ["colour: Adobe transform 0 without JFIF -> RGB"],
                   rc=UNSUPPORTED, psnr=0, head=[W.adobe(0)]))
    add(image_case("rgb_ids_no_marker", _rgb_ids_frame(20, 20), ["colour: IDs 'R' 'G' 'B' without markers -> RGB"],
                   rc=UNSUPPORTED, psnr=0, head=[]))
    add(image_case("adobe_transform0_after_app1", ycc(20, 20), ["colour: Adobe transform 0 after EXIF -> RGB"],
                   rc=UNSUPPORTED, psnr=0, head=[W.exif_with_thumbnail(_thumbnail()), W.adobe(0)]))
    add(image_case("no_jfif_large", ycc(1000, 1200, (2, 2)), ["colour: no JFIF at 1000 px"], head=[]))
    # ---------------------------------------------------------------- SOF1: 16-bit DQT, table slots 2 and 3
    b, s = _sof1_slots(48, 56, q16=False)
    add(Case("sof1_slots_2_3", b, features=("SOF1", "Huffman and DQT slots 2 and 3"), source=s, psnr=28))
    b, s = _sof1_slots(48, 56, q16=True)
    add(Case("sof1_q16_slots_2_3", b, features=("SOF1", "16-bit DQT above 255", "slots 2 and 3"), source=s,
             psnr=20))
    b, s = _sof1_slots(1000, 1008, q16=True)
    add(Case("sof1_q16_large", b, features=("SOF1 16-bit DQT at 1000 px",), source=s, psnr=20))
    add(image_case("sof1_12bit", gray(16, 16), ["SOF1 12-bit samples"], rc=UNSUPPORTED, precision=12,
                   sof_marker=0xC1, pillow_opens=False))
    add(image_case("gray_q16", gray(41, 23), ["16-bit DQT, grayscale"], q16=True,
                   qtables={0: W.scaled_qtable(40) * 7}, psnr=20))
    # ---------------------------------------------------------------- Huffman: codes longer than the 9-bit lookahead
    add(image_case("long_codes_16", ycc(64, 72, (2, 2)), ["Huffman codes of 10 - 16 bits (slow path)"],
                   kind="noise", max_len=16, qtables={0: W.flat_qtable(1), 1: W.flat_qtable(2)}))
    add(image_case("long_codes_gray", gray(50, 70), ["Huffman codes of 10 - 16 bits (slow path)"], kind="noise",
                   max_len=16, qtables={0: W.flat_qtable(1)}))
    add(image_case("short_codes_9", ycc(40, 40), ["Huffman codes of at most 9 bits"], kind="noise", max_len=9,
                   qtables={0: W.flat_qtable(3), 1: W.flat_qtable(3)}))
    add(image_case("long_codes_large", ycc(1000, 1000, (2, 1)), ["slow path at 1000 px"], kind="noise", max_len=16,
                   qtables={0: W.flat_qtable(1), 1: W.flat_qtable(1)}))
    # ---------------------------------------------------------------- raw coefficients
    add(raw_case("raw_categories", ycc(24, 40), _syntax_block, {0: W.flat_qtable(1), 1: W.flat_qtable(1)},
                 ["DC category 11", "AC category 10", "ZRL", "coefficient 63 without EOB"]))
    add(raw_case("raw_categories_gray", gray(16, 64), _syntax_block, {0: W.flat_qtable(1)},
                 ["DC category 11", "AC category 10", "ZRL", "coefficient 63 without EOB"]))
    add(raw_case("raw_dc_wrap", gray(8, 8 * 40), _dc_wrap(40), {0: W.flat_qtable(1)},
                 ["DC predictor wrap-around (repeated +2047)"], device="flag"))
    add(raw_case("raw_dc_wrap_restart", gray(16, 8 * 40), _dc_wrap(40, 17), {0: W.flat_qtable(1)},
                 ["DC predictor wrap-around, reset by restart markers"], device="flag", restart=17))
    add(raw_case("raw_q16_overflow", ycc(16, 64), _overflow_block,
                 {0: np.full(64, 32767), 1: np.full(64, 12000)}, ["dequantised values outside int16"],
                 device="flag", q16=True, sof_marker=0xC1))
    add(raw_case("raw_range_overflow", gray(8, 64), _range_block, {0: W.flat_qtable(1)},
                 ["IDCT output outside the range-limit table"], device="flag"))
    # ---------------------------------------------------------------- restart intervals
    add(image_case("dri_1", ycc(24, 40, (2, 1)), ["DRI 1 MCU"], restart=1))
    add(image_case("dri_7_of_5_per_row", ycc(40, 40, (2, 2)), ["DRI not dividing an MCU row"], restart=7))
    add(image_case("dri_larger_than_image", ycc(24, 24), ["DRI larger than the image"], restart=500))
    add(image_case("dri_wraps_rst7", gray(40, 56), ["more than 8 intervals (RSTn wraps)"], restart=2))
    add(image_case("rst_after_fill", ycc(32, 48, (2, 2)), ["fill 0xFF before RSTn"], restart=2, rst_fill=3))
    add(image_case("pad_bits_zero", ycc(32, 40), ["pad bits 0 before RSTn and EOI"], kind="noise", restart=3,
                   pad_bit=0))
    add(image_case("dri_large", ycc(1016, 1000, (2, 2)), ["restart intervals at 1000 px"], restart=11, rst_fill=1))
    add(Case("rst_out_of_sequence", _rst_out_of_sequence(24, 40), MALFORMED, None, ("RSTn out of sequence",)))
    # ---------------------------------------------------------------- marker walking
    add(image_case("exif_thumbnail", ycc(30, 44, (2, 2)), ["APP1 EXIF holding a JPEG thumbnail (SOI ... EOI)"],
                   head=[W.exif_with_thumbnail(_thumbnail())]))
    add(image_case("app1_com_app2", ycc(26, 34, (2, 1)), ["APP1, COM, APP2 before the frame"],
                   head=[W.jfif(), W.exif_with_thumbnail(_thumbnail()), W.com(b"a comment \xff\xd9"),
                         W.app(2, b"ICC_PROFILE\x00\x01\x01" + bytes(range(256)))]))
    add(image_case("fill_before_markers", ycc(22, 30, (2, 2)), ["fill 0xFF before markers"],
                   head=[W.jfif(fill=2), W.com(b"x", fill=5)], pre_sof=[W.app(5, b"app5", fill=1)]))
    add(image_case("tables_after_sof", ycc(25, 31, (2, 2)), ["DQT / DHT between SOF and SOS"],
                   mid=[W.com(b"between"), W.dqt((3, W.flat_qtable(9), 0))]))
    b, s = _split_tables(27, 35)
    add(Case("one_table_per_segment", b, features=("DQT / DHT one table per segment",), source=s, psnr=30))
    b, s = _redefinition(36, 28)
    add(Case("redefined_tables", b, features=("redefined DQT / DHT: the last before SOS wins",
                                             "several tables in one DQT / DHT segment"), source=s, psnr=30))
    add(image_case("marker_after_scan", ycc(20, 28), ["COM and APP after the scan"],
                   after_scan=[W.com(b"after"), W.app(3, b"late")]))
    add(image_case("bytes_after_eoi", ycc(20, 28), ["bytes after EOI"], trailing=b"\x00\x01garbage\xff\xd8\xff"))
    add(image_case("exif_large", ycc(1000, 1003, (2, 1)), ["EXIF / COM at 1000 px"],
                   head=[W.exif_with_thumbnail(_thumbnail()), W.com(b"c")]))
    # ---------------------------------------------------------------- refused sampling and scans
    add(image_case("sampling_440", ycc(32, 32, (1, 2)), ["4:4:0"], rc=UNSUPPORTED))
    add(image_case("sampling_411", ycc(32, 64, (4, 1)), ["4:1:1"], rc=UNSUPPORTED, psnr=25))
    # 12 blocks per MCU: T.81 allows 10, and libjpeg refuses it too
    add(image_case("y22_c22", ycc(32, 32, (2, 2), chroma=(2, 2)), ["Y 2x2 with chroma 2x2"], rc=UNSUPPORTED,
                   pillow_opens=False))
    add(image_case("y22_c21", ycc(32, 32, (2, 2), chroma=(2, 1)), ["Y 2x2 with chroma 2x1"], rc=UNSUPPORTED))
    add(image_case("gray_2x2", gray(24, 24, hv=(2, 2)), ["grayscale with sampling 2x2"], rc=UNSUPPORTED))
    b, s = _nonint_multiscan(32, 40)
    add(Case("non_interleaved_3_scans", b, UNSUPPORTED, None, ("non-interleaved multi-scan baseline",), s, 30))
    # ---------------------------------------------------------------- chroma edges, non-replicated MCU padding
    for sampling in ((2, 1), (2, 2)):
        tag = "422" if sampling == (2, 1) else "420"
        for (h, w) in [(1, 1), (1, 2), (2, 3), (3, 4), (5, 5), (8, 6), (9, 17), (16, 16), (17, 18), (18, 9),
                       (4, 1), (18, 18)]:
            add(image_case(f"edge_{tag}_{h}x{w}", ycc(h, w, sampling), [f"{tag}: chroma width 1 - 3, MCU padding"],
                           kind="noise", seed=h * 31 + w, pad="noise"))
    add(image_case("edge_gray_noise_pad_13x11", gray(13, 11), ["grayscale, noise in MCU padding"], kind="noise",
                   pad="noise"))
    add(image_case("aspect_16x4000", ycc(16, 4000, (2, 2)), ["extreme aspect ratio 16 x 4000"], pad="noise",
                   restart=33))
    add(image_case("aspect_4000x16", ycc(4000, 16, (2, 1)), ["extreme aspect ratio 4000 x 16"], pad="noise"))
    return C


CASES = _case_list()
BY_NAME = {c.name: c for c in CASES}
assert len(BY_NAME) == len(CASES)


def pillow_rgb(raw):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(raw)).convert("RGB"))
