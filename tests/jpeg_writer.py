"""A small baseline / extended-sequential (SOF0 / SOF1) Huffman JPEG writer for the device decoder's syntax tests,
written from ITU-T T.81.  It exists to produce the JPEG syntax other encoders write and Pillow's encoder never does:
files without JFIF, Adobe / EXIF / ICC / COM segments, arbitrary component IDs and table slots, 16-bit quantisation
tables, Huffman tables with codes up to 16 bits, restart intervals of any length, fill bytes, redefined tables,
non-replicated MCU padding, multi-scan files, and raw quantised coefficients outside what an FDCT of 8-bit samples
yields.

No FDCT accuracy is needed: the reference for each file is Pillow's decode of the same bytes.

Layout of a file: `encode()` returns the bytes and what was written (scan range, restart-interval starts) so that the
tests can compare dirb200_jpeg_parse's descriptor with it.
"""
import heapq
import math
from dataclasses import dataclass, field

import numpy as np

# zigzag index k -> natural (row-major) index, built from T.81 Figure A.6's diagonal walk
ZIGZAG = []
for _s in range(15):
    _cells = [(r, _s - r) for r in range(8) if 0 <= _s - r < 8]
    ZIGZAG += [r * 8 + c for r, c in (_cells if _s % 2 else _cells[::-1])]
ZIGZAG = np.array(ZIGZAG)

# orthonormal 8-point DCT-II basis: F = D @ f @ D.T is T.81's FDCT (A.3.3)
_u = np.arange(8)[:, None]
_x = np.arange(8)[None, :]
DCT = np.where(_u == 0, math.sqrt(1 / 8), math.sqrt(2 / 8)) * np.cos((2 * _x + 1) * _u * math.pi / 16)


# ------------------------------------------------------------------------------------------------ marker segments
def segment(marker, payload=b"", fill=0):
    """0xFF (plus `fill` extra 0xFF fill bytes), the marker code, then length + payload (none for SOI / EOI / RSTn)."""
    head = b"\xff" * (1 + fill) + bytes([marker])
    if marker in (0xD8, 0xD9) or 0xD0 <= marker <= 0xD7:
        return head + payload
    return head + (len(payload) + 2).to_bytes(2, "big") + payload


def jfif(fill=0):
    return segment(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00", fill)


def adobe(transform, fill=0):
    return segment(0xEE, b"Adobe\x00\x64\x00\x00\x00\x00" + bytes([transform]), fill)


def app(n, payload, fill=0):
    return segment(0xE0 + n, payload, fill)


def com(text, fill=0):
    return segment(0xFE, text, fill)


def exif_with_thumbnail(thumbnail):
    """APP1 'Exif' holding a minimal TIFF header and an embedded JPEG thumbnail (its own SOI ... EOI)."""
    tiff = b"MM\x00\x2a\x00\x00\x00\x08" + b"\x00\x00" + b"\x00\x00\x00\x00"
    return app(1, b"Exif\x00\x00" + tiff + thumbnail)


def dqt(*tables, fill=0):
    """tables: (slot, 64 values in natural order, precision 0 (8-bit) or 1 (16-bit)); one segment holds them all."""
    out = b""
    for slot, q, pq in tables:
        q = np.asarray(q).reshape(64)[ZIGZAG]
        out += bytes([(pq << 4) | slot]) + (q.astype(">u2").tobytes() if pq else q.astype(np.uint8).tobytes())
    return segment(0xDB, out, fill)


def dht(*tables, fill=0):
    """tables: (class 0 DC / 1 AC, slot, BITS [16], HUFFVAL); one segment holds them all."""
    out = b""
    for tc, th, bits, vals in tables:
        out += bytes([(tc << 4) | th]) + bytes(bits) + bytes(vals)
    return segment(0xC4, out, fill)


def dri(n, fill=0):
    return segment(0xDD, int(n).to_bytes(2, "big"), fill)


def sof(frame, marker=0xC0, precision=8, fill=0):
    p = bytes([precision]) + frame.height.to_bytes(2, "big") + frame.width.to_bytes(2, "big") + bytes([len(frame.comps)])
    for c in frame.comps:
        p += bytes([c.id, (c.h << 4) | c.v, c.tq])
    return segment(marker, p, fill)


def sos(comps, fill=0):
    p = bytes([len(comps)])
    for c in comps:
        p += bytes([c.id, (c.td << 4) | c.ta])
    return segment(0xDA, p + b"\x00\x3f\x00", fill)


# ------------------------------------------------------------------------------------------------ frame and blocks
@dataclass
class Comp:
    id: int
    h: int = 1
    v: int = 1
    tq: int = 0            # quantisation table slot
    td: int = 0            # DC Huffman table slot
    ta: int = 0            # AC Huffman table slot


@dataclass
class Frame:
    height: int
    width: int
    comps: list

    @property
    def hmax(self):
        return max(c.h for c in self.comps)

    @property
    def vmax(self):
        return max(c.v for c in self.comps)

    def mcus(self, scan):
        """(mcus_x, mcus_y) of a scan over the components `scan` (A.2.2 / A.2.3)."""
        if len(scan) == 1:
            bw, bh = self.comp_blocks(scan[0], interleaved=False)
            return bw, bh
        return math.ceil(self.width / (8 * self.hmax)), math.ceil(self.height / (8 * self.vmax))

    def comp_size(self, c):
        """The component's sample dimensions (A.1.1): (width, height)."""
        return math.ceil(self.width * c.h / self.hmax), math.ceil(self.height * c.v / self.vmax)

    def comp_blocks(self, c, interleaved=True):
        """Blocks the component holds (width, height): MCU-padded when interleaved."""
        if interleaved and len(self.comps) > 1:
            return (math.ceil(self.width / (8 * self.hmax)) * c.h, math.ceil(self.height / (8 * self.vmax)) * c.v)
        w, h = self.comp_size(c)
        return math.ceil(w / 8), math.ceil(h / 8)


def ycbcr(rgb):
    """JFIF's RGB -> YCbCr, float."""
    r, g, b = [rgb[..., i].astype(np.float64) for i in range(3)]
    return np.stack([0.299 * r + 0.587 * g + 0.114 * b,
                     -0.168736 * r - 0.331264 * g + 0.5 * b + 128,
                     0.5 * r - 0.418688 * g - 0.081312 * b + 128], -1)


def quantise(image, frame, qtables, pad="edge", seed=0, multiscan=False):
    """Quantised coefficient blocks [bh, bw, 64] (natural order) per component of an 8-bit image (H x W gray or
    H x W x 3 RGB, converted to YCbCr): box-filter downsampling, then the component plane padded to its blocks by
    edge replication (pad="edge", as libjpeg's encoder does) or with seeded noise (pad="noise"), the FDCT, rounding."""
    rng = np.random.RandomState(seed)
    planes = image[..., None].astype(np.float64) if image.ndim == 2 else ycbcr(image)
    out = []
    for i, c in enumerate(frame.comps):
        p = planes[..., i]
        fh, fv = frame.hmax // c.h, frame.vmax // c.v
        H, W = p.shape
        p = np.pad(p, ((0, -H % fv), (0, -W % fh)), mode="edge")
        p = p.reshape(p.shape[0] // fv, fv, p.shape[1] // fh, fh).mean(axis=(1, 3))
        cw, ch = frame.comp_size(c)
        p = p[:ch, :cw]
        bw, bh = frame.comp_blocks(c, interleaved=not multiscan)
        full = np.pad(p, ((0, bh * 8 - ch), (0, bw * 8 - cw)), mode="edge")
        if pad == "noise":
            noise = rng.uniform(0, 255, size=full.shape)
            inside = np.zeros(full.shape, bool)
            inside[:ch, :cw] = True
            full = np.where(inside, full, noise)
        blocks = full.reshape(bh, 8, bw, 8).transpose(0, 2, 1, 3) - 128.0
        coef = np.einsum("ux,abxy,vy->abuv", DCT, blocks, DCT)
        q = np.asarray(qtables[c.tq], np.float64).reshape(8, 8)
        out.append(np.round(coef / q).astype(np.int64).reshape(bh, bw, 64))
    return out


# ------------------------------------------------------------------------------------------------ Huffman coding
def dc_category(v):
    return int(abs(int(v))).bit_length()


def block_symbols(blk, pred):
    """The (symbol, extra-bits value, extra-bit count) sequence of one block (F.1.2): DC difference, then AC run /
    size symbols with ZRL and EOB.  blk: natural order; pred: the previous DC."""
    zz = [int(x) for x in np.asarray(blk).reshape(64)[ZIGZAG]]
    diff = zz[0] - pred
    s = dc_category(diff)
    out = [("dc", s, diff + (1 << s) - 1 if diff < 0 else diff, s)]
    run = 0
    last = max([k for k in range(1, 64) if zz[k]], default=0)
    for k in range(1, last + 1):
        if zz[k] == 0:
            run += 1
            continue
        while run > 15:
            out.append(("ac", 0xF0, 0, 0))
            run -= 16
        s = dc_category(zz[k])
        out.append(("ac", (run << 4) | s, zz[k] + (1 << s) - 1 if zz[k] < 0 else zz[k], s))
        run = 0
    if last < 63:
        out.append(("ac", 0x00, 0, 0))
    return out


def table_from_frequencies(freq, max_len=16):
    """BITS [16] and HUFFVAL of a Huffman code for the symbols of `freq` (symbol -> count), lengths limited to
    max_len with T.81 Annex K.2's procedure (Figures K.1 - K.3, a reserved symbol keeping the all-ones code free)."""
    syms = sorted(s for s, f in freq.items() if f > 0)
    if not syms:
        syms = [0]
    heap = [(freq.get(s, 1) or 1, i, [s]) for i, s in enumerate(syms)] + [(0, -1, [None])]
    heapq.heapify(heap)
    size = {s: 0 for s in syms}
    size[None] = 0
    tick = len(syms)
    while len(heap) > 1:
        f1, _, a = heapq.heappop(heap)
        f2, _, b = heapq.heappop(heap)
        for s in a + b:
            size[s] += 1
        heapq.heappush(heap, (f1 + f2, tick, a + b))
        tick += 1
    bits = [0] * 64
    for s, n in size.items():
        bits[max(n, 1)] += 1
    i = 63
    while i > max_len:                                  # Figure K.3: Adjust_BITS
        if bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
        else:
            i -= 1
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1                                        # the reserved symbol's code
    order = sorted(syms, key=lambda s: (size[s], s))
    return bits[1:17], order


def code_table(bits, vals):
    """symbol -> (code, length) of a BITS / HUFFVAL pair (T.81 Annex C)."""
    codes, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            codes[vals[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return codes


class BitWriter:
    def __init__(self):
        self.bits = []

    def put(self, value, n):
        if n:
            self.bits.append(format(value & ((1 << n) - 1), f"0{n}b"))

    def flush(self, pad_bit):
        """The bytes so far, the last one padded with pad_bit, with 0xFF stuffed as 0xFF 0x00."""
        s = "".join(self.bits)
        s += str(pad_bit) * (-len(s) % 8)
        self.bits = []
        raw = int(s, 2).to_bytes(len(s) // 8, "big") if s else b""
        return raw.replace(b"\xff", b"\xff\x00")


def scan_blocks(frame, scan, coefs):
    """The scan's blocks in coding order, grouped by MCU: lists of (component index, block)."""
    idx = [frame.comps.index(c) for c in scan]
    mx, my = frame.mcus(scan)
    for m in range(mx * my):
        y, x = divmod(m, mx)
        mcu = []
        for i in idx:
            c = frame.comps[i]
            if len(scan) == 1:
                mcu.append((i, coefs[i][y, x]))
            else:
                for v in range(c.v):
                    for h in range(c.h):
                        mcu.append((i, coefs[i][y * c.v + v, x * c.h + h]))
        yield mcu


def scan_frequencies(frame, scan, coefs, restart=0):
    """(DC counts, AC counts) per table slot of the scan's symbols."""
    freq = {0: {}, 1: {}}
    pred = {}
    for m, mcu in enumerate(scan_blocks(frame, scan, coefs)):
        if restart and m % restart == 0:
            pred = {}
        for i, blk in mcu:
            c = frame.comps[i]
            for cls, sym, _, _ in block_symbols(blk, pred.get(i, 0)):
                slot = c.td if cls == "dc" else c.ta
                d = freq[0 if cls == "dc" else 1].setdefault(slot, {})
                d[sym] = d.get(sym, 0) + 1
            pred[i] = int(blk[0])
    return freq


def entropy_code(frame, scan, coefs, huff, restart=0, pad_bit=1, rst_fill=0):
    """The entropy-coded segment of one scan: (bytes, offsets just after each RSTn marker within them).
    huff: {(class, slot): (BITS, HUFFVAL)}."""
    codes = {k: code_table(*v) for k, v in huff.items()}
    bw = BitWriter()
    out, starts = b"", []
    pred = {}
    mcus = list(scan_blocks(frame, scan, coefs))
    for m, mcu in enumerate(mcus):
        for i, blk in mcu:
            c = frame.comps[i]
            for cls, sym, extra, n in block_symbols(blk, pred.get(i, 0)):
                code, length = codes[(0, c.td) if cls == "dc" else (1, c.ta)][sym]
                bw.put(code, length)
                bw.put(extra, n)
            pred[i] = int(blk[0])
        if restart and (m + 1) % restart == 0 and m + 1 < len(mcus):
            out += bw.flush(pad_bit) + b"\xff" * (1 + rst_fill) + bytes([0xD0 + ((m + 1) // restart - 1) % 8])
            starts.append(len(out))
            pred = {}
    return out + bw.flush(pad_bit), starts


# ------------------------------------------------------------------------------------------------ whole files
@dataclass
class Written:
    raw: bytes
    scan_begin: int = -1             # first byte of the (first) scan's entropy-coded data
    scan_end: int = -1               # the 0xFF of the marker that ends it
    interval_starts: list = field(default_factory=list)
    huff: dict = field(default_factory=dict)          # {(class, slot): (BITS, HUFFVAL)} in force at the scan
    qtables: dict = field(default_factory=dict)       # slot -> 64 values (natural order) in force at the scan
    frame: object = None
    restart: int = 0


def encode(frame, coefs, qtables, huff=None, *, sof_marker=0xC0, precision=8, q16=False, restart=0, head=None,
           pre_sof=(), mid=(), after_scan=(), trailing=b"", pad_bit=1, rst_fill=0, scans=None, max_len=16,
           dqt_segments=None, dht_segments=None):
    """A complete file: SOI, `head` (default: the JFIF APP0), DQT, `pre_sof`, SOF, DHT, DRI, `mid`, then per scan
    SOS + entropy-coded data, `after_scan`, EOI, `trailing`.

    coefs: per component [bh, bw, 64] quantised blocks, natural order.  qtables: slot -> 64 values (natural order),
    written 16-bit if q16.  huff: {(class, slot): (BITS, HUFFVAL)}; missing tables are derived from the scan's symbol
    frequencies with codes up to max_len bits.  scans: lists of components (default: one interleaved scan of all).
    dqt_segments / dht_segments replace the default one-segment DQT / DHT (for split, repeated or redefined tables)."""
    scans = scans or [frame.comps]
    huff = dict(huff or {})
    freq = {}
    for scan in scans:
        for cls, counts in scan_frequencies(frame, scan, coefs, restart).items():
            for slot, f in counts.items():
                total = freq.setdefault((cls, slot), {})
                for sym, n in f.items():
                    total[sym] = total.get(sym, 0) + n
    for key, f in freq.items():
        if key not in huff:
            huff[key] = table_from_frequencies(f, max_len)
    if dqt_segments is None:
        dqt_segments = [dqt(*[(s, q, int(q16)) for s, q in sorted(qtables.items())])]
    if dht_segments is None:
        dht_segments = [dht(*[(c, s, b, v) for (c, s), (b, v) in sorted(huff.items())])]
    raw = segment(0xD8) + (jfif() if head is None else b"".join(head))
    raw += b"".join(dqt_segments) + b"".join(pre_sof) + sof(frame, sof_marker, precision)
    raw += b"".join(dht_segments) + (dri(restart) if restart else b"") + b"".join(mid)
    w = Written(b"")
    for scan in scans:
        raw += sos(scan)
        data, starts = entropy_code(frame, scan, coefs, huff, restart, pad_bit, rst_fill)
        if w.scan_begin < 0:
            w.scan_begin = len(raw)
            w.interval_starts = [len(raw)] + [len(raw) + s for s in starts]
            w.scan_end = len(raw) + len(data)
        raw += data
    raw += b"".join(after_scan) + segment(0xD9) + trailing
    w.raw = raw
    w.huff, w.qtables, w.frame, w.restart = huff, qtables, frame, restart
    return w


def flat_qtable(v):
    return np.full(64, v, np.int64)


def scaled_qtable(quality, chroma=False):
    """A smooth quantisation table (not libjpeg's): larger steps at higher frequencies, scaled by quality in 1..100."""
    u, v = np.meshgrid(np.arange(8), np.arange(8))
    base = 8 + 6 * (u + v) + (6 if chroma else 0)
    scale = 5000 / quality if quality < 50 else 200 - 2 * quality
    return np.clip((base * scale + 50) // 100, 1, 255).astype(np.int64).reshape(64)
