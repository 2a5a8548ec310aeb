"""CPU half of the device JPEG decode: dirb200_jpeg_parse (host code, no CUDA call) on files Pillow writes from seeded
arrays, its refusals, AgeDB(device_decode=True) and jpeg_collate.  tests/test_gpu_jpeg_decode.py checks the pixels."""
import io
import math

import numpy as np
import pytest
import torch

import jpeg_cases as J


def _desc(raw):
    import datasets as D
    rc, desc, intervals = D.parse_jpeg(raw)
    return rc, (desc.view(D.JPEG_DESC_DTYPE)[0] if rc == 0 else None), intervals


def _restart_starts(raw, begin):
    """Byte offsets just after each RSTn marker of the scan that starts at `begin` (an independent scan)."""
    out, p = [begin], begin
    while True:
        f = raw.index(b"\xff", p)
        q = f + 1
        while raw[q] == 0xFF:
            q += 1
        if raw[q] == 0:
            p = q + 1
        elif 0xD0 <= raw[q] <= 0xD7:
            out.append(q + 1)
            p = q + 1
        else:
            return out, f


@pytest.mark.parametrize("setting", sorted(J.SETTINGS))
@pytest.mark.parametrize("h,w", [(1, 1), (7, 9), (16, 16), (33, 31), (225, 224)])
def test_parse_reports_the_frame_tables_and_intervals(setting, h, w):
    from PIL import Image
    raw = J.case("noise", h, w, setting, seed=h * 1000 + w)
    rc, d, intervals = _desc(raw)
    assert rc == 0
    im = Image.open(io.BytesIO(raw))
    assert (int(d["height"]), int(d["width"])) == (h, w)
    assert int(d["ncomp"]) == len(im.layer)
    for c, (_, hs, vs, tq) in enumerate(im.layer):
        assert (int(d["comp_h"][c]), int(d["comp_v"][c]), int(d["comp_tq"][c])) == (hs, vs, tq)
    for tq, table in im.quantization.items():
        assert list(d["qt"][tq]) == list(table)                # both in natural order
    hmax, vmax = int(d["comp_h"].max() if d["ncomp"] == 3 else 1), int(d["comp_v"].max() if d["ncomp"] == 3 else 1)
    assert (int(d["hmax"]), int(d["vmax"])) == (hmax, vmax)
    mcus = math.ceil(w / (8 * hmax)) * math.ceil(h / (8 * vmax))
    assert (int(d["mcus_x"]), int(d["mcus_y"])) == (math.ceil(w / (8 * hmax)), math.ceil(h / (8 * vmax)))
    ri = int(d["restart_interval"])
    opts = J.SETTINGS[setting]
    if "restart_marker_blocks" in opts:
        assert ri == opts["restart_marker_blocks"]
    elif "restart_marker_rows" in opts:
        assert ri == opts["restart_marker_rows"] * int(d["mcus_x"])
    else:
        assert ri == 0
    assert int(d["n_intervals"]) == (math.ceil(mcus / ri) if ri else 1)
    starts, end = _restart_starts(raw, int(d["scan_begin"]))
    assert intervals.tolist() == starts and int(d["scan_end"]) == end
    assert raw[end:end + 2] == b"\xff\xd9"


def _pillow_bytes(arr, mode=None, fmt="JPEG", **opts):
    from PIL import Image
    im = Image.fromarray(arr)
    if mode:
        im = im.convert(mode)
    bio = io.BytesIO()
    im.save(bio, fmt, **opts)
    return bio.getvalue()


def test_parse_refuses_what_the_device_does_not_decode():
    arr = J.content("noise", 24, 40, 3)
    cases = {
        "progressive": _pillow_bytes(arr, progressive=True),
        "cmyk": _pillow_bytes(arr, mode="CMYK"),
        "rgb_coded": _pillow_bytes(arr, keep_rgb=True),
        "png": _pillow_bytes(arr, fmt="PNG"),
    }
    for name, raw in cases.items():
        rc, _, _ = _desc(raw)
        assert rc == 1, (name, rc)                             # DIRB200_JPEG_UNSUPPORTED
    # keep_rgb writes component IDs 'R', 'G', 'B' (and an Adobe marker): the RGB colour space
    raw = cases["rgb_coded"]
    sof = raw.index(b"\xff\xc0")
    assert raw[sof + 10] == ord("R") and raw[sof + 13] == ord("G") and raw[sof + 16] == ord("B")


def test_parse_returns_negative_for_every_truncation_and_a_bad_huffman_table():
    raw = J.case("smooth", 20, 28, "420", seed=5)
    assert _desc(raw)[0] == 0
    for k in range(len(raw)):
        assert _desc(raw[:k])[0] < 0, k
    # a DHT whose codes run out: two 1-bit codes use the all-ones code (libjpeg: JERR_BAD_HUFF_TABLE); the symbol
    # count is kept so that the segment still parses
    b = bytearray(raw)
    p = raw.index(b"\xff\xc4")
    bits = p + 5
    donor = next(i for i in range(16) if b[bits + i] >= 2)
    assert b[bits] == 0
    b[bits] += 2
    b[bits + donor] -= 2
    assert _desc(bytes(b))[0] < 0


def test_parse_refuses_null_pointers():
    import _lib
    desc = np.zeros(int(_lib.raw("dirb200_jpeg_desc_bytes")()), np.uint8)
    iv = np.zeros(4, np.int32)
    assert _lib.raw("dirb200_jpeg_parse")(None, 10, desc.ctypes.data_as(_lib.P), iv.ctypes.data_as(_lib.P), 4) == -1
    assert "null" in _lib.last_error()


def _write_dataset(tmp_path, files):
    import pandas as pd
    for name, raw in files.items():
        (tmp_path / name).write_bytes(raw)
    ages = [float(20 + 3 * i) for i in range(len(files))]
    return pd.DataFrame({"path": list(files), "age": ages, "split": ["train"] * len(files)})


def test_dataset_device_decode_returns_the_file_or_the_host_resized_image(tmp_path):
    import datasets as D
    arr = J.content("smooth", 50, 43, 1)
    files = {"a.jpg": J.encode(arr, quality=90), "b.png": _pillow_bytes(arr, fmt="PNG"),
             "c.jpg": _pillow_bytes(arr, progressive=True)}
    df = _write_dataset(tmp_path, files)
    dec = D.AgeDB(df=df, data_dir=str(tmp_path), img_size=32, device_decode=True)
    ref = D.AgeDB(df=df, data_dir=str(tmp_path), img_size=32, device_transform=True)
    assert dec.device_transform
    img, label, weight = dec[0]
    assert isinstance(img, D.EncodedJpeg) and img.raw == files["a.jpg"] and img.size == 32
    rc, desc, iv = D.parse_jpeg(files["a.jpg"])
    assert rc == 0 and np.array_equal(img.desc, desc) and np.array_equal(img.intervals, iv)
    assert img.hw == (50, 43)
    assert float(label[0]) == 20.0 and float(weight[0]) == 1.0
    for i in (1, 2):                                           # PNG and progressive JPEG: the device_transform sample
        got, want = dec[i][0], ref[i][0]
        assert got.dtype == torch.uint8 and torch.equal(got, want)


def test_jpeg_collate_keeps_batch_order(tmp_path):
    import datasets as D
    files = {}
    for i in range(6):
        arr = J.content("noise", 20 + i, 30 - i, i)
        files[f"{i}.{'png' if i % 3 == 1 else 'jpg'}"] = _pillow_bytes(arr, fmt="PNG") if i % 3 == 1 else J.encode(arr)
    df = _write_dataset(tmp_path, files)
    ds = D.AgeDB(df=df, data_dir=str(tmp_path), img_size=24, device_decode=True)
    items = [ds[i] for i in range(len(ds))]
    batch, labels, weights = D.jpeg_collate(items)
    assert isinstance(batch, D.JpegBatch) and batch.n == 6 and batch.size == 24
    assert batch.jpeg_pos == [0, 2, 3, 5] and batch.host_pos == [1, 4]
    assert labels.shape == (6, 1) and labels[:, 0].tolist() == list(df["age"].values)
    assert weights.shape == (6, 1)
    names = list(files)
    for j, pos in enumerate(batch.jpeg_pos):
        lo, hi = int(batch.offsets[j]), int(batch.offsets[j + 1])
        assert batch.data[lo:hi].numpy().tobytes() == files[names[pos]]
        h, w = batch.hw[j].tolist()
        assert int(batch.rgb_offsets[j + 1] - batch.rgb_offsets[j]) == h * w * 3
    assert torch.equal(batch.host[0], items[1][0]) and torch.equal(batch.host[1], items[4][0])
    assert batch.intervals.numel() == 4 and batch.decode_ws > 0 and batch.resize_ws > 0


def test_train_parser_accepts_device_decode():
    import train
    args = train.build_parser().parse_args(["--device_decode"])
    assert args.device_decode and not args.device_transform
    assert not train.build_parser().parse_args([]).device_decode
