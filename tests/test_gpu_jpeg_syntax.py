"""The device JPEG decode (csrc/jpeg.cu) on the syntax other encoders write (tests/jpeg_syntax_cases.py): every case
the parser accepts is either byte for byte Pillow's image with status 0, or flagged by the device and then decoded
by Pillow -- in one launch mixed with Pillow-written files, one image per launch, and end to end through
AgeDB(device_decode=True) and a DataLoader."""
import numpy as np
import pytest
import torch

import jpeg_cases as J
import jpeg_syntax_cases as S

pytestmark = pytest.mark.gpu

ACCEPTED = [c for c in S.CASES if c.rc == 0]
EXACT = [c for c in ACCEPTED if c.device == "exact"]
FLAGGED = [c for c in ACCEPTED if c.device == "flag"]


def _pillow_written():
    return [J.case(kind, h, w, setting, seed=3) for (kind, h, w, setting) in
            [("noise", 33, 31, "420"), ("saturated", 16, 16, "444_q100"), ("smooth", 225, 224, "422"),
             ("noise", 7, 9, "gray"), ("smooth", 15, 17, "420_restart_rows")]]


def test_every_accepted_case_in_one_launch_with_pillow_written_files():
    pillow = _pillow_written()
    raws = []
    for i, c in enumerate(ACCEPTED):                     # accepted cases interleaved with Pillow's own files
        raws.append(c.raw)
        if i % 7 == 0:
            raws.append(pillow[(i // 7) % len(pillow)])
    got, status = J.device_decode(raws)
    by_raw = {c.raw: c for c in ACCEPTED}
    wrong, flags = [], []
    for k, raw in enumerate(raws):
        c = by_raw.get(raw)
        if c is None or c.device == "exact":
            if status[k] != 0 or not np.array_equal(got[k], S.pillow_rgb(raw)):
                wrong.append((c.name if c else "pillow", int(status[k])))
        elif status[k] == 0:
            flags.append(c.name)
    assert not wrong, wrong
    assert not flags, f"not flagged: {flags}"


@pytest.mark.parametrize("name", [c.name for c in ACCEPTED])
def test_each_accepted_case_alone(name):
    c = S.BY_NAME[name]
    got, status = J.device_decode([c.raw])
    if c.device == "exact":
        assert status[0] == 0
        assert np.array_equal(got[0], S.pillow_rgb(c.raw))
    else:
        assert status[0] != 0


@pytest.mark.parametrize("name", [c.name for c in FLAGGED])
def test_flagged_case_keeps_its_neighbours_and_ends_as_pillows_image(name, tmp_path):
    import datasets as D
    import pandas as pd
    from PIL import Image
    c = S.BY_NAME[name]
    neighbours = [S.BY_NAME["long_codes_16"].raw, S.BY_NAME["dri_7_of_5_per_row"].raw]
    got, status = J.device_decode([neighbours[0], c.raw, neighbours[1]])
    assert status[1] != 0 and status[0] == 0 and status[2] == 0
    assert np.array_equal(got[0], S.pillow_rgb(neighbours[0])) and np.array_equal(got[2], S.pillow_rgb(neighbours[1]))
    names = ["n0.jpg", "flagged.jpg", "n1.jpg"]
    for n, r in zip(names, [neighbours[0], c.raw, neighbours[1]]):
        (tmp_path / n).write_bytes(r)
    df = pd.DataFrame({"path": names, "age": [1.0, 2.0, 3.0], "split": ["train"] * 3})
    ds = D.AgeDB(df=df, data_dir=str(tmp_path), img_size=40, device_decode=True)
    ref = D.AgeDB(df=df, data_dir=str(tmp_path), img_size=40, device_transform=True)
    batch, _, _ = D.jpeg_collate([ds[i] for i in range(3)])
    out = batch.cuda().cpu()
    assert batch.flagged == [1]
    assert torch.equal(out[1], D.host_resize_u8(Image.open(tmp_path / "flagged.jpg").convert("RGB"), 40))
    for i in range(3):
        assert torch.equal(out[i], ref[i][0])


def test_dataset_device_decode_through_a_loader_equals_device_transform(tmp_path):
    """A few cases of each group end to end: AgeDB(device_decode=True) + DataLoader + jpeg_collate, then the device's
    decode and dirb200_resize_bilinear_u8, against AgeDB(device_transform=True)."""
    import datasets as D
    import pandas as pd
    from torch.utils.data import DataLoader
    names = ["no_jfif_ids_012", "adobe_transform1", "sof1_q16_slots_2_3", "long_codes_16", "raw_categories",
             "raw_q16_overflow", "dri_7_of_5_per_row", "rst_after_fill", "exif_thumbnail", "redefined_tables",
             "edge_420_2x3", "edge_422_1x1", "adobe_transform0", "sampling_440", "aspect_16x4000"]
    for n in names:
        (tmp_path / f"{n}.jpg").write_bytes(S.BY_NAME[n].raw)
    df = pd.DataFrame({"path": [f"{n}.jpg" for n in names], "age": [float(i) for i in range(len(names))],
                       "split": ["train"] * len(names)})
    for size in (32, 224):
        dec = D.AgeDB(df=df, data_dir=str(tmp_path), img_size=size, device_decode=True)
        ref = D.AgeDB(df=df, data_dir=str(tmp_path), img_size=size, device_transform=True)
        want = torch.stack([ref[i][0] for i in range(len(ref))]).cuda()
        loader = DataLoader(dec, batch_size=len(dec), shuffle=False, num_workers=2, collate_fn=D.jpeg_collate)
        D.take_device_decode_stats()
        (batch, _, _), = list(loader)
        got = batch.cuda()
        assert torch.equal(got, want)
        refused = sum(S.BY_NAME[n].rc != 0 for n in names)
        flagged = sum(S.BY_NAME[n].rc == 0 and S.BY_NAME[n].device == "flag" for n in names)
        assert D.take_device_decode_stats() == {"device": len(names) - refused - flagged, "flagged": flagged,
                                                "host": refused}
