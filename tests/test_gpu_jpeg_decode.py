"""Device JPEG decode and Pillow bilinear resize (csrc/jpeg.cu), byte for byte against the local Pillow: the decode over
sizes x content x encoder settings in one launch and one image at a time, the resize up and down, AgeDB(device_decode)
through a DataLoader against AgeDB(device_transform), the host fallback of images the device flags, and train.py
--device_decode."""
import io

import numpy as np
import pytest
import torch

import jpeg_cases as J

pytestmark = pytest.mark.gpu


def test_pillow_decodes_with_libjpeg_turbo():
    import PIL.features
    assert PIL.features.check_feature("libjpeg_turbo"), "byte parity is defined against libjpeg-turbo"


def _matrix():
    cases = []
    for (h, w) in J.SIZES:
        for kind in J.CONTENTS:
            for setting in J.SETTINGS:
                if (h, w) == (2000, 1500) and setting not in ("gray", "420", "444_q100", "420_restart_rows"):
                    continue                                   # keep the largest size to the main forms
                cases.append(((h, w, kind, setting), J.case(kind, h, w, setting, seed=h * 7 + w)))
    return cases


def test_decode_equals_pillow_in_one_launch():
    cases = _matrix()
    raws = [r for _, r in cases]
    got, status = J.device_decode(raws)
    assert (status == 0).all(), [cases[i][0] for i in np.nonzero(status)[0]]
    bad = [key for (key, raw), g in zip(cases, got) if not np.array_equal(g, J.pillow_rgb(raw))]
    assert not bad, bad


@pytest.mark.parametrize("setting", ["gray", "444", "422", "420", "444_q100", "420_restart_rows"])
def test_decode_equals_pillow_one_image_per_launch(setting):
    for (h, w) in J.SIZES[:-1]:
        raw = J.case("noise", h, w, setting, seed=h + w)
        got, status = J.device_decode([raw])
        assert status[0] == 0 and np.array_equal(got[0], J.pillow_rgb(raw)), (h, w)


def _resize_call(images, out_h, out_w):
    import _lib
    hw = np.asarray([im.shape[:2] for im in images], dtype=np.int32)
    offs = np.concatenate([[0], np.cumsum([im.size for im in images])[:-1]]).astype(np.int64)
    dev = torch.device("cuda")
    src = torch.from_numpy(np.concatenate([im.reshape(-1) for im in images])).to(dev)
    d_off, d_hw = torch.from_numpy(offs).to(dev), torch.from_numpy(hw).to(dev)
    out = torch.empty(len(images), out_h, out_w, 3, dtype=torch.uint8, device=dev)
    wsb = int(_lib.raw("dirb200_resize_bilinear_workspace_bytes")(hw.ctypes.data_as(_lib.P), len(images), out_h, out_w))
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    _lib.call("dirb200_resize_bilinear_u8", _lib.ptr(src), _lib.ptr(d_off), _lib.ptr(d_hw), len(images), out_h, out_w,
              _lib.ptr(out), _lib.ptr(ws), wsb, _lib.stream_ptr())
    return out.cpu().numpy()


@pytest.mark.parametrize("out_hw", [(32, 32), (224, 224), (256, 256), (100, 60)])
def test_resize_equals_pillow_bilinear_and_torchvision_resize(out_hw):
    from PIL import Image
    from torchvision import transforms
    rng = np.random.RandomState(out_hw[0] * 1000 + out_hw[1])
    sizes = [(1, 1), (2, 3), (7, 9), (31, 33), (224, 224), (250, 250), (256, 255), (500, 500), (1000, 800), (13, 600),
             (1500, 900), (900, 1500)]
    sizes += [tuple(int(v) for v in rng.randint(1, 1500, size=2)) for _ in range(6)]
    images = [rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8) for (h, w) in sizes]
    got = _resize_call(images, *out_hw)
    for k, im in enumerate(images):
        want = np.asarray(Image.fromarray(im).resize((out_hw[1], out_hw[0]), Image.BILINEAR))
        assert np.array_equal(got[k], want), (sizes[k], out_hw)
        if out_hw[0] == out_hw[1]:
            tv = np.asarray(transforms.Resize(out_hw)(Image.fromarray(im)))
            assert np.array_equal(got[k], tv), sizes[k]


def _dataset_files(tmp_path):
    import pandas as pd
    from PIL import Image
    files = {}
    for i, setting in enumerate(J.SETTINGS):
        kind = J.CONTENTS[i % 3]
        h, w = [(225, 224), (120, 97), (33, 31), (300, 410)][i % 4]
        files[f"{setting}.jpg"] = J.case(kind, h, w, setting, seed=i)
    arr = J.content("smooth", 140, 90, 11)
    bio = io.BytesIO()
    Image.fromarray(arr).save(bio, "JPEG", progressive=True)
    files["progressive.jpg"] = bio.getvalue()
    bio = io.BytesIO()
    Image.fromarray(arr).save(bio, "PNG")
    files["image.png"] = bio.getvalue()
    for name, raw in files.items():
        (tmp_path / name).write_bytes(raw)
    names = list(files)
    df = pd.DataFrame({"path": names, "age": [float(10 + 5 * i) for i in range(len(names))],
                       "split": ["train"] * len(names)})
    return df, files


def test_dataset_device_decode_through_a_loader_equals_device_transform(tmp_path):
    import datasets as D
    from torch.utils.data import DataLoader
    df, _ = _dataset_files(tmp_path)
    S = 64
    dec = D.AgeDB(df=df, data_dir=str(tmp_path), img_size=S, device_decode=True)
    ref = D.AgeDB(df=df, data_dir=str(tmp_path), img_size=S, device_transform=True)
    want = torch.stack([ref[i][0] for i in range(len(ref))]).cuda()
    loader = DataLoader(dec, batch_size=len(dec), shuffle=False, num_workers=2, pin_memory=True,
                        collate_fn=D.jpeg_collate)
    D.take_device_decode_stats()
    (batch, labels, weights), = list(loader)
    got = batch.cuda(non_blocking=True)
    assert got.dtype == torch.uint8 and got.shape == (len(dec), S, S, 3)
    assert torch.equal(got, want)
    assert batch.flagged == []
    assert D.take_device_decode_stats() == {"device": len(dec) - 2, "flagged": 0, "host": 2}
    assert labels[:, 0].tolist() == list(df["age"].values)
    # the rest of the pipeline: the same draws give the same tensors
    for train in (True, False):
        torch.manual_seed(3)
        a = D.gpu_transform_batch(got, train=train)
        torch.manual_seed(3)
        b = D.gpu_transform_batch(want, train=train)
        assert torch.equal(a, b)


def _scan_range(raw):
    import datasets as D
    rc, desc, _ = D.parse_jpeg(raw)
    d = desc.view(D.JPEG_DESC_DTYPE)[0]
    return int(d["scan_begin"]), int(d["scan_end"])


def _anomalies():
    good = J.case("noise", 64, 80, "420", seed=1)
    b, e = _scan_range(good)
    truncated = good[:b + (e - b) // 2] + good[e:]                  # half the scan gone, EOI kept
    mid = b + (e - b) // 2
    invalid = good[:mid] + b"\xff\x00" * 8 + good[mid + 16:]        # 64 one-bits: no Huffman code is all ones
    return good, {"truncated": truncated, "invalid_code": invalid}


@pytest.mark.parametrize("which", ["truncated", "invalid_code"])
def test_anomalies_are_flagged_and_decoded_by_pillow(which, tmp_path):
    import datasets as D
    good, bad = _anomalies()
    raw = bad[which]
    neighbours = [J.case("smooth", 40, 50, "444", seed=2), J.case("saturated", 17, 15, "gray", seed=3)]
    got, status = J.device_decode([neighbours[0], raw, neighbours[1]])
    assert status[1] != 0 and status[0] == 0 and status[2] == 0
    assert np.array_equal(got[0], J.pillow_rgb(neighbours[0])) and np.array_equal(got[2], J.pillow_rgb(neighbours[1]))
    # through the dataset: the flagged image ends as Pillow's result (or raises Pillow's exception)
    import pandas as pd
    from PIL import Image
    names = ["n0.jpg", "bad.jpg", "n1.jpg"]
    for name, r in zip(names, [neighbours[0], raw, neighbours[1]]):
        (tmp_path / name).write_bytes(r)
    df = pd.DataFrame({"path": names, "age": [1.0, 2.0, 3.0], "split": ["train"] * 3})
    ds = D.AgeDB(df=df, data_dir=str(tmp_path), img_size=48, device_decode=True)
    batch, _, _ = D.jpeg_collate([ds[i] for i in range(3)])
    try:
        want = D.host_resize_u8(Image.open(tmp_path / "bad.jpg").convert("RGB"), 48)
    except Exception as e:                                          # Pillow's exception is the result
        with pytest.raises(type(e)):
            batch.cuda()
        return
    out = batch.cuda()
    assert batch.flagged == [1]
    ref = D.AgeDB(df=df, data_dir=str(tmp_path), img_size=48, device_transform=True)
    assert torch.equal(out[1].cpu(), want)
    for i in (0, 2):
        assert torch.equal(out[i].cpu(), ref[i][0])


def test_train_script_device_decode_matches_device_transform(tmp_path, monkeypatch):
    import train
    data = tmp_path / "data"
    data.mkdir()
    import pandas as pd
    rows = []
    for i in range(24):
        setting = list(J.SETTINGS)[i % len(J.SETTINGS)]
        h, w = 40 + 3 * i, 56 - i
        name = f"{i}.jpg"
        (data / name).write_bytes(J.case(J.CONTENTS[i % 3], h, w, setting, seed=100 + i))
        rows.append((name, float(5 + 4 * i), ["train", "train", "val", "test"][i % 4]))
    pd.DataFrame(rows, columns=["path", "age", "split"]).to_csv(data / "agedb.csv", index=False)

    first = {}
    real = train.gpu_transform_batch

    def capture(images, train=True, **kw):
        out = real(images, train=train, **kw)
        first.setdefault(run, (images.clone(), out.clone()))
        return out

    monkeypatch.setattr(train, "gpu_transform_batch", capture)
    for run in ("--device_transform", "--device_decode"):
        torch.manual_seed(0)
        train.main([run, "--data_dir", str(data), "--batch_size", "8", "--epoch", "1", "--workers", "0",
                    "--img_size", "32", "--print_freq", "1", "--store_root", str(tmp_path / run.strip("-")),
                    "--lr", "1e-4"])
    a, b = first["--device_transform"], first["--device_decode"]
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
