"""Seeded JPEG test images for the device decoder's tests: content kinds, the encoder settings Pillow offers for the
supported set, and a direct call of dirb200_jpeg_decode at full resolution."""
import io

import numpy as np

SIZES = [(1, 1), (7, 9), (8, 8), (15, 17), (16, 16), (33, 31), (225, 224), (640, 480), (2000, 1500)]   # (h, w)
CONTENTS = ("smooth", "noise", "saturated")
# name -> Pillow save() options; "gray" encodes a single-component image
SETTINGS = {
    "gray": dict(gray=True, quality=90),
    "444": dict(subsampling=0, quality=90),
    "422": dict(subsampling=1, quality=90),
    "420": dict(subsampling=2, quality=90),
    "420_optimize": dict(subsampling=2, quality=90, optimize=True),
    "420_q1": dict(subsampling=2, quality=1),
    "422_q50": dict(subsampling=1, quality=50),
    "444_q100": dict(subsampling=0, quality=100),
    "420_q100": dict(subsampling=2, quality=100),
    "444_restart_blocks": dict(subsampling=0, quality=90, restart_marker_blocks=3),
    "420_restart_rows": dict(subsampling=2, quality=90, restart_marker_rows=1),
}


def content(kind, h, w, seed, gray=False):
    rng = np.random.RandomState(seed)
    shape = (h, w) if gray else (h, w, 3)
    if kind == "noise":                                  # full range: reaches the IDCT's range limit
        return rng.randint(0, 256, size=shape).astype(np.uint8)
    if kind == "saturated":
        return (rng.randint(0, 2, size=shape) * 255).astype(np.uint8)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    phase = rng.uniform(0, 6.28)
    base = 128 + 100 * np.sin(xx / 7.0 + yy / 11.0 + phase)
    if gray:
        return base.astype(np.uint8)
    return np.stack([base, 255 - base, (128 + 120 * np.cos(yy / 5.0 - xx / 13.0))], -1).clip(0, 255).astype(np.uint8)


def encode(arr, **opts):
    from PIL import Image
    opts = {k: v for k, v in opts.items() if k != "gray"}
    bio = io.BytesIO()
    Image.fromarray(arr).save(bio, "JPEG", **opts)
    return bio.getvalue()


def case(kind, h, w, setting, seed=0):
    opts = SETTINGS[setting]
    return encode(content(kind, h, w, seed, gray=opts.get("gray", False)), **opts)


def pillow_rgb(raw):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(raw)).convert("RGB"))


def device_decode(raws, device="cuda"):
    """dirb200_jpeg_decode of supported files in one launch: (list of uint8 HWC arrays, status int32 [n])."""
    import torch
    import _lib
    from datasets import parse_jpeg
    parsed = [parse_jpeg(r) for r in raws]
    assert all(p[0] == 0 for p in parsed), [p[0] for p in parsed]
    descs = np.stack([p[1] for p in parsed])
    hw = descs.view(np.int32)[:, :2].astype(np.int64)
    offsets = np.concatenate([[0], np.cumsum([len(r) for r in raws])]).astype(np.int64)
    rgb_offsets = np.concatenate([[0], np.cumsum(hw[:, 0] * hw[:, 1] * 3)]).astype(np.int64)
    dev = torch.device(device)
    t = lambda a: torch.from_numpy(np.array(a)).to(dev)
    data = t(np.frombuffer(b"".join(raws), dtype=np.uint8))
    d_off, d_desc, d_rgb_off = t(offsets), t(descs), t(rgb_offsets)
    d_iv = t(np.concatenate([p[2] for p in parsed]))
    rgb = torch.empty(int(rgb_offsets[-1]), dtype=torch.uint8, device=dev)
    status = torch.full((len(raws),), -1, dtype=torch.int32, device=dev)
    wsb = int(_lib.raw("dirb200_jpeg_decode_workspace_bytes")(descs.ctypes.data_as(_lib.P), len(raws)))
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    _lib.call("dirb200_jpeg_decode", _lib.ptr(data), _lib.ptr(d_off), _lib.ptr(d_desc), _lib.ptr(d_iv), len(raws),
              _lib.ptr(rgb), _lib.ptr(d_rgb_off), _lib.ptr(status), _lib.ptr(ws), wsb, _lib.stream_ptr())
    rgb, status = rgb.cpu().numpy(), status.cpu().numpy()
    out = [rgb[rgb_offsets[i]:rgb_offsets[i + 1]].reshape(int(hw[i, 0]), int(hw[i, 1]), 3) for i in range(len(raws))]
    return out, status
