"""Makes tests/golden/nyud2_transform.npz: the random draws the reference's own NYUD2-DIR training chain
(nyud2-dir/loaddata.py:108-125 with nyud2-dir/nyu_transform.py) consumes, recorded while it transforms seeded
synthetic 320 x 240 samples (the size Scale(240) gives, so Scale is a no-op).  tests/test_nyud2_input_pipeline_cpu.py
checks that loaddata.draw_nyud2_train_params reproduces them exactly from the same seeds.

Recorded per sample, in consumption order: random.random() (flip), random.uniform(-5, 5) (angle), Lighting's normal_
draws, ColorJitter's randperm(3), and the three random.uniform(-0.4, 0.4) weights in the order applied.

    python tests/golden/make_golden_nyud2_transform.py      (needs oracle/_ref from __graft_entry__.build())
"""
import os
import random
import sys

import numpy as np
import torch
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

N = 12
PY_SEED, TORCH_SEED = 20261016, 7


def main():
    from oracle import nyu_transform_ref
    nt, _ = nyu_transform_ref.load()
    from torchvision import transforms
    pca = {'eigval': torch.Tensor([0.2175, 0.0188, 0.0045]),
           'eigvec': torch.Tensor([[-0.5675, 0.7192, 0.4009], [-0.5808, -0.0045, -0.8140], [-0.5836, -0.6948, 0.4203]])}
    chain = transforms.Compose([nt.Scale(240), nt.RandomHorizontalFlip(), nt.RandomRotate(5),
                                nt.CenterCrop([304, 228], [152, 114]), nt.ToTensor(),
                                nt.Lighting(0.1, pca['eigval'], pca['eigvec']),
                                nt.ColorJitter(brightness=0.4, contrast=0.4, saturation=0.4),
                                nt.Normalize([0.485, 0.456, 0.406], [0.229, 0.224, 0.225])])
    log = []

    class Recorder:
        def random(self):
            v = random.random()
            log.append(("random", v))
            return v

        def uniform(self, a, b):
            v = random.uniform(a, b)
            log.append(("uniform", v))
            return v

    real_randperm, real_normal = torch.randperm, torch.Tensor.normal_

    def randperm(n, *a, **k):
        v = real_randperm(n, *a, **k)
        log.append(("randperm", v.tolist()))
        return v

    def normal_(self, *a, **k):
        v = real_normal(self, *a, **k)
        log.append(("normal", v.tolist()))
        return v

    data = np.random.RandomState(0)
    samples = [{'image': Image.fromarray(data.randint(0, 256, (240, 320, 3)).astype(np.uint8)),
                'depth': Image.fromarray(data.randint(0, 256, (240, 320)).astype(np.uint8))} for _ in range(N)]
    random.seed(PY_SEED)
    torch.manual_seed(TORCH_SEED)
    nt.random, torch.randperm, torch.Tensor.normal_ = Recorder(), randperm, normal_
    try:
        for s in samples:
            chain(s)
    finally:
        nt.random, torch.randperm, torch.Tensor.normal_ = random, real_randperm, real_normal
    kinds = [k for k, _ in log]
    assert kinds == ["random", "uniform", "normal", "randperm", "uniform", "uniform", "uniform"] * N, kinds[:10]
    rec = np.array(log, dtype=object).reshape(N, 7, 2)[:, :, 1]
    np.savez(os.path.join(HERE, "nyud2_transform.npz"), py_seed=PY_SEED, torch_seed=TORCH_SEED,
             flip_u=np.array(rec[:, 0], np.float64), angle=np.array(rec[:, 1], np.float64),
             normal=np.array(list(rec[:, 2]), np.float32), perm=np.array(list(rec[:, 3]), np.int64),
             jitter=np.array(rec[:, 4:7].tolist(), np.float64))


if __name__ == "__main__":
    main()
