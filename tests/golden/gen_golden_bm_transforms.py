"""Generate tests/golden/ref_bm_transforms.npz from the UNMODIFIED SipMask-benchmark test transform
(fcos_core/data/transforms/transforms.py, loaded by file path: it needs only torchvision and PIL).  Run from the
repository root where /root/reference exists:  python tests/golden/gen_golden_bm_transforms.py

  sizes_src [M, 2], sizes_out [M, 2] : (h, w) -> the (oh, ow) of Resize(800, 1333).get_size on a seeded grid of sources
                                       plus edge cases (1x1, 1x2048, 56x1345, 800xN, exact-ratio ties)
  img_i, out_i, size_i, rule_i       : a seeded uint8 RGB image, the reference's tensor for it, the (oh, ow) it was
                                       resized to and rule_i = (min_size, max_size).  rule (96, 160) cases run
                                       Resize -> ToTensor -> Normalize(to_bgr255); rule (0, 0) cases call torchvision
                                       F.resize with size_i directly (a one-axis change, which the size rule never
                                       produces), then ToTensor -> Normalize.
"""
import importlib.util
import os
import random

import numpy as np
import torch
from PIL import Image
from torchvision.transforms import functional as F

OUT = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference/SipMask-benchmark/fcos_core/data/transforms/transforms.py'
MEAN = [102.9801, 115.9465, 122.7717]          # configs/sipmask/*.yaml via config/defaults.py: PIXEL_MEAN, PIXEL_STD = 1


def load_transforms():
    spec = importlib.util.spec_from_file_location('bm_transforms', REF)
    T = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(T)
    return T


def size_grid(T):
    rs = np.random.RandomState(0)
    src = [(int(h), int(w)) for h, w in rs.randint(1, 2049, (400, 2))]
    src += [(1, 1), (1, 2048), (2048, 1), (56, 1345), (1345, 56), (800, 800), (800, 1000), (1000, 800), (800, 1333),
            (800, 1334), (800, 2048), (480, 800), (600, 1000), (1000, 600), (750, 1250), (1199, 2000), (400, 667), (3, 5),
            (480, 640), (427, 640), (640, 427), (1080, 1920), (2048, 1536), (333, 17)]
    r = T.Resize(800, 1333)
    out = [r.get_size((w, h)) for h, w in src]                   # PIL sizes are (w, h)
    return np.asarray(src, np.int64), np.asarray(out, np.int64)


def images(T):
    rs = np.random.RandomState(1)
    norm = T.Normalize(mean=MEAN, std=[1., 1., 1.], to_bgr255=True)
    cases = [((40, 50), (96, 160)),          # upscale
             ((300, 250), (96, 160)),        # downscale beyond 2x
             ((96, 130), (96, 160)),         # short side already 96: not resized
             ((45, 170), (96, 160)),         # long side capped by max_size
             ((61, 83), None)]               # one axis only: F.resize((61, 40))
    d = {}
    for i, (hw, rule) in enumerate(cases):
        img = rs.randint(0, 256, hw + (3,), dtype=np.uint8)
        pil = Image.fromarray(img, 'RGB')
        if rule is not None:
            resize = T.Resize(*rule)
            size = resize.get_size(pil.size)
            x = resize(pil)
        else:
            size = (61, 40)
            x = F.resize(pil, list(size))
        x, _ = T.ToTensor()(x, None)
        x = norm(x)
        d['img_%d' % i] = img
        d['out_%d' % i] = x.numpy()
        d['size_%d' % i] = np.asarray(size, np.int64)
        d['rule_%d' % i] = np.asarray(rule or (0, 0), np.int64)
    return d


def main():
    random.seed(0)                                               # Resize.get_size draws from a one-element list
    T = load_transforms()
    src, out = size_grid(T)
    d = dict(sizes_src=src, sizes_out=out, count=np.int64(5))
    d.update(images(T))
    path = os.path.join(OUT, 'ref_bm_transforms.npz')
    np.savez_compressed(path, **d)
    print('wrote %s (%d bytes)' % (path, os.path.getsize(path)))


if __name__ == '__main__':
    torch.set_num_threads(1)
    main()
