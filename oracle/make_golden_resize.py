"""Records the image loaders' Pillow resize / random crop / flip, so omt_resample_u8 and layout.resize_u8 are pinned to them.

    python -m oracle.make_golden_resize     (writes tests/golden/u8_resize.pt; needs Pillow and torchvision)

The three geometric transforms run, as the reference composes them, on seeded uint8 source images (sources()): a few of
photo size, many small ones, upscales, extreme aspect ratios (one taller than 100x its width, which Pillow resizes
vertical pass first), 1-pixel sides and sources already at the output size.  Output sizes are small (RES) to keep the
fixture small.  Each transform is the part of the loader's Compose before ToTensor, applied to the PIL image:
- "image": ImageDataset without --resizecrop (OmniTokenizer/data.py:93-99): Resize((res, res), BICUBIC).
- "resizecrop": ImageDataset with --resizecrop (data.py:84-90): Resize((1.5 res, 1.5 res), BICUBIC), RandomCrop(res).
- "dit": DiT with the OmniTokenizer VAE (Diffusion/DiT/train.py:192-198): Resize((s, s)) (default BILINEAR),
  RandomHorizontalFlip().
The random transforms draw from torch's CPU generator seeded with SEED before each transform's pass over the images; the
parameters they drew (top, left, flip) are read back from torchvision's own calls and stored with the bytes.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "u8_resize.pt")
RES = 32
SEED = 21
SOURCE_SEED = 5
# (H, W): photo-sized, upscales, extreme aspect ratios, 1-pixel sides, at-size sources of each transform, and a tall
# 450 x 4 image (H > 100 W: Pillow's vertical-first order)
SIZES = [(375, 500), (333, 500), (500, 375),
         (31, 17), (9, 13), (1, 1), (1, 40), (40, 1), (2, 300), (300, 2), (450, 4), (7, 700),
         (32, 32), (48, 48), (32, 48), (48, 32), (33, 31), (64, 64), (100, 80), (16, 200)]


def sources(seed=SOURCE_SEED):
    """The fixture's source images, (H, W, 3) uint8, regenerated from the seed."""
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8) for h, w in SIZES]


def transforms_by_name(res=RES):
    """name -> (the geometric part of the loader's Compose, a function reading back the params its last call drew)."""
    from torchvision import transforms
    from torchvision.transforms import InterpolationMode

    class Crop(transforms.RandomCrop):              # records what RandomCrop.get_params returned
        def get_params(self, img, output_size):
            self.drawn = transforms.RandomCrop.get_params(img, output_size)
            return self.drawn

    class Flip(transforms.RandomHorizontalFlip):    # records whether the image was flipped
        def forward(self, img):
            out = super().forward(img)
            self.drawn = out is not img
            return out

    side = int(res * 1.5)
    crop, flip = Crop(res), Flip()
    return {
        "image": (transforms.Compose([transforms.Resize((res, res), interpolation=InterpolationMode.BICUBIC)]),
                  lambda: (0, 0, False)),
        "resizecrop": (transforms.Compose([transforms.Resize((side, side), interpolation=InterpolationMode.BICUBIC), crop]),
                       lambda: (int(crop.drawn[0]), int(crop.drawn[1]), False)),
        "dit": (transforms.Compose([transforms.Resize((res, res)), flip]), lambda: (0, 0, bool(flip.drawn))),
    }


def build(res=RES, seed=SEED):
    from PIL import Image
    srcs = sources()
    g = {"sizes": SIZES, "res": res, "seed": seed, "source_seed": SOURCE_SEED,
         "source_sum": [int(s.long().sum()) for s in srcs]}
    for name, (tf, drawn) in transforms_by_name(res).items():
        torch.manual_seed(seed)
        outs, params = [], []
        for s in srcs:
            outs.append(torch.from_numpy(np.asarray(tf(Image.fromarray(s.numpy()))).copy()))
            params.append(drawn())
        g[name] = {"out": torch.stack(outs), "params": params, "rng_after": torch.get_rng_state()}
    return g


def main():
    g = build()
    torch.save(g, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e3:.1f} KB)")


if __name__ == "__main__":
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    main()
