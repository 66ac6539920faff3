"""Records the Latte video loaders' transforms, so omt_resample_clips and layout.resize_clip are pinned to them.

    python -m oracle.make_golden_clips     (writes tests/golden/clip_resize.pt; needs the reference tree)

The reference's Diffusion/Latte/datasets/video_transforms.py is imported unmodified by file path (the package's
__init__ needs decord) and composed exactly as datasets/__init__.py composes it:
- "ucf": ucf101 / ffs: ToTensorVideo, RandomHorizontalFlipVideo, UCFCenterCropVideo(s), Normalize(.5, .5, inplace);
- "sky": ToTensorVideo, CenterCropResizeVideo(s), Normalize;
- "taichi": ToTensorVideo, RandomHorizontalFlipVideo, Normalize.
Sources are seeded uint8 clips shaped like torchvision.io.read_video(..., output_format='TCHW'): a (F, H, W, 3) buffer
viewed as (F, 3, H, W).  Each transform's pass draws its flips from Python's random seeded with SEED; a subclass records
them.  The pass runs with torch on one thread, as in the loaders' DataLoader workers (torch's bilinear kernel depends on
it, layout.clip_interp_form).  Outputs are small (S, F) to keep the fixture under 1 MB.
"""
import importlib.util
import os
import random
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "clip_resize.pt")
S = 32
F = 5
SEED = 3
SOURCE_SEED = 8
# UCF-101's 240 x 320, portrait, 1080p, upscales from 1 x 1 and 2 x 3, short sides already at S, and both of
# center_crop's round-half-to-even cases: (43 - 32) / 2 = 5.5 -> 6 and (45 - 32) / 2 = 6.5 -> 6
SIZES = [(240, 320), (320, 240), (1080, 1920), (1, 1), (2, 3), (32, 43), (45, 32)]
# "taichi" does not resize, so its clips keep their own (small) frame sizes
TAICHI_SIZES = [(32, 32), (8, 12), (1, 1)]


def sources(sizes=SIZES, seed=SOURCE_SEED, frames=F):
    """(F, H, W, 3) uint8 clips, regenerated from the seed."""
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 256, (frames, h, w, 3), generator=g, dtype=torch.uint8) for h, w in sizes]


def video_transforms():
    from oracle import ref_loader
    path = os.path.join(ref_loader.REF_ROOT, "Diffusion", "Latte", "datasets", "video_transforms.py")
    spec = importlib.util.spec_from_file_location("latte_video_transforms", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def transforms_by_name(s=S):
    """name -> (the loader's Compose, a function reading back the flip its last call drew)."""
    from torchvision import transforms
    vt = video_transforms()

    class Flip(vt.RandomHorizontalFlipVideo):        # records whether the clip was flipped
        def __call__(self, clip):
            out = super().__call__(clip)
            self.drawn = out is not clip
            return out

    flip = Flip()
    norm = transforms.Normalize(mean=[0.5, 0.5, 0.5], std=[0.5, 0.5, 0.5], inplace=True)
    return {
        "ucf": (transforms.Compose([vt.ToTensorVideo(), flip, vt.UCFCenterCropVideo(s), norm]), lambda: bool(flip.drawn)),
        "sky": (transforms.Compose([vt.ToTensorVideo(), vt.CenterCropResizeVideo(s), norm]), lambda: False),
        "taichi": (transforms.Compose([vt.ToTensorVideo(), flip, norm]), lambda: bool(flip.drawn)),
    }


def build(s=S, seed=SEED):
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        g = {"sizes": SIZES, "taichi_sizes": TAICHI_SIZES, "s": s, "frames": F, "seed": seed, "source_seed": SOURCE_SEED,
             "cpu_capability": torch.backends.cpu.get_cpu_capability(), "num_threads": 1}
        for name, (tf, drawn) in transforms_by_name(s).items():
            srcs = sources(TAICHI_SIZES if name == "taichi" else SIZES)
            g.setdefault("source_sum", {})[name] = [int(c.long().sum()) for c in srcs]
            random.seed(seed)
            outs, flips = [], []
            for c in srcs:
                outs.append(tf(c.permute(0, 3, 1, 2)).contiguous())     # read_video's TCHW view of a THWC buffer
                flips.append(drawn())
            g[name] = {"out": outs, "flips": flips, "random_after": random.getstate()}
        return g
    finally:
        torch.set_num_threads(threads)


def main():
    g = build()
    torch.save(g, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e3:.1f} KB, CPU capability {g['cpu_capability']})")


if __name__ == "__main__":
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    main()
