"""Records the reference data pipelines' uint8 -> fp32 normalisations, so the byte tables of encode_u8 are pinned to them.

    OMT_REFERENCE_ROOT=<reference checkout> python -m oracle.make_golden_u8     (writes tests/golden/u8_norm.pt)

Each transform runs, as the reference composes it, on seeded uint8 clips in which every channel holds every byte value
once (a random permutation of 0..255 per channel and frame), plus VideoNorm's quirk clips whose maximum byte is 0, 1
and 2 (only the last is divided by 255):
- "video_norm": VideoNorm (OmniTokenizer/video_utils.py:33-58) in DecordVideoDataset.__getitem__'s order (data.py:229-232),
  (T, H, W, 3) -> float -> permute(0, 3, 1, 2) -> VideoNorm -> permute(1, 0, 2, 3) = (3, T, H, W).
- "image_norm": torchvision ToTensor + Normalize((.5, .5, .5), (1, 1, 1)) on an (H, W, 3) array (data.py:88-97; also DiT
  train.py:185-198's std = 1 branch) -> (3, H, W).
- "dit_norm": ToTensor + Normalize(.5, .5, inplace=True) (DiT train.py:185-198) -> (3, H, W).
- "latte_norm": Latte's video_transforms.to_tensor + Normalize(.5, .5, inplace=True) (Latte datasets/*, e.g.
  sky_datasets.py:90-94) on a (T, 3, H, W) clip -> (T, 3, H, W).
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_loader as rl  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "u8_norm.pt")
T, H, W, C = 2, 16, 16, 3          # H * W = 256: each (frame, channel) plane is one permutation of the byte values
SEED = 8


def full_clip(seed=SEED) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    planes = [torch.randperm(256, generator=g).to(torch.uint8).view(H, W) for _ in range(T * C)]
    return torch.stack(planes).view(T, C, H, W).permute(0, 2, 3, 1).contiguous()      # (T, H, W, C)


def quirk_clips(seed=SEED + 1):
    g = torch.Generator().manual_seed(seed)
    out = {}
    for mx in (0, 1, 2):
        c = torch.randint(0, mx + 1, (T, H, W, C), generator=g).to(torch.uint8)
        c[0, 0, 0, 0] = mx                                                              # the maximum is reached
        out[mx] = c
    return out


def _load_file(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    assert rl.available(), "the reference tree is needed (OMT_REFERENCE_ROOT)"
    rl.load()                                                    # stubs + the OmniTokenizer package without __init__.py
    sys.modules.setdefault("decord", types.SimpleNamespace(VideoReader=object, cpu=None, gpu=None, bridge=None))
    import OmniTokenizer.video_utils as vu
    from torchvision import transforms
    vt = _load_file("latte_video_transforms", os.path.join(rl.REF_ROOT, "Diffusion", "Latte", "datasets", "video_transforms.py"))

    clip = full_clip()
    quirks = quirk_clips()
    g = {"shape": (T, H, W, C), "clip": clip, "quirk": quirks}

    def video_norm(c):                                           # data.py:229-232
        vid = torch.from_numpy(c.numpy()).float().permute(0, 3, 1, 2)
        return vu.VideoNorm()(vid).permute(1, 0, 2, 3).contiguous()

    g["video_norm"] = video_norm(clip)
    g["video_norm_quirk"] = {mx: video_norm(c) for mx, c in quirks.items()}
    image_tf = transforms.Compose([transforms.ToTensor(), transforms.Normalize((0.5, 0.5, 0.5), (1.0, 1.0, 1.0))])
    dit_tf = transforms.Compose([transforms.ToTensor(), transforms.Normalize(mean=[0.5, 0.5, 0.5], std=[0.5, 0.5, 0.5], inplace=True)])
    g["image_norm"] = torch.stack([image_tf(np.ascontiguousarray(clip[t].numpy())) for t in range(T)])     # (T, 3, H, W)
    g["dit_norm"] = torch.stack([dit_tf(np.ascontiguousarray(clip[t].numpy())) for t in range(T)])
    latte_tf = transforms.Compose([vt.ToTensorVideo(), transforms.Normalize(mean=[0.5, 0.5, 0.5], std=[0.5, 0.5, 0.5], inplace=True)])
    g["latte_norm"] = latte_tf(clip.permute(0, 3, 1, 2).contiguous())                                      # (T, 3, H, W)
    torch.save(g, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e3:.1f} KB)")


if __name__ == "__main__":
    main()
