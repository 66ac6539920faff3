"""Records vqgan_eval.py's --infer_downsample and --replacewithgt, so omt_eval_downsample, the LANCZOS resize tables and
their host twins are pinned to the script's own lines.

    python -m oracle.make_golden_eval_downsample     (writes tests/golden/eval_downsample.pt; needs Pillow, torchvision)

Video branch (vqgan_eval.py:121-148), on seeded uint8 clips and seeded fp32 reconstructions standing in for x_recons:
    real_videos = batch['video'] + 0.5                     batch['video']: VideoNorm of the clip (oracle/u8_norm.py)
    fake_videos = torch.clamp(x_recons + 0.5, 0, 1)
    both rearranged "b c t h w -> (b t) c h w", F.interpolate(scale_factor=1/d, mode="bilinear", align_corners=False),
    rearranged back; with --replacewithgt k the first k fake frames are the real ones (:142-145);
    shift_dim(videos * 255, 1, -1).byte() is what get_fvd_logits receives (:147-148).
Each clip set runs at d = 2, 3 (scale_factor 1/3 is not exact in binary) and 4, with torch on one thread and on
several: the two pick different CPU bilinear kernels for outputs with h + w > 128.  One clip of each set holds only the
bytes 0 and 1, VideoNorm's undivided branch.

Image branch (vqgan_eval.py:201-220), on seeded uint8 images and fp32 reconstructions:
    input_ = ToTensor + Normalize((.5, .5, .5), (1, 1, 1)) of the image  (OmniTokenizer/data.py:93-99)
    ((input_ + 0.5).numpy() * 255).astype(np.uint8)  and  (torch.clamp(recon_ + 0.5, 0, 1).numpy() * 255).astype(np.uint8)
    Image.fromarray(...).resize((res // d, res // d), Image.ANTIALIAS)
Pillow 10 removed the name ANTIALIAS; it was LANCZOS's alias, which is used when the name is gone.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "eval_downsample.pt")
SEED = 17
# (B, T, H, W): 48 x 216 at d = 2 comes out 24 x 108 (h + w > 128: the thread count picks the kernel); 63 x 50 has odd
# sides that no factor divides evenly
CLIP_SHAPES = [(2, 1, 48, 216), (2, 3, 63, 50)]
FACTORS = (2, 3, 4)
REPLACE = {"shape": 1, "d": 3, "ks": (0, 2)}
IMAGE_RES, IMAGE_B = 64, 2


def several_threads() -> int:
    return max(2, min(8, os.cpu_count() or 2))


def clip_inputs(shape, g):
    """uint8 clips (B, T, H, W, 3), the last one of bytes 0 / 1 only, and fp32 reconstructions (B, 3, T, H, W)."""
    B, T, H, W = shape
    u8 = torch.randint(0, 256, (B, T, H, W, 3), generator=g, dtype=torch.uint8)
    u8[-1] = torch.randint(0, 2, (T, H, W, 3), generator=g, dtype=torch.uint8)
    recons = (torch.randn(B, 3, T, H, W, generator=g) * 0.4).float()
    return u8, recons


def interpolate(videos, d):
    """vqgan_eval.py:124-135."""
    from einops import rearrange
    import torch.nn.functional as F
    B = videos.shape[0]
    v = rearrange(videos, "b c t h w -> (b t) c h w")
    v = F.interpolate(v, scale_factor=1 / d, mode="bilinear", align_corners=False)
    return rearrange(v, "(b t) c h w -> b c t h w", b=B)


def to_bytes(videos):
    """vqgan_eval.py:147-148: shift_dim(videos * 255, 1, -1).byte()."""
    return (videos * 255).movedim(1, -1).byte().contiguous()


def video_case(u8, recons, d, replacewithgt=None):
    from oracle.u8_norm import video_norm
    real_videos = video_norm(u8) + 0.5
    fake_videos = torch.clamp(recons + 0.5, 0, 1)
    real_videos, fake_videos = interpolate(real_videos, d), interpolate(fake_videos, d)
    if replacewithgt is not None:
        fake_videos = torch.cat((real_videos[:, :, :replacewithgt], fake_videos[:, :, replacewithgt:]), dim=2)
    return to_bytes(real_videos), to_bytes(fake_videos)


def image_case(u8, recons, d):
    from PIL import Image
    from torchvision.transforms import functional as TF
    antialias = getattr(Image, "ANTIALIAS", Image.LANCZOS)
    side = IMAGE_RES // d
    real, fake = [], []
    for im, recon_ in zip(u8, recons):
        input_ = TF.normalize(TF.to_tensor(Image.fromarray(im.numpy())), (0.5, 0.5, 0.5), (1.0, 1.0, 1.0))
        input_ = ((input_.permute(1, 2, 0) + 0.5).numpy() * 255).astype(np.uint8)
        recon_ = (torch.clamp(recon_.permute(1, 2, 0) + 0.5, 0, 1).numpy() * 255).astype(np.uint8)
        real.append(np.asarray(Image.fromarray(input_).resize((side, side), antialias)))
        fake.append(np.asarray(Image.fromarray(recon_).resize((side, side), antialias)))
    return torch.from_numpy(np.stack(real)), torch.from_numpy(np.stack(fake))


def build(seed=SEED):
    old = torch.get_num_threads()
    g = torch.Generator().manual_seed(seed)
    out = {"seed": seed, "cpu_capability": torch.backends.cpu.get_cpu_capability(), "several": several_threads(),
           "clips": [], "video": [], "replace": [], "images": {}}
    try:
        for shape in CLIP_SHAPES:
            u8, recons = clip_inputs(shape, g)
            out["clips"].append({"shape": shape, "u8": u8, "recons": recons})
            for d in FACTORS:
                for threads in (1, several_threads()):
                    torch.set_num_threads(threads)
                    real, fake = video_case(u8, recons, d)
                    out["video"].append({"clip": len(out["clips"]) - 1, "d": d, "one_thread": threads == 1,
                                         "real": real, "fake": fake})
        c = out["clips"][REPLACE["shape"]]
        torch.set_num_threads(several_threads())
        for k in REPLACE["ks"]:
            real, fake = video_case(c["u8"], c["recons"], REPLACE["d"], replacewithgt=k)
            out["replace"].append({"clip": REPLACE["shape"], "d": REPLACE["d"], "one_thread": False, "k": k,
                                   "real": real, "fake": fake})
        u8 = torch.randint(0, 256, (IMAGE_B, IMAGE_RES, IMAGE_RES, 3), generator=g, dtype=torch.uint8)
        recons = (torch.randn(IMAGE_B, 3, IMAGE_RES, IMAGE_RES, generator=g) * 0.4).float()
        out["images"] = {"res": IMAGE_RES, "u8": u8, "recons": recons,
                         "out": {d: image_case(u8, recons, d) for d in FACTORS}}
        return out
    finally:
        torch.set_num_threads(old)


def main():
    g = build()
    torch.save(g, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e3:.1f} KB, CPU capability {g['cpu_capability']})")


if __name__ == "__main__":
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    main()
