"""CPU restatement of the reference's uint8 -> fp32 video normalisation, as its data loader applies it.

DecordVideoDataset.__getitem__ (OmniTokenizer/data.py:229-232) turns each decoded clip (T, H, W, 3) uint8 into
`torch.from_numpy(frames).float().permute(0, 3, 1, 2)`, applies VideoNorm (OmniTokenizer/video_utils.py:33-58) and
permutes to (3, T, H, W).  VideoNorm divides by 255 only when the clip's maximum exceeds 1, then subtracts the mean
and divides by the std, in place, in fp32.  Pinned to the live reference by tests/golden/u8_norm.pt
(oracle/make_golden_u8.py).
"""
import torch


def video_norm(frames: torch.Tensor, mean=(0.5, 0.5, 0.5), std=(1.0, 1.0, 1.0)) -> torch.Tensor:
    """(B, T, H, W, C) uint8 clips -> (B, C, T, H, W) fp32, each clip normalised on its own as the loader does."""
    C = frames.shape[-1]
    m = torch.tensor(mean).view(1, C, 1, 1)
    s = torch.tensor(std).view(1, C, 1, 1)
    out = []
    for clip in frames.cpu():
        img = clip.float().permute(0, 3, 1, 2)            # T, C, H, W
        if torch.max(img) > 1 and m.max() <= 1:
            img.div_(255.0)
        out.append(img.sub_(m).div_(s).permute(1, 0, 2, 3))
    return torch.stack(out).contiguous()
