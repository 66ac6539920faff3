"""The pixels of a JPEG save and reload on the device: what Pillow's img.save(f, "JPEG", quality=q) followed by
Image.open(f).convert("RGB") gives, byte for byte (libjpeg-turbo's baseline 4:2:0 chain; oracle/jpeg_oracle.py is the
step-by-step host restatement).  vqgan_eval.py saves every input and reconstruction of a dataset whose paths end in
.jpg / .JPEG this way, and pytorch-fid reads them back (consumers.eval_step_fid(saved_as="jpeg")).

No file and no bitstream is made: entropy coding is lossless, so the pixels depend only on the integer transform chain,
which omt_jpeg_roundtrip_u8 runs in two launches.  Every check runs before the launch.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _cabi
from .metricnet import bounded

DEFAULT_QUALITY = 75            # Pillow's JPEG quality when save() is given none
MAX_SCRATCH = 4                 # scratch buffers kept per process; the oldest goes first
_scratch = {}
_tables = {}

# ITU-T T.81 Annex K, tables K.1 (luminance) and K.2 (chrominance), natural order
_BASE = np.array([
    [16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55,
     14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
     18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
     49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99],
    [17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99,
     24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32], dtype=np.int64)


def check_quality(quality, what: str = "jpeg") -> int:
    if isinstance(quality, bool) or not isinstance(quality, (int, np.integer)) or not 1 <= int(quality) <= 100:
        raise ValueError(f"{what}: JPEG quality {quality!r} is not an integer in 1..100")
    return int(quality)


def quant_tables(quality: int = DEFAULT_QUALITY) -> np.ndarray:
    """uint16 [2, 64] (luminance, chrominance) in natural order, the tables Pillow writes at this quality
    (Image.open(f).quantization): libjpeg's scaling of Annex K, s = 5000 / q below 50 and 200 - 2 q from 50,
    (base s + 50) / 100 clamped to 1..255 (baseline)."""
    q = check_quality(quality, "quant_tables")
    s = 5000 // q if q < 50 else 200 - 2 * q
    return np.clip((_BASE * s + 50) // 100, 1, 255).astype(np.uint16)


def scratch_bytes(B: int, H: int, W: int) -> int:
    """omt_jpeg_roundtrip_u8's scratch: B images' decoded Y plane and two half-size chroma planes, sides rounded to 16."""
    hp, wp = -(-H // 16) * 16, -(-W // 16) * 16
    return B * hp * wp * 3 // 2


def roundtrip_u8(images: torch.Tensor, quality: int = DEFAULT_QUALITY) -> torch.Tensor:
    """(B, H, W, 3) uint8 RGB on a CUDA device -> a new (B, H, W, 3) uint8 tensor: each image saved as a JPEG of this
    quality by Pillow and read back as RGB.  The scratch is kept per device and size (at most MAX_SCRATCH of them), so a
    later call of the same shape can be captured in a CUDA graph."""
    q = check_quality(quality, "roundtrip_u8")
    if not isinstance(images, torch.Tensor) or images.dtype != torch.uint8:
        raise TypeError(f"roundtrip_u8: expected uint8 images, got {getattr(images, 'dtype', type(images))}")
    if images.dim() != 4 or images.shape[-1] != 3:
        raise ValueError(f"roundtrip_u8: expected (B, H, W, 3) RGB images, got shape {tuple(images.shape)}")
    if images.device.type != "cuda":
        raise ValueError(f"roundtrip_u8: images on {images.device}, not a CUDA device")
    B, H, W, _ = (int(v) for v in images.shape)
    if H < 1 or W < 1:
        raise ValueError(f"roundtrip_u8: empty {H}x{W} images")
    out = torch.empty_like(images, memory_format=torch.contiguous_format)
    if B == 0:
        return out
    src = images.contiguous()
    tables = bounded(_tables, 100, q, lambda: np.ascontiguousarray(quant_tables(q)))
    n = scratch_bytes(B, H, W)
    scratch = bounded(_scratch, MAX_SCRATCH, (src.device, n),
                      lambda: torch.empty(n, dtype=torch.uint8, device=src.device))
    _cabi.call("omt_jpeg_roundtrip_u8", src, out, B, H, W, tables.ctypes.data, scratch)
    return out
