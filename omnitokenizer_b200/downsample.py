"""vqgan_eval.py's --infer_downsample on the device: the reconstructions scored at resolution / d.

* Video (:121-136, then :147-148): omt_eval_downsample turns the decoder's fp32 reconstruction, or the loader's uint8
  clips through the per-byte value table of their VideoNorm branch, into the uint8 clips get_fvd_logits takes,
  F.interpolate(scale_factor=1 / d) * 255 .byte() in torch's fp32 CPU arithmetic (layout.downsample_clips is its host
  twin).  With d = 1 the interpolation is the identity, so the same launch maps the real bytes alone.
* Images (:205-219): omt_resample_u8 with Pillow's LANCZOS tables (layout.eval_downsample_resize) on a batch of
  same-size images already on the device.

Every check runs before the first launch.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from . import _cabi
from . import layout as L
from .engine import DESC_WORDS
from .metricnet import bounded, clip_descs

FORM_F32, FORM_U8 = 0, 1        # OMT_DS_F32 / OMT_DS_U8
MAX_SETUPS = 16                 # descriptor sets kept per process; the oldest goes first
_setups = {}
_tables = {}


def real_value_table(norm: L.U8Norm) -> torch.Tensor:
    """fp32 [n_tab, 256]: batch['video'] + 0.5 (vqgan_eval.py:122) for every loader byte, the normalised value
    (layout.u8_norm_table, the pipeline's own op order) plus 0.5 in torch's fp32; one table per VideoNorm branch."""
    tab = L.u8_norm_table(norm, 3)
    if not bool((tab == tab[:, :1]).all()):
        raise ValueError(f"normalisation {norm.name!r} differs per channel; the downsample's value map is one table per "
                         f"branch")
    return (tab[:, 0] + 0.5).contiguous()


def out_size(H: int, W: int, d: int, what: str = "infer_downsample"):
    """(oh, ow) of an H x W frame at scale_factor 1 / d; refuses a factor that leaves no pixel."""
    g = L.downsample_geometry(int(H), int(W), int(d))
    if g.rh < 1 or g.rw < 1:
        raise ValueError(f"{what}: infer_downsample {d} of {H}x{W} frames leaves {g.rh}x{g.rw} pixels")
    return g.rh, g.rw


def _interp_setup(B: int, T: int, H: int, W: int, d: int, one_thread: bool, device):
    g = L.downsample_geometry(H, W, d)
    tab_host = torch.from_numpy(np.concatenate([L.clip_axis_table(H, g.rh, g.scale_h).reshape(-1),
                                                L.clip_axis_table(W, g.rw, g.scale_w).reshape(-1)]))
    desc_host = clip_descs(B, T * H * W * 3, H, W, g.rh, g.rw)
    desc_host[:, -1] = L.clip_interp_form(g, one_thread)
    return desc_host, tab_host, desc_host.to(device), tab_host.to(device)


def clips_u8(src: torch.Tensor, d: int, real_norm: Optional[L.U8Norm] = None, one_thread: Optional[bool] = None,
             what: str = "infer_downsample") -> torch.Tensor:
    """One omt_eval_downsample launch (two more for VideoNorm's per-clip test): (B, T, oh, ow, 3) uint8 on src's device.
    src: the decoder's fp32 reconstruction (B, 3, T, H, W) (real_norm None), or the loader's uint8 clips (B, T, H, W, 3)
    whose values are real_value_table(real_norm) picked per clip.  one_thread: the reference runs F.interpolate with
    torch on one thread, which picks torch's channels-last kernel for 3-channel frames (layout.clip_interp_form); None
    reads torch.get_num_threads() of this process.  The descriptors of a shape are built and uploaded on its first call,
    so a later call can be captured in a CUDA graph."""
    d = L.check_infer_downsample(d, what)
    if not isinstance(src, torch.Tensor) or src.dim() != 5 or src.device.type != "cuda" or not src.is_contiguous():
        raise ValueError(f"{what}: expected a contiguous 5-D CUDA tensor, got {getattr(src, 'shape', type(src))}")
    if real_norm is None:
        if src.dtype != torch.float32 or src.shape[1] != 3:
            raise ValueError(f"{what}: the reconstruction must be fp32 (B, 3, T, H, W), got {src.dtype} {tuple(src.shape)}")
        B, _, T, H, W = (int(v) for v in src.shape)
        form, lut, sel_needed = FORM_F32, None, False
    else:
        if src.dtype != torch.uint8 or src.shape[-1] != 3:
            raise ValueError(f"{what}: real clips must be uint8 (B, T, H, W, 3), got {src.dtype} {tuple(src.shape)}")
        B, T, H, W, _ = (int(v) for v in src.shape)
        form, sel_needed = FORM_U8, real_norm.max_test
        lut = bounded(_tables, MAX_SETUPS, (src.device, real_norm), lambda: real_value_table(real_norm).to(src.device))
    if min(B, T) < 1:
        raise ValueError(f"{what}: empty clip batch {tuple(src.shape)}")
    oh, ow = out_size(H, W, d, what)
    if one_thread is None:
        one_thread = torch.get_num_threads() == 1
    key = (src.device, B, T, H, W, d, bool(one_thread))
    desc_host, tab_host, desc, tab = bounded(_setups, MAX_SETUPS, key,
                                             lambda: _interp_setup(B, T, H, W, d, bool(one_thread), src.device))
    out = torch.empty(B, T, oh, ow, 3, dtype=torch.uint8, device=src.device)
    sel = None
    if sel_needed:
        sel = torch.empty(B, dtype=torch.int32, device=src.device)
        _cabi.call("omt_u8_norm_select", src, B, T * H * W * 3, sel)
    _cabi.call("omt_eval_downsample", src, src.numel(), form, desc, desc_host, tab, tab_host, tab_host.numel(), lut, sel,
               B, T, oh, ow, out)
    return out


def _image_setup(B: int, h: int, w: int, side: int, device):
    bounds_h, k_h = L.resample_coeffs(w, side, "antialias")
    bounds_v, k_v = L.resample_coeffs(h, side, "antialias")
    parts = [bounds_h.reshape(-1), k_h.reshape(-1), bounds_v.reshape(-1), k_v.reshape(-1)]
    offs = np.cumsum([0] + [p.size for p in parts])
    tab_host = torch.from_numpy(np.concatenate(parts).astype(np.int32))
    need_h, need_v = int(w != side), int(h != side)
    desc_host = torch.zeros(B, DESC_WORDS, dtype=torch.int32)
    desc_host[:, :2] = (torch.arange(B, dtype=torch.int64) * h * w * 3).view(torch.int32).view(B, 2)
    desc_host[:, 2:] = torch.tensor([h, w, side, side, 0, 0, 0, need_h, need_v,
                                     offs[0] if need_h else 0, offs[1] if need_h else 0, k_h.shape[1] if need_h else 0,
                                     offs[2] if need_v else 0, offs[3] if need_v else 0, k_v.shape[1] if need_v else 0,
                                     int(L.vertical_first(h, w, side, side))], dtype=torch.int32)
    return desc_host, tab_host, desc_host.to(device), tab_host.to(device)


def images_u8(images: torch.Tensor, d: int, what: str = "infer_downsample") -> torch.Tensor:
    """vqgan_eval.py:207-208 / :218-219 on the device: (B, h, w, 3) uint8 images of the eval resolution h == w ->
    img.resize((h // d, h // d), Image.ANTIALIAS), one omt_resample_u8 launch, (B, h // d, h // d, 3) uint8."""
    d = L.check_infer_downsample(d, what)
    if not isinstance(images, torch.Tensor) or images.dtype != torch.uint8 or images.dim() != 4 or images.shape[-1] != 3:
        raise ValueError(f"{what}: expected (B, h, w, 3) uint8 images, got {getattr(images, 'shape', type(images))}")
    if images.device.type != "cuda" or not images.is_contiguous():
        raise ValueError(f"{what}: expected contiguous images on a CUDA device, got them on {images.device}")
    B, h, w, _ = (int(v) for v in images.shape)
    if h != w:
        raise ValueError(f"{what}: the eval resizes square {h}x{h} images, got {h}x{w}")
    if B < 1:
        raise ValueError(f"{what}: empty image batch {tuple(images.shape)}")
    side = L.eval_downsample_resize(h, d).size[0]
    desc_host, tab_host, desc, tab = bounded(_setups, MAX_SETUPS, (images.device, "images", B, h, side),
                                             lambda: _image_setup(B, h, w, side, images.device))
    out = torch.empty(B, side, side, 3, dtype=torch.uint8, device=images.device)
    _cabi.call("omt_resample_u8", images, images.numel(), desc, desc_host, tab, tab_host, tab_host.numel(), B, side, side,
               out)
    return out
