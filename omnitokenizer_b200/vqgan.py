"""Drop-in `OmniTokenizer_VQGAN`: the reference's module API and checkpoint layout over the
omnitok_b200 CUDA kernels.

Mirrors /root/reference/OmniTokenizer/omnitokenizer.py:63-768 for the inference surface that
vqgan_eval.py, lm_transformer.py, transformer_eval.py and the DiT/Latte trainers touch:
``__init__(args)``, ``add_model_specific_args``, ``load_state_dict`` / ``state_dict`` (same key names
and shapes, including the dead keys), ``load_from_checkpoint``, ``encode``, ``decode``,
``forward(x, log_image=True)`` and the attributes those callers poke.  The parameter containers
below define NO torch forward math -- every per-token operation runs in libomnitok_b200.so
(omnitokenizer_b200/engine.py); there is no CPU or eager fallback.

Out of scope (SURVEY.md 8): GAN training (discriminators, LPIPS, optimizers).  Their checkpoint
keys are reported as `unexpected_keys` by ``load_state_dict(strict=False)``, which is how
vqgan_eval.py:62-71 already loads.
"""
from __future__ import annotations

import argparse
import random
import math
from typing import Optional

import torch
import torch.nn as nn

from . import layout as L
from .consumers import EVAL_U8, IMAGE_NORM, LATTE_NORM, VIDEO_NORM
from .engine import Engine


# --------------------------------------------------------------------------------------------
# parameter containers (names == reference state_dict keys; SURVEY.md Appendix B)
# --------------------------------------------------------------------------------------------

class _Slot(nn.Module):
    """Parameter-free placeholder for the reference's Rearrange / GEGLU / Dropout entries so that
    nn.Sequential indices (and therefore state_dict keys) line up."""


class _GammaBetaNorm(nn.Module):          # modules/attention.py:73-80
    def __init__(self, dim):
        super().__init__()
        self.gamma = nn.Parameter(torch.ones(dim))
        self.register_buffer("beta", torch.zeros(dim))


class _PEG(nn.Module):                    # modules/attention.py:298-302
    def __init__(self, dim):
        super().__init__()
        self.dsconv = nn.Conv3d(dim, dim, 3, groups=dim)


class _ContinuousPositionBias(nn.Module):  # modules/attention.py:535-560 (dead under SDPA; keys kept)
    def __init__(self, dim, heads, layers=2):
        super().__init__()
        self.net = nn.ModuleList([])
        self.net.append(nn.Sequential(nn.Linear(2, dim), nn.LeakyReLU(0.1)))
        for _ in range(layers - 1):
            self.net.append(nn.Sequential(nn.Linear(dim, dim), nn.LeakyReLU(0.1)))
        self.net.append(nn.Linear(dim, heads))


class _Attention(nn.Module):              # modules/attention.py:342-393
    def __init__(self, dim, dim_head, heads, spatial_pos):
        super().__init__()
        inner = dim_head * heads
        if spatial_pos == "rel":
            self.spatial_rel_pos_bias = _ContinuousPositionBias(dim=dim, heads=heads)
        self.norm = _GammaBetaNorm(dim)
        self.context_norm = _GammaBetaNorm(dim)
        self.to_q = nn.Linear(dim, inner, bias=False)
        self.to_kv = nn.Linear(dim, inner * 2, bias=False)
        self.q_scale = nn.Parameter(torch.ones(dim_head))
        self.k_scale = nn.Parameter(torch.ones(dim_head))
        self.to_out = nn.Linear(inner, dim, bias=False)


class _WindowAttention(nn.Module):        # modules/attention.py:216-252
    def __init__(self, dim, window_size, heads):
        super().__init__()
        ws = window_size
        self.norm = _GammaBetaNorm(dim)
        self.relative_position_bias_table = nn.Parameter(torch.zeros((2 * ws - 1) * (2 * ws - 1), heads))
        coords = torch.stack(torch.meshgrid(torch.arange(ws), torch.arange(ws), indexing="ij")).flatten(1)
        rel = (coords[:, :, None] - coords[:, None, :]).permute(1, 2, 0).contiguous()
        rel[:, :, 0] += ws - 1
        rel[:, :, 1] += ws - 1
        rel[:, :, 0] *= 2 * ws - 1
        self.register_buffer("relative_position_index", rel.sum(-1))
        self.qkv = nn.Linear(dim, dim * 3, bias=False)
        self.proj = nn.Linear(dim, dim)
        nn.init.trunc_normal_(self.relative_position_bias_table, std=0.02)


def _feed_forward(dim, mult):             # modules/attention.py:159-168
    inner = int(mult * (2 / 3) * dim)
    return nn.Sequential(nn.LayerNorm(dim), nn.Linear(dim, inner * 2, bias=False), _Slot(), _Slot(),
                         nn.Linear(inner, dim, bias=False))


class _Transformer(nn.Module):            # modules/attention.py:588-652
    def __init__(self, dim, block, dim_head, heads, ff_mult, window_size, spatial_pos):
        super().__init__()
        self.layers = nn.ModuleList([])
        for blk in block:
            if blk == "t":
                self.layers.append(nn.ModuleList([_PEG(dim), _Attention(dim, dim_head, heads, spatial_pos), None,
                                                  _feed_forward(dim, ff_mult)]))
            elif blk == "w":
                self.layers.append(nn.ModuleList([None, _WindowAttention(dim, window_size, heads), None,
                                                  _feed_forward(dim, ff_mult)]))
            else:
                raise NotImplementedError(
                    f"transformer block {blk!r}: pooling ('a','m','l') / upsampling ('n','r') blocks are used by no "
                    f"shipped config and are not implemented")
        self.block = block
        self.norm_out = _GammaBetaNorm(dim)


def _pair(v):
    return v if isinstance(v, tuple) else (v, v)


def _check_patch_embed(a):
    if a.patch_embed not in ("linear", "cnn"):
        raise NotImplementedError(f"patch_embed={a.patch_embed!r}: the reference itself raises for anything but linear / cnn")
    if a.patch_embed == "cnn" and getattr(a, "norm_type", "batch") != "batch":
        # Normalize(image_channels=3, 'group') is GroupNorm(32 groups, 3 channels): the reference cannot even construct it
        raise NotImplementedError("patch_embed='cnn' needs --norm_type batch (GroupNorm(32, 3) is invalid in the reference too)")


class OmniTokenizer_Encoder(nn.Module):   # omnitokenizer.py:772-868
    def __init__(self, a):
        super().__init__()
        _check_patch_embed(a)
        self.image_size = _pair(a.resolution)
        self.patch_size = _pair(a.patch_size)
        self.temporal_patch_size = a.temporal_patch_size
        self.block = a.enc_block
        k = a.image_channels * a.patch_size * a.patch_size
        dim = a.embedding_dim
        p, pt = a.patch_size, a.temporal_patch_size
        if a.patch_embed == "cnn":      # omnitokenizer.py:823-838: Conv3d + Normalize('batch' = SyncBatchNorm) + Rearrange
            self.to_patch_emb_first_frame = nn.Sequential(nn.Conv3d(a.image_channels, dim, (1, p, p), stride=(1, p, p)),
                                                          nn.BatchNorm3d(dim), _Slot())
            self.to_patch_emb = nn.Sequential(nn.Conv3d(a.image_channels, dim, (pt, p, p), stride=(pt, p, p)),
                                              nn.BatchNorm3d(dim), _Slot())
        else:
            self.to_patch_emb_first_frame = nn.Sequential(_Slot(), nn.LayerNorm(k), nn.Linear(k, dim), nn.LayerNorm(dim))
            self.to_patch_emb = nn.Sequential(_Slot(), nn.LayerNorm(k * pt), nn.Linear(k * pt, dim), nn.LayerNorm(dim))
        kw = dict(dim=dim, dim_head=a.dim_head, heads=a.heads, ff_mult=a.ff_mult, window_size=a.twod_window_size)
        self.enc_spatial_transformer = _Transformer(block=a.enc_block, spatial_pos=a.spatial_pos, **kw)
        # temporal transformers are built without spatial_pos -> default "rel" -> dead bias-MLP keys
        self.enc_temporal_transformer = _Transformer(block="t" * a.temporal_depth, spatial_pos="rel", **kw)


class OmniTokenizer_Decoder(nn.Module):   # omnitokenizer.py:950-1035
    def __init__(self, a):
        super().__init__()
        self.image_size = _pair(a.resolution)
        self.patch_size = _pair(a.patch_size)
        self.block = a.dec_block
        k = a.image_channels * a.patch_size * a.patch_size
        dim = a.embedding_dim
        kw = dict(dim=dim, dim_head=a.dim_head, heads=a.heads, ff_mult=a.ff_mult, window_size=a.twod_window_size)
        self.dec_spatial_transformer = _Transformer(block=a.dec_block, spatial_pos=a.spatial_pos, **kw)
        self.dec_temporal_transformer = _Transformer(block="t" * a.temporal_depth, spatial_pos="rel", **kw)
        _check_patch_embed(a)
        p, pt = a.patch_size, a.temporal_patch_size
        if a.patch_embed == "cnn":      # omnitokenizer.py:1019-1035: Rearrange + ConvTranspose3d + Normalize(channels)
            self.to_pixels_first_frame = nn.Sequential(_Slot(), nn.ConvTranspose3d(dim, a.image_channels, (1, p, p),
                                                                                  stride=(1, p, p)), nn.BatchNorm3d(a.image_channels))
            self.to_pixels = nn.Sequential(_Slot(), nn.ConvTranspose3d(dim, a.image_channels, (pt, p, p), stride=(pt, p, p)),
                                           nn.BatchNorm3d(a.image_channels))
        else:
            self.to_pixels_first_frame = nn.Sequential(nn.Linear(dim, k), _Slot())
            self.to_pixels = nn.Sequential(nn.Linear(dim, k * pt), _Slot())


class Codebook(nn.Module):                # modules/codebook.py:11-28
    def __init__(self, n_codes, embedding_dim, no_random_restart=False, restart_thres=1.0, usage_sigma=0.99):
        super().__init__()
        self.register_buffer("embeddings", torch.randn(n_codes, embedding_dim))
        self.register_buffer("N", torch.zeros(n_codes))
        self.register_buffer("z_avg", self.embeddings.data.clone())
        self.register_buffer("codebook_usage", torch.zeros(n_codes))
        self.call_cnt = 0
        self.usage_sigma = usage_sigma
        self.n_codes = n_codes
        self.embedding_dim = embedding_dim
        self._need_init = True
        self.no_random_restart = no_random_restart
        self.restart_thres = restart_thres

    def dictionary_lookup(self, encodings):
        return torch.nn.functional.embedding(encodings, self.embeddings)


_BACKFILL = dict(twod_window_size=4, defer_temporal_pool=False, defer_spatial_pool=False, spatial_pos="rel",
                 logitslaplace_weight=0.0, gen_upscale=None, initialize_vit=False, use_vae=False, kl_weight=0.000001,
                 apply_diffaug=False, apply_noise=False, apply_blur=False, sigmoid_in_disc=False,
                 activation_in_disc="leaky_relu", video_perceptual_weight=0.0, grad_clip_val_disc=1.0,
                 disloss_check_thres=None, perloss_check_thres=None, recloss_check_thres=None, resolution_scale=None)


class OmniTokenizer_VQGAN(nn.Module):
    """H100-native stand-in for OmniTokenizer.OmniTokenizer_VQGAN (omnitokenizer.py:63)."""

    def __init__(self, args):
        super().__init__()
        self.args = args
        # same hasattr back-fills as the reference so old checkpoints' Namespaces construct (omnitokenizer.py:70-236)
        if not hasattr(args, "enc_block"):
            args.enc_block = "t" * args.spatial_depth
        if not hasattr(args, "dec_block"):
            args.dec_block = "t" * args.spatial_depth
        for k, v in _BACKFILL.items():
            if not hasattr(args, k):
                setattr(args, k, v)
        for k, v in dict(patch_embed="linear", attn_dropout=0.0, ff_dropout=0.0, ff_mult=4.0, dim_head=64, heads=8,
                         image_channels=3, use_external_codebook=False, l2_code=False, no_random_restart=False,
                         restart_thres=1.0, causal_in_temporal_transformer=False, causal_in_peg=False,
                         temporal_depth=4, sample_every_n_frames=1, downsample=(4, 4, 4)).items():
            if not hasattr(args, k):
                setattr(args, k, v)
        self.embedding_dim = args.embedding_dim
        self.n_codes = args.n_codes
        self.logitslaplace_weight = args.logitslaplace_weight
        self.gen_upscale = args.gen_upscale
        self.resolution = args.resolution
        self.patch_size = args.patch_size
        self.resolution_scale = args.resolution_scale
        if args.defer_temporal_pool or args.defer_spatial_pool or args.gen_upscale is not None:
            raise NotImplementedError("defer_*_pool / gen_upscale are multi-resolution training options that change the "
                                      "architecture (pooling / upsampling blocks), outside the encode/decode hot path "
                                      "(SURVEY.md 8f.4)")
        if args.use_external_codebook:
            raise NotImplementedError("--use_external_codebook (vendored lucidrains quantizers) is never set by the shipped "
                                      "scripts and is out of scope")
        self.encoder = OmniTokenizer_Encoder(args)
        self.decoder = OmniTokenizer_Decoder(args)
        self.use_vae = args.use_vae
        self.kl_weight = args.kl_weight
        self.codebook = Codebook(args.n_codes, args.codebook_dim, no_random_restart=args.no_random_restart,
                                 restart_thres=args.restart_thres)
        out = args.codebook_dim * 2 if self.use_vae else args.codebook_dim
        self.pre_vq_conv = nn.Sequential(_Slot(), nn.Linear(args.embedding_dim, out), _Slot())
        self.post_vq_conv = nn.Sequential(_Slot(), nn.Linear(args.codebook_dim, args.embedding_dim), _Slot())
        self.use_external_codebook = args.use_external_codebook
        self.l2_code = args.l2_code
        self.hparams = argparse.Namespace(args=args)
        self._engine: Optional[Engine] = None
        self._engine_key = None
        self.requires_grad_(False)      # inference module: the CUDA path has no autograd

    # ---------------------------------------------------------------- plumbing
    @property
    def device(self):
        return self.codebook.embeddings.device

    @property
    def latent_shape(self):               # omnitokenizer.py:239-245
        a = self.args
        inp = (a.sequence_length // a.sample_every_n_frames, a.resolution, a.resolution)
        return tuple(s // d for s, d in zip(inp, a.downsample))

    def _apply(self, fn, *a, **k):
        self._engine = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        self._engine = None
        return super().load_state_dict(state_dict, strict=strict, **kw)

    @classmethod
    def load_from_checkpoint(cls, path, strict: bool = False, map_location="cpu", **kw):
        """Lightning-style loader (download.py:49, README.md:66): ckpt['hyper_parameters']['args'] + ['state_dict']."""
        ckpt = torch.load(path, map_location=map_location, weights_only=False)
        model = cls(ckpt["hyper_parameters"]["args"])
        model.load_state_dict(ckpt["state_dict"], strict=strict)
        return model

    def engine(self) -> Engine:
        """Packed-weight engine; rebuilt when weights / device / VAE mode change."""
        dev = self.device
        if dev.type != "cuda":
            raise RuntimeError("OmniTokenizer_VQGAN (omnitok_b200) runs on a CUDA device only; move the module with "
                               ".cuda() first -- there is no CPU fallback")
        key = (dev, bool(self.use_vae), sum(p._version for p in self.parameters()),
               self.codebook.embeddings.data_ptr(), self.codebook.embeddings._version)
        if self._engine is None or self._engine_key != key:
            with torch.cuda.device(dev):
                self._engine = Engine(self, dev)
            self._engine_key = key
        return self._engine

    def prepare(self):
        """Pack weights now (otherwise done lazily on first encode/decode)."""
        self.engine()
        return self

    def _track_usage(self, counts, M):
        """Eval-time side effects of Codebook.forward (modules/codebook.py:122-140): batch usage from the fixed-size
        histogram the search kernel filled (replaces torch.unique, no host sync), EMA of codebook_usage, call_cnt."""
        cb = self.codebook
        usage = counts[:cb.n_codes].float() / M
        if cb.call_cnt == 0:
            cb.codebook_usage.data = usage
        else:
            cb.codebook_usage.data = cb.usage_sigma * cb.codebook_usage.data + (1 - cb.usage_sigma) * usage
        cb.call_cnt += 1
        return usage

    def _empty_encode(self, x, is_image, include_embeddings):
        """B == 0 (a surplus rank of a batch-sharded run): right-shaped empty results, no kernel launch."""
        a = self.args
        T = 1 if is_image else x.shape[2]
        Tp, h, w = 1 + (T - 1) // a.temporal_patch_size, x.shape[-2] // a.patch_size, x.shape[-1] // a.patch_size
        if self.use_vae:
            shape = (0, a.codebook_dim, h, w) if is_image else (0, a.codebook_dim, Tp, h, w)
            return torch.empty(shape, device=self.device)
        enc = torch.empty((0, Tp, h, w), dtype=torch.int64, device=self.device)
        if include_embeddings:
            return torch.empty((0, a.codebook_dim, Tp, h, w), device=self.device), enc
        return enc

    # ---------------------------------------------------------------- the hot path
    @torch.no_grad()
    def encode(self, x, is_image, include_embeddings=False):
        """omnitokenizer.py:247-266."""
        eng = self.engine()
        if x.shape[0] == 0:
            return self._empty_encode(x, is_image, include_embeddings)
        with torch.cuda.device(self.device):
            xv = x.unsqueeze(2) if is_image else x
            ws, dims = eng.encode(xv.float(), "raw" if self.use_vae else "vq")
            return self._encode_result(eng, ws.idx, eng.z_view(ws), ws.counts, dims, is_image, include_embeddings)

    def _u8_frames(self, frames, is_image):
        """Checks uint8 frames (B, T, H, W, C) / images (B, H, W, C) and returns them as (B, T, H, W, C)."""
        if not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8:
            raise TypeError(f"expected uint8 frames, got {getattr(frames, 'dtype', type(frames))}")
        if frames.ndim != (4 if is_image else 5):
            raise ValueError(f"expected {'(B, H, W, C)' if is_image else '(B, T, H, W, C)'} frames, got {tuple(frames.shape)}")
        if frames.shape[-1] != self.args.image_channels:
            raise ValueError(f"expected {self.args.image_channels} channels (last dimension), got {frames.shape[-1]}")
        return frames.unsqueeze(1) if is_image else frames

    @torch.no_grad()
    def encode_u8(self, frames, is_image, include_embeddings=False, norm=VIDEO_NORM):
        """encode() straight from the uint8 frames the data loaders produce: (B, T, H, W, C), or (B, H, W, C) images,
        channels last (decord / PIL / decode_u8 layout).  The patch-gather kernel applies the loader's normalisation
        `norm` (a layout.U8Norm; default VIDEO_NORM, VideoNorm of the reference's video datasets) by table
        lookup, so the result -- codes, embeddings, VAE latents, usage statistics, CPU RNG draws -- is exactly
        encode(norm(frames) as (B, C, T, H, W) fp32, is_image, include_embeddings).  The copy to the device is 4x smaller."""
        f = self._u8_frames(frames, is_image)
        eng = self.engine()
        if f.shape[0] == 0:
            shape = (0, f.shape[4], f.shape[2], f.shape[3]) if is_image else (0, f.shape[4], f.shape[1], f.shape[2], f.shape[3])
            return self._empty_encode(torch.empty(shape, device="meta"), is_image, include_embeddings)
        with torch.cuda.device(self.device):
            ws, dims = eng.encode_u8(f, "raw" if self.use_vae else "vq", norm)
            return self._encode_result(eng, ws.idx, eng.z_view(ws), ws.counts, dims, is_image, include_embeddings)

    def _images_u8(self, images, resize, params):
        """Checks a ragged list of decoded uint8 images (H_i, W_i, C) in host memory, the transform and its parameters, and
        the output size against encode's shape rules (with encode's messages) -- all before any launch.  Returns (list,
        params), drawing the parameters from the CPU generator as the loader's transforms would when params is None."""
        from .jpeg import Pending
        images = list(images)
        L.check_resize(resize)
        C = self.args.image_channels
        for i, im in enumerate(images):
            if isinstance(im, Pending):             # a JPEG file of encode_jpeg_u8 / forward_jpeg_u8, decoded to RGB
                if C != 3:
                    raise ValueError(f"image {i}: a JPEG decodes to 3 channels; the model takes {C}")
                continue
            if not isinstance(im, torch.Tensor) or im.dtype != torch.uint8:
                raise TypeError(f"image {i}: expected a uint8 tensor, got {getattr(im, 'dtype', type(im))}")
            if im.ndim != 3 or im.shape[2] != C or im.shape[0] < 1 or im.shape[1] < 1:
                raise ValueError(f"image {i}: expected (H, W, {C}) with H, W >= 1, got {tuple(im.shape)}")
            if im.device.type != "cpu":
                raise ValueError(f"image {i}: expected a decoded image in host memory, got one on {im.device}")
        h, w = resize.out_size
        eng = self.engine()
        eng._shape((max(len(images), 1), C, 1, h, w))
        if params is None:
            params = L.resize_params(len(images), resize)
        L.check_resize_params(params, len(images), resize)
        return images, params

    @torch.no_grad()
    def encode_images_u8(self, images, resize, norm=IMAGE_NORM, include_embeddings=False, params=None):
        """encode_u8(images after the loader's transform, is_image=True) from the decoded images themselves: a ragged list of
        (H_i, W_i, C) uint8 tensors in host memory, any sizes.  `resize` (a layout.U8Resize, e.g. layout.image_resize(res))
        is the loader's Pillow resize + random crop + flip; omt_resample_u8 applies it on the device byte for byte as Pillow
        and torchvision do, so the result -- codes, embeddings, VAE latents, usage statistics, CPU RNG draws -- equals
        encode_u8 of the stacked host-transformed images.  params: per image (top, left, flip); None draws them from the
        CPU generator as RandomCrop / RandomHorizontalFlip would (layout.resize_params), before the VAE noise."""
        return self._encode_images(images, None, resize, norm, include_embeddings, params)

    @torch.no_grad()
    def encode_jpeg_u8(self, sources, resize, norm=IMAGE_NORM, include_embeddings=False, params=None):
        """encode_images_u8 of Image.open(f).convert("RGB") of each source, decoded on the device: sources is a list of
        JPEG files (bytes-like or paths, jpeg.decode_u8's forms) and, where a caller decoded a file itself (e.g. one
        jpeg.probe refuses), (H, W, 3) uint8 host tensors.  The files are parsed first (a refused or malformed one raises
        before any launch), then decoded straight into omt_resample_u8's packed source; the result -- codes, embeddings,
        VAE latents, usage statistics, CPU RNG draws -- equals encode_images_u8 of Pillow's decoded images."""
        from . import jpeg
        images, jpegs = jpeg.split_sources(sources)
        return self._encode_images(images, jpegs, resize, norm, include_embeddings, params)

    def _encode_images(self, images, jpegs, resize, norm, include_embeddings, params):
        images, params = self._images_u8(images, resize, params)
        if not images:
            h, w = resize.out_size
            return self.encode_u8(torch.empty((0, h, w, self.args.image_channels), dtype=torch.uint8), True,
                                  include_embeddings, norm)
        eng = self.engine()
        with torch.cuda.device(self.device):
            ws, dims = eng.encode_images_u8(images, resize, params, "raw" if self.use_vae else "vq", norm, jpegs)
            return self._encode_result(eng, ws.idx, eng.z_view(ws), ws.counts, dims, True, include_embeddings)

    @torch.no_grad()
    def encode_clips_u8(self, clips, resize, norm=LATTE_NORM, include_embeddings=False, params=None):
        """encode(x, is_image=False) of the clips Latte's video loaders make of their decoded frames, from the decoded
        frames themselves: a list of (F, H_i, W_i, C) uint8 tensors in host memory (read_video's frames, channels last),
        the same F for every clip, any frame sizes.  `resize` (a layout.ClipResize, e.g. layout.ucf_clip_resize(256)) is
        the loader's flip + bilinear resize + centre crop and `norm` its Normalize; omt_resample_clips applies them on the
        device bit for bit as torch does on the CPU, so the result -- codes, embeddings, VAE latents, usage statistics,
        CPU RNG draws -- equals encode of the stacked pipeline output rearranged 'b f c h w -> b c f h w'.  params: per
        clip, whether it is flipped; None draws them from Python's random as RandomHorizontalFlipVideo does
        (layout.clip_params).  Everything is checked, with encode's messages, before any launch."""
        clips = list(clips)
        L.check_clip_resize(resize)
        C = self.args.image_channels
        if not clips:
            raise ValueError("encode_clips_u8 needs at least one clip")
        for i, c in enumerate(clips):
            if not isinstance(c, torch.Tensor) or c.dtype != torch.uint8:
                raise TypeError(f"clip {i}: expected a uint8 tensor, got {getattr(c, 'dtype', type(c))}")
            if c.ndim != 4 or c.shape[3] != C or min(c.shape[:3]) < 1:
                raise ValueError(f"clip {i}: expected (F, H, W, {C}) with F, H, W >= 1, got {tuple(c.shape)}")
            if c.device.type != "cpu":
                raise ValueError(f"clip {i}: expected decoded frames in host memory, got a clip on {c.device}")
            if c.shape[0] != clips[0].shape[0]:
                raise ValueError(f"every clip must have the same number of frames: {clips[0].shape[0]} and {c.shape[0]}")
        sizes = {tuple(L.clip_out_size(int(c.shape[1]), int(c.shape[2]), resize)) for c in clips}
        if len(sizes) > 1:
            raise ValueError(f"the clips come out at different sizes {sorted(sizes)}: without a resize every clip must "
                             f"have the same frame size")
        for c in clips:
            L.clip_geometry(int(c.shape[1]), int(c.shape[2]), resize)      # the reference's center_crop ValueError
        L.clip_norm_table(norm)
        eng = self.engine()
        eng._shape((len(clips), C, int(clips[0].shape[0])) + sizes.pop())
        if params is None:
            params = L.clip_params(len(clips), resize)
        L.check_clip_params(params, len(clips), resize)
        with torch.cuda.device(self.device):
            ws, dims = eng.encode_clips_u8(clips, resize, params, "raw" if self.use_vae else "vq", norm)
            return self._encode_result(eng, ws.idx, eng.z_view(ws), ws.counts, dims, False, include_embeddings)

    def _encode_result(self, eng, idx, z, counts, dims, is_image, include_embeddings):
        """What encode() returns (omnitokenizer.py:247-266), with Codebook.forward's usage side effects, from the encoder's
        rows of the dims (B,T',h,w) batch: idx [M] codes, z [M, cd] (VQ) or [M, 2 cd] moments (VAE), counts the code histogram."""
        B, Tp, h, w = dims
        if not self.use_vae:
            enc = idx.view(B, Tp, h, w).clone()
            self._track_usage(counts, idx.numel())           # Codebook.forward runs inside encode() too
            if include_embeddings:
                e = eng.E[idx]
                st = (e - z) + z
                return st.view(B, Tp, h, w, -1).permute(0, 4, 1, 2, 3).contiguous(), enc
            return enc
        hpar = z                                                              # (M, 2*cd) moments
        c = hpar.shape[1] // 2
        hpar = hpar.view(B, Tp, h, w, 2 * c).permute(0, 4, 1, 2, 3)
        mean, logvar = hpar[:, :c], torch.clamp(hpar[:, c:], -30.0, 20.0)     # vae.py:7-8
        noise = torch.randn(mean.shape).to(device=self.device)                # CPU generator, vae.py:16
        z = mean + torch.exp(0.5 * logvar) * noise
        return z.squeeze(2) if is_image else z.contiguous()

    @torch.no_grad()
    def encode_batch(self, xs, include_embeddings=False):
        """encode() of a mixed list in ONE pass: xs[i] is an image (C, H, W) or a video (C, T, H, W), every element with the
        same H x W and channel count (clip lengths may differ).  Returns a list in input order; element i is what
        encode(xs[i][None], is_image)[0] returns -- codes (T', h, w), the (embeddings, codes) pair with include_embeddings,
        or VAE latents (c, h, w) / (c, T', h, w) -- except that image codes (and embeddings) come without the frame axis,
        (h, w) and (cd, h, w), the form decode_batch takes for an image.  Bit for bit, with the side effects of the
        sequential calls: codebook_usage / call_cnt move once per element in input order, VAE noise is drawn from the CPU
        generator per element in input order.  Every element is checked (with encode's messages) before any launch."""
        xs = list(xs)
        if not xs:
            return []
        eng = self.engine()
        cin = self.args.image_channels
        for x in xs:
            if x.ndim not in (3, 4):
                raise ValueError(f"encode_batch takes images (C, H, W) and videos (C, T, H, W), got {tuple(x.shape)}")
            if x.shape[0] != cin:
                raise ValueError(f"expected {cin} channels, got {x.shape[0]}")
            if tuple(x.shape[-2:]) != tuple(xs[0].shape[-2:]):
                raise ValueError(f"every element of a batch must have the same frame size: "
                                 f"{tuple(xs[0].shape[-2:])} and {tuple(x.shape[-2:])}")
        with torch.cuda.device(self.device):
            ws, lay = eng.encode_batch([x.unsqueeze(1) if x.ndim == 3 else x for x in xs], "raw" if self.use_vae else "vq")
            z, hist = eng.z_view(ws), None
            if not self.use_vae:          # per-element code histograms (sorted order) from the packed codes: one scatter, no host sync
                n = self.codebook.n_codes
                hist = torch.zeros(lay.B * n, dtype=torch.int64, device=self.device)
                hist = hist.scatter_add_(0, eng.row_sample(ws, lay) * n + ws.idx, torch.ones_like(ws.idx)).view(lay.B, n)
            out = []
            for i, x in enumerate(xs):
                r, is_image = lay.rows(i), x.ndim == 3
                res = self._encode_result(eng, ws.idx[r], z[r], None if hist is None else hist[lay.pos[i]],
                                          (1, lay.tps[i], lay.h, lay.w), is_image, include_embeddings)
                if self.use_vae:
                    out.append(res[0])
                elif include_embeddings:
                    out.append((res[0][0, :, 0], res[1][0, 0]) if is_image else (res[0][0], res[1][0]))
                else:
                    out.append(res[0, 0] if is_image else res[0])
            return out

    def _check_cnn_grid(self, h, w):
        # the cnn decoder's Rearrange pins h to image_size // patch_size (omnitokenizer.py:1021): other grids raise there
        if self.args.patch_embed == "cnn" and h != self.resolution // self.patch_size:
            raise ValueError(f"patch_embed='cnn' decodes only the configured resolution ({self.resolution}): "
                             f"token grid {h}x{w} != {self.resolution // self.patch_size}")

    def _decode_inputs(self, encodings, is_image):
        """The index / flat-index / VAE 4-D 'b c h w' / 5-D 'b t h w c' conventions of omnitokenizer.py:268-317
        -> (dims (B,T',h,w), idx [M] | None, zc [M, cd] | None)."""
        if not self.use_vae:
            enc = encodings
            if enc.ndim == 2:
                B = enc.shape[0]
                if is_image:
                    h = w = int(math.sqrt(enc.shape[1])); Tp = 1
                else:
                    h = w = self.resolution // self.patch_size; Tp = enc.shape[1] // (h * w)
            elif enc.ndim == 3 and is_image:                                   # (B, h, w) is not a reference form
                raise ValueError("image indices must be (B, h*w) or (B, 1, h, w)")
            else:
                B, Tp, h, w = enc.shape
            self._check_cnn_grid(h, w)
            idx = enc.reshape(-1).to(device=self.device, dtype=torch.int64)
            if B > 0:
                # F.embedding device-asserts on out-of-range indices (omnitokenizer.py:270); same here, without a host sync
                torch._assert_async(((idx >= 0) & (idx < self.codebook.n_codes)).all(),
                                    "decode: code index out of range [0, n_codes)")
            return (B, Tp, h, w), idx, None
        z = encodings.to(device=self.device, dtype=torch.float32)
        if is_image:
            if z.ndim == 3:
                B = z.shape[0]; h = w = int(math.sqrt(z.shape[1])); Tp = 1
                zc = z.reshape(B * h * w, -1)
            else:
                B, c, h, w = z.shape; Tp = 1
                zc = z.permute(0, 2, 3, 1).reshape(B * h * w, c)
        else:
            if z.ndim == 3:
                B = z.shape[0]; h = w = self.resolution // self.patch_size; Tp = z.shape[1] // (h * w)
                zc = z.reshape(B * Tp * h * w, -1)
            else:
                B, Tp, h, w, c = z.shape
                zc = z.reshape(B * Tp * h * w, c)
        self._check_cnn_grid(h, w)
        return (B, Tp, h, w), None, zc

    def _decode(self, encodings, is_image, u8=None):
        eng = self.engine()
        with torch.cuda.device(self.device):
            dims, idx, zc = self._decode_inputs(encodings, is_image)
            B, Tp, h, w = dims
            if B == 0:
                T, H, W = 1 + (Tp - 1) * self.args.temporal_patch_size, h * self.patch_size, w * self.patch_size
                if u8 is not None:
                    return torch.empty((0, T, H, W, self.args.image_channels), dtype=torch.uint8, device=self.device)
                video = torch.empty((0, self.args.image_channels, T, H, W), device=self.device)
                return video.squeeze(2) if is_image else video
            return eng.decode(dims, idx=idx, zc=zc, u8=u8)

    @torch.no_grad()
    def decode(self, encodings, is_image):
        """omnitokenizer.py:268-317 (index / flat-index / VAE 4-D 'b c h w' / 5-D 'b t h w c' conventions)."""
        video = self._decode(encodings, is_image)
        return video.squeeze(2) if is_image else video

    @torch.no_grad()
    def decode_u8(self, encodings, is_image, affine=(1.0, 0.5, 0.0, 1.0, 255.0)):
        """decode() fused with the consumers' uint8 conversion: returns (B, T, H, W, C) uint8 (T = 1 for images) =
        trunc(clamp(x * mul + add, lo, hi) * post), bit-identical to the torch expression on decode()'s result.
        Default affine: vqgan_eval.py:139,147-148 `(clamp(x_recons + 0.5, 0, 1) * 255).byte()` in 'b t h w c' order;
        (255, 128, 0, 255, 1): DiT sample_ddp.py:163.  The device->host copy is 4x smaller than the fp32 video."""
        return self._decode(encodings, is_image, u8=affine)

    def _decode_batch(self, encodings, u8=None):
        """decode_batch / decode_u8_batch: element i in decode's form without the batch dimension -- VQ codes (h, w) of an
        image or (T', h, w) of a video, VAE latents (c, h, w) of an image or (T', h, w, c) of a video."""
        encs = list(encodings)
        if not encs:
            return []
        eng = self.engine()
        tps, is_image, grid = [], [], None
        img_ndim, forms = (3, "(c, h, w) / (T', h, w, c) latents") if self.use_vae else (2, "(h, w) / (T', h, w) codes")
        for e in encs:
            img = e.ndim == img_ndim
            if e.ndim != img_ndim + 1 and not img:
                raise ValueError(f"decode_batch takes {forms}, got {tuple(e.shape)}")
            if img:
                tp, g = 1, tuple(e.shape[-2:])
            else:
                tp, g = e.shape[0], tuple(e.shape[1:3])
            if grid is not None and g != grid:
                raise ValueError(f"every element of a batch must have the same token grid: {grid} and {g}")
            grid = g
            self._check_cnn_grid(*g)
            eng._check_latent_frames(int(tp))
            tps.append(int(tp))
            is_image.append(img)
        eng._check_packed(tps)
        h, w = grid
        with torch.cuda.device(self.device):
            if not self.use_vae:
                idx = [e.reshape(-1).to(device=self.device, dtype=torch.int64) for e in encs]
                allidx = torch.cat(idx)
                torch._assert_async(((allidx >= 0) & (allidx < self.codebook.n_codes)).all(),
                                    "decode: code index out of range [0, n_codes)")
                outs = eng.decode_batch(tps, h, w, idx=idx, u8=u8)
            else:
                # rows (t, h, w) x latent channels, as decode reads the 4-D 'b c h w' / 5-D 'b t h w c' forms
                zc = [(e.permute(1, 2, 0) if img else e).to(device=self.device, dtype=torch.float32) for e, img in zip(encs, is_image)]
                zc = [z.reshape(-1, z.shape[-1]) for z in zc]
                outs = eng.decode_batch(tps, h, w, zc=zc, u8=u8)
        return [o.squeeze(1) if img and u8 is None else o for o, img in zip(outs, is_image)]

    @torch.no_grad()
    def decode_batch(self, encodings):
        """decode() of a mixed list in ONE pass; element i is what decode(encodings[i][None], is_image)[0] returns, bit for
        bit: (C, H, W) for an image, (C, T, H, W) for a video.  Forms of the elements: see _decode_batch (the forms
        encode_batch returns, with VAE video latents as decode takes them, 't h w c')."""
        return self._decode_batch(encodings)

    @torch.no_grad()
    def decode_u8_batch(self, encodings, affine=(1.0, 0.5, 0.0, 1.0, 255.0)):
        """decode_u8() of a mixed list in ONE pass: element i is decode_u8(encodings[i][None], is_image, affine)[0],
        uint8 (T, H, W, C) with T = 1 for images."""
        return self._decode_batch(encodings, u8=tuple(float(v) for v in affine))

    @torch.no_grad()
    def forward(self, x, optimizer_idx=None, log_image=False):
        """omnitokenizer.py:330-413, inference form (log_image=True).  The training branches
        (optimizer_idx 0/1: GAN / perceptual losses) are out of scope."""
        if optimizer_idx is not None or not log_image:
            raise NotImplementedError("only forward(x, log_image=True) (the vqgan_eval.py call) is implemented; the GAN "
                                      "training step is out of scope")
        eng = self.engine()
        is_image = x.ndim == 4
        if self.resolution_scale is not None:
            # multi-resolution option (omnitokenizer.py:334-355): ONE random.choices draw per call picks the scale, every
            # frame is resized bilinearly (align_corners=True) before the encoder; x is returned at that resolution
            scale = random.choices(self.resolution_scale)[0]
            side = int(x.shape[-2] * scale)
            flat = x if is_image else x.permute(0, 2, 1, 3, 4).reshape(-1, x.shape[1], x.shape[3], x.shape[4])
            flat = torch.nn.functional.interpolate(flat.float(), size=(side, side), mode="bilinear", align_corners=True)
            x = flat if is_image else flat.reshape(x.shape[0], x.shape[2], x.shape[1], side, side).permute(0, 2, 1, 3, 4).contiguous()
        with torch.cuda.device(self.device):
            xv = (x.unsqueeze(2) if is_image else x).float()
            ws, dims = eng.encode(xv, "raw" if self.use_vae else "vq")
            B = dims[0]
            x_recon, vq_output = self._forward_decode(eng, ws, dims)
            if is_image:
                x_recon = x_recon.squeeze(2)
                frames, frames_recon = x, x_recon
            else:
                T = x.shape[2]
                frame_idx = torch.randint(0, T, [B]).to(self.device)                  # omnitokenizer.py:401 (one CPU RNG draw)
                ar = torch.arange(B, device=self.device)
                frames, frames_recon = x[ar, :, frame_idx], x_recon[ar, :, frame_idx]
            return frames, frames_recon, x, x_recon, vq_output

    def _forward_decode(self, eng, ws, dims, u8=None):
        """forward()'s quantise -> decode -> statistics on the encoder output in the workspace.  Returns (x_recon 5-D, or
        uint8 'b t h w c' with u8 = the output affine; vq_output or None for the VAE)."""
        B, Tp, h, w = dims
        M = ws.M
        vq_output = None
        if not self.use_vae:
            z = eng.z_view(ws).clone()
            idx, counts = ws.idx.clone(), ws.counts.clone()
            x_recon = eng.decode(dims, idx=idx, straight_through=True, u8=u8)     # decoder sees (e - z) + z
            zq = eng.zq_view(ws).clone()
            cb = self.codebook
            n_codes = cb.n_codes
            usage = self._track_usage(counts, M)                                  # codebook.py:54-72, 133-138
            e = eng.E[idx]
            commitment = 0.25 * torch.mean((z - e) ** 2)                           # codebook.py:93
            perplexity = torch.exp(-torch.sum(usage * torch.log(usage + 1e-10)))   # codebook.py:122-123
            avg_usage = (cb.codebook_usage.data > (1 / n_codes)).sum() / n_codes
            vq_output = dict(embeddings=zq.view(B, Tp, h, w, -1).permute(0, 4, 1, 2, 3).contiguous(),
                             encodings=idx.view(B, Tp, h, w), commitment_loss=commitment, perplexity=perplexity,
                             avg_usage=avg_usage, batch_usage=usage)
        else:
            hpar = eng.z_view(ws)
            c = hpar.shape[1] // 2
            hp5 = hpar.view(B, Tp, h, w, 2 * c).permute(0, 4, 1, 2, 3)
            mean, logvar = hp5[:, :c], torch.clamp(hp5[:, c:], -30.0, 20.0)
            noise = torch.randn(mean.shape).to(device=self.device)               # drawn BEFORE randint (:368 vs :401)
            z = mean + torch.exp(0.5 * logvar) * noise
            zc = z.permute(0, 2, 3, 4, 1).reshape(M, c).contiguous()
            x_recon = eng.decode(dims, zc=zc, u8=u8)
        return x_recon, vq_output

    @torch.no_grad()
    def forward_u8(self, frames, norm=VIDEO_NORM, out_affine=EVAL_U8):
        """forward(x, log_image=True) from uint8 frames, with uint8 out: frames (B, T, H, W, C) or images (B, H, W, C),
        normalised in the patch gather by `norm` (default VIDEO_NORM).  Returns (x_recon, vq_output): x_recon is
        the reconstruction as uint8 'b t h w c' (T = 1 for images) = _to_u8(forward's x_recon, out_affine) byte for byte
        (default: vqgan_eval.py:139,147-148), vq_output is forward's (None for the VAE).  out_affine None: x_recon is
        forward's fp32 reconstruction 'b c t h w' on the device instead (T = 1 for images).  The CPU RNG is consumed as
        forward consumes it (VAE noise, then the random frame's randint), so a seeded eval loop stays in step."""
        if self.resolution_scale is not None:
            raise NotImplementedError("resolution_scale resizes the fp32 frames between the / 255 and the shift "
                                      "(omnitokenizer.py:334-355); no byte table expresses that -- use forward()")
        is_image = frames.ndim == 4
        f = self._u8_frames(frames, is_image)
        eng = self.engine()
        with torch.cuda.device(self.device):
            ws, dims = eng.encode_u8(f, "raw" if self.use_vae else "vq", norm)
            u8 = None if out_affine is None else tuple(float(v) for v in out_affine)
            x_recon, vq_output = self._forward_decode(eng, ws, dims, u8=u8)
            if not is_image:
                torch.randint(0, f.shape[1], [f.shape[0]])                      # forward's random-frame draw (omnitokenizer.py:401)
            return x_recon, vq_output

    @torch.no_grad()
    def forward_images_u8(self, images, resize, norm=IMAGE_NORM, out_affine=EVAL_U8, params=None):
        """forward_u8 of the images the loader's transform `resize` makes of a ragged list of decoded (H_i, W_i, C) uint8
        host images (see encode_images_u8): returns (x_recon uint8 (B, 1, h, w, C), vq_output), equal to forward_u8 on the
        stacked host-transformed images, with the same CPU RNG draws (the transform's parameters first when params is None)."""
        return self._forward_images(images, None, resize, norm, out_affine, params)

    @torch.no_grad()
    def forward_jpeg_u8(self, sources, resize, norm=IMAGE_NORM, out_affine=EVAL_U8, params=None):
        """forward_images_u8 of JPEG files decoded on the device, sources as encode_jpeg_u8 takes them; equal to
        forward_images_u8 of Pillow's decoded images, with the same CPU RNG draws."""
        from . import jpeg
        images, jpegs = jpeg.split_sources(sources)
        return self._forward_images(images, jpegs, resize, norm, out_affine, params)

    def _forward_images(self, images, jpegs, resize, norm, out_affine, params):
        if self.resolution_scale is not None:
            raise NotImplementedError("resolution_scale resizes the fp32 frames between the / 255 and the shift "
                                      "(omnitokenizer.py:334-355); no byte table expresses that -- use forward()")
        images, params = self._images_u8(images, resize, params)
        if not images:
            raise ValueError("forward_images_u8 needs at least one image")
        eng = self.engine()
        with torch.cuda.device(self.device):
            ws, dims = eng.encode_images_u8(images, resize, params, "raw" if self.use_vae else "vq", norm, jpegs)
            return self._forward_decode(eng, ws, dims, u8=tuple(float(v) for v in out_affine))

    # ---------------------------------------------------------------- CLI surface
    @staticmethod
    def add_model_specific_args(parent_parser):
        """Same flag set as omnitokenizer.py:694-768 (stacks after base.VQGAN's and VideoData's parsers)."""
        parser = argparse.ArgumentParser(parents=[parent_parser], add_help=False)
        A = parser.add_argument
        for name, typ, default in (("--lr_min", float, 0.), ("--warmup_steps", int, 0), ("--warmup_lr_init", float, 0.),
                                   ("--grad_accumulates", int, 1), ("--grad_clip_val", float, 1.0),
                                   ("--grad_clip_val_disc", float, 1.0), ("--disloss_check_thres", float, None),
                                   ("--perloss_check_thres", float, None), ("--recloss_check_thres", float, None),
                                   ("--kl_weight", float, 0.), ("--video_perceptual_weight", float, 0.),
                                   ("--activation_in_disc", str, "leaky_relu"), ("--logitslaplace_weight", float, 0.),
                                   ("--dis_warmup_steps", int, 0), ("--dis_lr_multiplier", float, 1.),
                                   ("--patch_size", int, 16), ("--gen_upscale", int, None), ("--enc_block", str, "tttt"),
                                   ("--dec_block", str, "tttt"), ("--twod_window_size", int, 4),
                                   ("--temporal_patch_size", int, 2), ("--spatial_depth", int, 4),
                                   ("--temporal_depth", int, 4), ("--dim_head", int, 64), ("--heads", int, 8),
                                   ("--attn_dropout", float, 0.), ("--ff_dropout", float, 0.), ("--ff_mult", float, 4.),
                                   ("--codebook_type", str, "vq"), ("--codebook_dim", int, None),
                                   ("--commitment_weight", float, 0.25)):
            A(name, type=typ, default=default)
        for name in ("--force_alternation", "--use_vae", "--initialize_vit", "--sigmoid_in_disc", "--apply_blur",
                     "--apply_noise", "--apply_diffaug", "--dis_minlr_multiplier", "--defer_temporal_pool",
                     "--defer_spatial_pool", "--causal_in_temporal_transformer", "--causal_in_peg",
                     "--use_external_codebook", "--fp32_quant", "--l2_code"):
            A(name, action="store_true")
        A("--recon_loss_type", type=str, default="l1", choices=["l1", "l2"])
        A("--patch_embed", type=str, default="linear", choices=["linear", "cnn", "pixelshuffle"])
        A("--spatial_pos", type=str, default="rel", choices=["rel", "rope"])
        A("--resolution_scale", default=None, nargs="+", type=float)
        return parser

    @staticmethod
    def add_base_model_args(parent_parser):
        """The flags the reference takes from base.VQGAN.add_model_specific_args (base.py:245-269) -- vqgan_eval.py:44
        stacks that parser first; provided here so scripts can run without the legacy CNN tokenizer module."""
        parser = argparse.ArgumentParser(parents=[parent_parser], add_help=False)
        A = parser.add_argument
        A("--embedding_dim", type=int, default=256); A("--n_codes", type=int, default=2048)
        A("--n_hiddens", type=int, default=240); A("--lr", type=float, default=3e-4)
        A("--downsample", nargs="+", type=int, default=(4, 4, 4)); A("--disc_channels", type=int, default=64)
        A("--disc_layers", type=int, default=3); A("--discriminator_iter_start", type=int, default=50000)
        A("--disc_loss_type", type=str, default="hinge", choices=["hinge", "vanilla"])
        A("--apply_allframes", action="store_true"); A("--image_gan_weight", type=float, default=1.0)
        A("--video_gan_weight", type=float, default=1.0); A("--l1_weight", type=float, default=4.0)
        A("--gan_feat_weight", type=float, default=0.0); A("--perceptual_weight", type=float, default=0.0)
        A("--i3d_feat", action="store_true"); A("--restart_thres", type=float, default=1.0)
        A("--no_random_restart", action="store_true")
        A("--norm_type", type=str, default="group", choices=["batch", "group"])
        A("--padding_type", type=str, default="replicate", choices=["replicate", "constant", "reflect", "circular"])
        return parser


VQGAN = OmniTokenizer_VQGAN   # the reference's class name inside omnitokenizer.py


CANONICAL_ARGV = ("--patch_embed linear --patch_size 8 --temporal_patch_size 4 --spatial_depth 4 --temporal_depth 4 "
                  "--embedding_dim 512 --disc_layers 3 --enc_block ttww --dec_block tttt --twod_window_size 8 "
                  "--causal_in_temporal_transformer --causal_in_peg --dim_head 64 --heads 8 --apply_noise --apply_blur "
                  "--spatial_pos rope --n_codes 8192 --codebook_dim 8 --l2_code --commitment_weight 1.0 "
                  "--no_random_restart --resolution 256 --sequence_length 17 --norm_type batch").split()


def parse_args(argv):
    """argparse Namespace of a command line as vqgan_eval.py parses it (base.VQGAN's, this module's and VideoData's
    flags), without the canonical flags: store_true flags absent from argv stay False."""
    p = argparse.ArgumentParser()
    p = OmniTokenizer_VQGAN.add_base_model_args(p)
    p = OmniTokenizer_VQGAN.add_model_specific_args(p)
    for f, d in (("--resolution", 256), ("--sequence_length", 17), ("--image_channels", 3),
                 ("--sample_every_n_frames", 1)):
        p.add_argument(f, type=int, default=d)
    return p.parse_args(list(argv))


def canonical_args(extra=()):
    """argparse Namespace of the canonical config used by every shipped eval script
    (scripts/recons/eval_video.sh:1-9)."""
    return parse_args(CANONICAL_ARGV + list(extra))
