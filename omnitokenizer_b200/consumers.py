"""The callers on either side of encode / decode (SURVEY.md section 8f), as thin host functions over the module API:

* vqgan_eval.py's per-batch step (forward(x, log_image=True) -> clamp/255/uint8 frames + usage accounting),
* the autoregressive LM's token wire format (lm_transformer.py:258-268 encode_to_z, :433-434 decode of sampled tokens),
* the latent-diffusion consumers of the VAE variant (DiT / Latte: the 0.18215 latent scale and their layouts).

Each function names the reference lines it stands in for.  They work with any object exposing the reference's
OmniTokenizer_VQGAN API; with this package's module the uint8 conversions run fused in the un-patchify kernel
(omt_unpatchify_u8: the device->host copy shrinks 4x) instead of as torch elementwise passes over the fp32 video.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import torch

from .layout import (ClipResize, U8Norm, U8Resize, clip_params, dit_resize, resize_clip, resize_params, resize_u8,
                     u8_normalize)

LATENT_SCALE = 0.18215            # Diffusion/DiT/train.py:242, Diffusion/Latte/train.py:216

EVAL_U8 = (1.0, 0.5, 0.0, 1.0, 255.0)        # (clamp(x + 0.5, 0, 1) * 255).byte()     vqgan_eval.py:139,147-148; Latte sample_ddp.py:206
DIT_U8 = (255.0, 128.0, 0.0, 255.0, 1.0)     # clamp(255 * x + 128.0, 0, 255).to(uint8)  DiT sample_ddp.py:163

# The data pipelines' uint8 -> fp32 normalisations (input side of encode_u8 / forward_u8): (u / 255 - mean) / std in fp32.
VIDEO_NORM = U8Norm("video_norm", (0.5, 0.5, 0.5), (1.0, 1.0, 1.0), max_test=True)   # VideoNorm, video_utils.py:33-58 (data.py:165,229-232)
IMAGE_NORM = U8Norm("image_norm", (0.5, 0.5, 0.5), (1.0, 1.0, 1.0))   # ToTensor + Normalize((.5,.5,.5), (1,1,1)), data.py:88-97
DIT_NORM = U8Norm("dit_norm", (0.5, 0.5, 0.5), (0.5, 0.5, 0.5))       # ToTensor + Normalize(.5, .5), DiT train.py:185-198
LATTE_NORM = U8Norm("latte_norm", (0.5, 0.5, 0.5), (0.5, 0.5, 0.5))   # ToTensorVideo + Normalize(.5, .5), Latte datasets/*


def _to_u8(video: torch.Tensor, affine) -> torch.Tensor:
    """torch form of the fused conversion: (B,C,T,H,W) fp32 -> (B,T,H,W,C) uint8, the reference's op order."""
    mul, add, lo, hi, post = affine
    t = torch.clamp(video * mul + add, lo, hi) * post
    return t.permute(0, 2, 3, 4, 1).contiguous().to(torch.uint8)


# ----------------------------------------------------------------------------------------------- vqgan_eval.py
@torch.no_grad()
def eval_step(vqgan, x: torch.Tensor, total_usage: Optional[torch.Tensor] = None):
    """One iteration of vqgan_eval.py's loops (:115-155 video, :185-196 image): forward(log_image=True), the
    reconstruction as the uint8 frames the FVD / FID feature extractors take ('b t h w c' = shift_dim(fake * 255, 1, -1)
    .byte(), :147-148), and the running codebook-usage sum (:150-152).  Returns (x_recons fp32, frames uint8, vq_output)."""
    _, _, _, x_recons, vq_output = vqgan(x, log_image=True)
    is_image = x.ndim == 4
    frames = _to_u8(x_recons.unsqueeze(2) if is_image else x_recons, EVAL_U8)
    if total_usage is not None and vq_output is not None:
        total_usage += vq_output["batch_usage"]
    return x_recons, frames, vq_output


@torch.no_grad()
def reconstruct_u8(vqgan, x: torch.Tensor) -> torch.Tensor:
    """encode -> decode with the eval script's uint8 conversion fused into the last kernel: (B,T,H,W,C) uint8 frames
    (T = 1 for images).  Equal to _to_u8(decode(encode(x)), EVAL_U8) byte for byte."""
    is_image = x.ndim == 4
    codes = vqgan.encode(x, is_image)
    if getattr(vqgan, "use_vae", False) and not is_image:
        codes = codes.permute(0, 2, 3, 4, 1)                # 'b c t h w' -> 'b t h w c' (omnitokenizer.py:313)
    if hasattr(vqgan, "decode_u8"):
        return vqgan.decode_u8(codes, is_image, EVAL_U8)
    rec = vqgan.decode(codes, is_image)
    return _to_u8(rec.unsqueeze(2) if is_image else rec, EVAL_U8)


# ----------------------------------------------------------------------------------------------- lm_transformer.py
@torch.no_grad()
def encode_to_z(vqgan, x: torch.Tensor, is_image: bool, sample_every_n_latent_frames: int = 0) -> Tuple[torch.Tensor, torch.Tensor]:
    """Net2NetTransformer.encode_to_z (lm_transformer.py:258-268): the GPT's view of a clip.
    Returns (embeddings channels-last (B, T'', h, w, C), targets int64 (B, T''*h*w)) where T'' keeps every n-th latent frame."""
    emb, targets = vqgan.encode(x, is_image, include_embeddings=True)
    return _z_wire_format(emb, targets, sample_every_n_latent_frames)


def _z_wire_format(emb, targets, sample_every_n_latent_frames):
    if sample_every_n_latent_frames > 0:
        emb = emb[:, :, ::sample_every_n_latent_frames]
        targets = targets[:, ::sample_every_n_latent_frames]
    emb = emb.movedim(1, -1).contiguous()                     # shift_dim(x, 1, -1)
    return emb, targets.reshape(targets.shape[0], -1)


@torch.no_grad()
def decode_tokens(vqgan, ix: torch.Tensor, is_image: bool, cond_stage_vocab_size: int = 0,
                  first_stage_vocab_size: Optional[int] = None) -> torch.Tensor:
    """Sampled GPT tokens back to pixels (lm_transformer.py:433-434, :453-454): the class-conditional vocabulary offset is
    removed and the result clamped into the codebook, then the flat (B, T'hw) indices go through decode()."""
    if first_stage_vocab_size is None:
        first_stage_vocab_size = vqgan.codebook.n_codes
    index = torch.clamp(ix - cond_stage_vocab_size, min=0, max=first_stage_vocab_size - 1)
    if index.ndim == 3 and index.shape[-1] == 1:
        index = index.squeeze(-1)
    return vqgan.decode(index, is_image)


# ----------------------------------------------------------------------------------------------- DiT / Latte (VAE mode)
@torch.no_grad()
def dit_encode_latents(vae, x: torch.Tensor) -> torch.Tensor:
    """Diffusion/DiT/train.py:242: images (B,3,H,W) -> scaled latents (B,8,h,w)."""
    return vae.encode(x, is_image=True).mul_(LATENT_SCALE)


@torch.no_grad()
def dit_decode_latents(vae, samples: torch.Tensor, as_uint8: bool = True) -> torch.Tensor:
    """Diffusion/DiT/sample_ddp.py:162-163: latents (B,8,h,w) -> images; as_uint8: (B,H,W,3) uint8 =
    clamp(255 * x + 128.0, 0, 255), the array the script hands to PIL."""
    z = samples / LATENT_SCALE
    if not as_uint8:
        return vae.decode(z, is_image=True)
    if hasattr(vae, "decode_u8"):
        return vae.decode_u8(z, True, DIT_U8)[:, 0]
    return _to_u8(vae.decode(z, is_image=True).unsqueeze(2), DIT_U8)[:, 0]


@torch.no_grad()
def latte_encode_latents(vae, x_bfchw: torch.Tensor) -> torch.Tensor:
    """Diffusion/Latte/train.py:215-217: clips 'b f c h w' -> scaled latents 'b f c h w' (f = latent frames)."""
    x = x_bfchw.permute(0, 2, 1, 3, 4).contiguous()           # 'b f c h w -> b c f h w'
    z = vae.encode(x, is_image=False).mul_(LATENT_SCALE)
    return z.permute(0, 2, 1, 3, 4).contiguous()              # 'b c f h w -> b f c h w'


@torch.no_grad()
def latte_decode_latents(vae, samples_bfchw: torch.Tensor, as_uint8: bool = True) -> torch.Tensor:
    """Diffusion/Latte/sample/sample_ddp.py:201-206: latents 'b f c h w' -> 'b f h w c' -> decode(z / 0.18215).
    as_uint8: (B, F, H, W, 3) uint8 = (clamp(x + 0.5, 0, 1) * 255).byte(), the frames written to the .mp4;
    otherwise the fp32 video 'b f c h w' (:204)."""
    z = samples_bfchw.permute(0, 1, 3, 4, 2) / LATENT_SCALE   # 'b f c h w -> b f h w c', then the latent scale
    if as_uint8 and hasattr(vae, "decode_u8"):
        return vae.decode_u8(z, False, EVAL_U8)
    video = vae.decode(z, is_image=False)                     # 'b c f h w'
    if not as_uint8:
        return video.permute(0, 2, 1, 3, 4).contiguous()
    return _to_u8(video, EVAL_U8)


# ----------------------------------------------------------------------------------------------- uint8 input side
# The same callers fed the uint8 frames their loaders decode (decord / PIL), before the loader's own normalisation.  With
# this package's module the normalisation runs in the patch-gather kernel (encode_u8 / forward_u8: the host->device copy
# shrinks 4x and the host does no float work); any other object gets the pipeline's fp32 input, computed on the host.
def _check_u8(frames: torch.Tensor, ndims: Tuple[int, ...], what: str):
    if not isinstance(frames, torch.Tensor) or frames.dtype != torch.uint8:
        raise TypeError(f"{what}: expected uint8 frames, got {getattr(frames, 'dtype', type(frames))}")
    if frames.ndim not in ndims:
        raise ValueError(f"{what}: expected channels-last frames of {' or '.join(map(str, ndims))} dimensions, "
                         f"got shape {tuple(frames.shape)}")


def _encode_u8(vqgan, frames: torch.Tensor, is_image: bool, norm: U8Norm, include_embeddings: bool = False):
    _check_u8(frames, (4,) if is_image else (5,), "encode_u8")
    if hasattr(vqgan, "encode_u8"):
        return vqgan.encode_u8(frames, is_image, include_embeddings=include_embeddings, norm=norm)
    x = u8_normalize(frames.unsqueeze(1) if is_image else frames, norm)
    return vqgan.encode(x.squeeze(2) if is_image else x, is_image, include_embeddings=include_embeddings)


@torch.no_grad()
def eval_step_u8(vqgan, frames: torch.Tensor, total_usage: Optional[torch.Tensor] = None, norm: U8Norm = VIDEO_NORM):
    """eval_step from the decoder's uint8 frames (B, T, H, W, C) (or images (B, H, W, C)): vqgan_eval.py's loop over a
    DecordVideoDataset whose VideoNorm (data.py:229-232) is applied in the kernel.  Returns (frames uint8 'b t h w c',
    vq_output), equal to eval_step's frames and vq_output on the normalised input."""
    _check_u8(frames, (4, 5), "eval_step_u8")
    is_image = frames.ndim == 4
    if hasattr(vqgan, "forward_u8"):
        out, vq_output = vqgan.forward_u8(frames, norm, EVAL_U8)
    else:
        x = u8_normalize(frames.unsqueeze(1) if is_image else frames, norm)
        _, _, _, x_recons, vq_output = vqgan(x.squeeze(2) if is_image else x, log_image=True)
        out = _to_u8(x_recons.unsqueeze(2) if is_image else x_recons, EVAL_U8)
    if total_usage is not None and vq_output is not None:
        total_usage += vq_output["batch_usage"]
    return out, vq_output


@torch.no_grad()
def eval_step_fvd(vqgan, frames: torch.Tensor, i3d, total_usage: Optional[torch.Tensor] = None,
                  norm: U8Norm = VIDEO_NORM):
    """The body of vqgan_eval.py's video loop (:114-152) from the loader's uint8 clips (B, T, H, W, 3) on the device:
    forward_u8 (eval_step_u8) for the reconstruction's bytes, and the FVD logits of both sides on the device
    (fvd.I3D).  The real side sees the bytes the script makes of the normalised clip, shift_dim((video + 0.5) * 255,
    1, -1).byte(), as a per-byte map with norm's branch picked per clip.  Returns (real_logits, fake_logits,
    vq_output); no frame crosses to the host."""
    from .fvd import real_byte_table
    _check_u8(frames, (5,), "eval_step_fvd")
    i3d.check_frames(frames)                 # every refusal before the first launch
    real_byte_table(norm)
    fake, vq_output = eval_step_u8(vqgan, frames, total_usage, norm)
    real_logits = i3d.logits(frames, real_norm=norm).clone()
    fake_logits = i3d.logits(fake).clone()
    return real_logits, fake_logits, vq_output


@torch.no_grad()
def encode_to_z_u8(vqgan, frames: torch.Tensor, is_image: bool, sample_every_n_latent_frames: int = 0,
                   norm: U8Norm = VIDEO_NORM) -> Tuple[torch.Tensor, torch.Tensor]:
    """encode_to_z (lm_transformer.py:258-268) from the uint8 frames of the LM's VideoNorm data loader."""
    emb, targets = _encode_u8(vqgan, frames, is_image, norm, include_embeddings=True)
    return _z_wire_format(emb, targets, sample_every_n_latent_frames)


@torch.no_grad()
def dit_encode_latents_u8(vae, images: torch.Tensor, norm: U8Norm = DIT_NORM) -> torch.Tensor:
    """dit_encode_latents from (B, H, W, 3) uint8 images (DiT train.py:185-198 ToTensor + Normalize, then :242)."""
    return _encode_u8(vae, images, True, norm).mul_(LATENT_SCALE)


@torch.no_grad()
def latte_encode_latents_u8(vae, clips: torch.Tensor, norm: U8Norm = LATTE_NORM) -> torch.Tensor:
    """latte_encode_latents from (B, F, H, W, 3) uint8 clips (Latte ToTensorVideo + Normalize, then train.py:215-217):
    scaled latents 'b f c h w'."""
    z = _encode_u8(vae, clips, False, norm).mul_(LATENT_SCALE)
    return z.permute(0, 2, 1, 3, 4).contiguous()              # 'b c f h w -> b f c h w'


# ----------------------------------------------------------------------------------------------- decoded images, any size
# The image callers' loaders resize every decoded image with Pillow before ToTensor (U8Resize presets in layout.py).  With
# this package's module that transform runs on the device (encode_images_u8 / forward_images_u8: omt_resample_u8, byte for
# byte Pillow's); any other object gets the same bytes from the host twin layout.resize_u8, then the uint8 path above.
def _host_transform(images: Sequence[torch.Tensor], resize: U8Resize) -> torch.Tensor:
    images = list(images)
    params = resize_params(len(images), resize)
    return torch.stack([resize_u8(im, resize, p) for im, p in zip(images, params)])


@torch.no_grad()
def eval_step_images_u8(vqgan, images: Sequence[torch.Tensor], resize: U8Resize, total_usage: Optional[torch.Tensor] = None,
                        norm: U8Norm = IMAGE_NORM):
    """eval_step_u8 over the decoded images of vqgan_eval.py's image loop (ImageDataset, OmniTokenizer/data.py:93-99:
    resize = layout.image_resize(resolution)), ragged (H_i, W_i, 3) uint8 host tensors.  Returns (frames uint8
    (B, 1, h, w, 3), vq_output)."""
    if hasattr(vqgan, "forward_images_u8"):
        out, vq_output = vqgan.forward_images_u8(images, resize, norm, EVAL_U8)
        if total_usage is not None and vq_output is not None:
            total_usage += vq_output["batch_usage"]
        return out, vq_output
    return eval_step_u8(vqgan, _host_transform(images, resize), total_usage, norm)


@torch.no_grad()
def eval_step_fid(vqgan, images: Sequence[torch.Tensor], resize: U8Resize, inception,
                  total_usage: Optional[torch.Tensor] = None, norm: U8Norm = IMAGE_NORM):
    """The body of vqgan_eval.py's image loop (:185-220) from the decoded ragged host images of ImageDataset, with the
    PNG round trip and the pytorch-fid run replaced by FID features on the device (fid.FIDInception): forward_images_u8
    for the reconstruction's bytes and vq_output, and the pool3 features of both sides.  The real side reads the
    transformed input bytes that call wrote into the encode_u8 slot (the random crop and flip are drawn once) and sees
    the bytes the script saves of the normalised input, ((x + 0.5) * 255).astype(uint8), as a per-byte map.  Returns
    (real_features, fake_features, vq_output), each features (B, 2048) fp32; no image crosses to the host.
    --infer_downsample (a PIL ANTIALIAS resize before saving) is not supported."""
    from .fvd import real_byte_table
    images = list(images)
    if not images:
        raise ValueError("eval_step_fid needs at least one image")
    real_byte_table(norm)                    # refuses a per-channel normalisation before the first launch
    if hasattr(vqgan, "forward_images_u8"):
        fake, vq_output = vqgan.forward_images_u8(images, resize, norm, EVAL_U8)
        if total_usage is not None and vq_output is not None:
            total_usage += vq_output["batch_usage"]
        real = vqgan.engine().encode_u8_frames(tuple(fake.shape))
    else:
        real = _host_transform(images, resize).to(inception.device)
        fake, vq_output = eval_step_u8(vqgan, real, total_usage, norm)
        real = real.unsqueeze(1)
    real_features = inception.features(real[:, 0], real_norm=norm).clone()
    fake_features = inception.features(fake[:, 0].contiguous()).clone()
    return real_features, fake_features, vq_output


@torch.no_grad()
def encode_to_z_images_u8(vqgan, images: Sequence[torch.Tensor], resize: U8Resize,
                          norm: U8Norm = IMAGE_NORM) -> Tuple[torch.Tensor, torch.Tensor]:
    """encode_to_z (lm_transformer.py:258-268) of the LM's image stage from its decoded images (ImageDataset transform)."""
    if hasattr(vqgan, "encode_images_u8"):
        emb, targets = vqgan.encode_images_u8(images, resize, norm, include_embeddings=True)
    else:
        emb, targets = _encode_u8(vqgan, _host_transform(images, resize), True, norm, include_embeddings=True)
    return _z_wire_format(emb, targets, 0)


@torch.no_grad()
def dit_encode_latents_images_u8(vae, images: Sequence[torch.Tensor], image_size: int, norm: U8Norm = IMAGE_NORM) -> torch.Tensor:
    """dit_encode_latents from DiT's decoded images with the OmniTokenizer VAE (Diffusion/DiT/train.py:192-198:
    Resize((s, s)) bilinear, RandomHorizontalFlip, ToTensor, Normalize(.5, 1) = IMAGE_NORM; then :242)."""
    resize = dit_resize(image_size)
    if hasattr(vae, "encode_images_u8"):
        return vae.encode_images_u8(images, resize, norm).mul_(LATENT_SCALE)
    return _encode_u8(vae, _host_transform(images, resize), True, norm).mul_(LATENT_SCALE)


# ----------------------------------------------------------------------------------------------- decoded clips, any size
# Latte's video loaders turn read_video's frames into fp32 before they resize (ClipResize presets in layout.py), so no
# uint8 clip of the model's size ever exists.  With this package's module the whole transform runs on the device
# (encode_clips_u8: omt_resample_clips, bit for bit torch's CPU arithmetic); any other object gets the fp32 clips from the
# host twin layout.resize_clip.
@torch.no_grad()
def latte_encode_latents_clips_u8(vae, clips: Sequence[torch.Tensor], resize: ClipResize,
                                  norm: U8Norm = LATTE_NORM) -> torch.Tensor:
    """latte_encode_latents of the clips Latte's loader makes of decoded (F, H_i, W_i, 3) uint8 frames (e.g.
    layout.ucf_clip_resize(256) for ucf101 / ffs: ToTensorVideo, RandomHorizontalFlipVideo, UCFCenterCropVideo,
    Normalize(.5, .5)): scaled latents 'b f c h w'."""
    if hasattr(vae, "encode_clips_u8"):
        z = vae.encode_clips_u8(clips, resize, norm).mul_(LATENT_SCALE)
        return z.permute(0, 2, 1, 3, 4).contiguous()          # 'b c f h w -> b f c h w'
    clips = list(clips)
    flips = clip_params(len(clips), resize)
    return latte_encode_latents(vae, torch.stack([resize_clip(c, resize, f, norm) for c, f in zip(clips, flips)]))
