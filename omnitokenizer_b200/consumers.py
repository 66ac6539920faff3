"""The callers on either side of encode / decode (SURVEY.md section 8f), as thin host functions over the module API:

* vqgan_eval.py's per-batch step (forward(x, log_image=True) -> clamp/255/uint8 frames + usage accounting),
* the autoregressive LM's token wire format (lm_transformer.py:258-268 encode_to_z, :433-434 decode of sampled tokens),
* the latent-diffusion consumers of the VAE variant (DiT / Latte: the 0.18215 latent scale and their layouts).

Each function names the reference lines it stands in for.  They work with any object exposing the reference's
OmniTokenizer_VQGAN API; with this package's module the uint8 conversions run fused in the un-patchify kernel
(omt_unpatchify_u8: the device->host copy shrinks 4x) instead of as torch elementwise passes over the fp32 video.
"""
from __future__ import annotations

import os
from typing import Optional, Sequence, Tuple

import torch

from . import layout as L
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


def check_replacewithgt(k, T: int, sequence_length: Optional[int], what: str) -> int:
    """vqgan_eval.py's --replacewithgt k (type=int): 0 <= k <= T, and the clip as long as --sequence_length (:145)."""
    if isinstance(k, bool) or not isinstance(k, int):
        raise TypeError(f"{what}: replacewithgt must be an integer frame count, got {k!r}")
    if not 0 <= k <= T:
        raise ValueError(f"{what}: replacewithgt {k} outside [0, {T}] for {T}-frame clips")
    if sequence_length is not None and T != sequence_length:
        raise ValueError(f"{what}: replacewithgt needs clips of sequence_length {sequence_length} frames, got T={T}")
    return k


@torch.no_grad()
def eval_step_fvd(vqgan, frames: torch.Tensor, i3d, total_usage: Optional[torch.Tensor] = None,
                  norm: U8Norm = VIDEO_NORM, infer_downsample: Optional[int] = None, replacewithgt: Optional[int] = None,
                  sequence_length: Optional[int] = None, one_thread: Optional[bool] = None):
    """The body of vqgan_eval.py's video loop (:114-152) from the loader's uint8 clips (B, T, H, W, 3) on the device:
    forward_u8 (eval_step_u8) for the reconstruction's bytes, and the FVD logits of both sides on the device
    (fvd.I3D).  The real side sees the bytes the script makes of the normalised clip, shift_dim((video + 0.5) * 255,
    1, -1).byte(), as a per-byte map with norm's branch picked per clip.  Returns (real_logits, fake_logits,
    vq_output); no frame crosses to the host.
    infer_downsample d (:121-136): both sides are scored at 1 / d of their size: forward_u8's fp32 reconstruction and
    the real values go through F.interpolate(scale_factor=1 / d) in torch's CPU arithmetic, then * 255 and .byte()
    (downsample.clips_u8; one_thread as there).  replacewithgt k (:142-145): the first k reconstructed frames are the
    real ones; sequence_length, when given, is the script's --sequence_length, which the clips must match."""
    from .metricnet import real_byte_table
    _check_u8(frames, (5,), "eval_step_fvd")
    i3d.check_frames(frames)                 # every refusal before the first launch
    real_byte_table(norm)
    if infer_downsample is None and replacewithgt is None:
        fake, vq_output = eval_step_u8(vqgan, frames, total_usage, norm)
        real_logits = i3d.logits(frames, real_norm=norm).clone()
        fake_logits = i3d.logits(fake).clone()
        return real_logits, fake_logits, vq_output

    from . import downsample
    d = 1 if infer_downsample is None else L.check_infer_downsample(infer_downsample, "eval_step_fvd")
    B, T, H, W, _ = (int(v) for v in frames.shape)
    k = 0 if replacewithgt is None else check_replacewithgt(replacewithgt, T, sequence_length, "eval_step_fvd")
    downsample.out_size(H, W, d, "eval_step_fvd")
    downsample.real_value_table(norm)
    if frames.device.type != "cuda" or frames.device != i3d.device:
        raise ValueError(f"eval_step_fvd: frames on {frames.device}, the I3D is on {i3d.device}")
    frames = frames.contiguous()
    if hasattr(vqgan, "forward_u8"):
        x_recons, vq_output = vqgan.forward_u8(frames, norm, None)
    else:
        _, _, _, x_recons, vq_output = vqgan(u8_normalize(frames, norm), log_image=True)
    if total_usage is not None and vq_output is not None:
        total_usage += vq_output["batch_usage"]
    # with d = 1 (replacewithgt alone) the interpolation is the identity and the launches only map the values to bytes
    real = downsample.clips_u8(frames, d, real_norm=norm, one_thread=one_thread, what="eval_step_fvd")
    fake = downsample.clips_u8(x_recons.float().contiguous(), d, one_thread=one_thread, what="eval_step_fvd")
    if k:
        fake[:, :k].copy_(real[:, :k])
    real_logits = i3d.logits(real).clone()
    fake_logits = i3d.logits(fake).clone()
    return real_logits, fake_logits, vq_output


@torch.no_grad()
def eval_step_quality(vqgan, frames: torch.Tensor, lpips=None, total_usage: Optional[torch.Tensor] = None,
                      norm: U8Norm = VIDEO_NORM):
    """vqgan_eval.py's loop body (:114-152) with the per-frame reconstruction metrics of
    evaluation/common_metrics_on_video_quality on the device: forward_u8 (eval_step_u8) for the reconstruction's bytes,
    then quality.frame_metrics of the real and reconstructed bytes (PSNR, SSIM and, with a quality.LPIPS model, the VGG
    LPIPS).  The real side sees the bytes the script makes of the normalised clip, ((video + 0.5) * 255).byte(), as a
    per-byte map with norm's branch picked per clip.  frames: the loader's uint8 (B, T, H, W, 3) on the device, or
    images (B, H, W, 3) as T = 1.  Returns (psnr (B, T) fp64, ssim (B, T) fp64, lpips (B, T) fp32 or None,
    fake_u8 (B, T, H, W, 3), vq_output); fake_u8 can feed i3d.logits as well.  No frame crosses to the host."""
    from . import quality
    from .metricnet import real_byte_table
    _check_u8(frames, (4, 5), "eval_step_quality")
    real = frames.unsqueeze(1) if frames.dim() == 4 else frames
    quality.check_pair(real, real, torch.uint8, "eval_step_quality")      # every refusal before the first launch
    quality._check_sizes(int(real.shape[2]), int(real.shape[3]), int(real.shape[4]), "eval_step_quality",
                         lpips is not None)
    real_byte_table(norm)
    fake, vq_output = eval_step_u8(vqgan, frames, total_usage, norm)
    if fake.dim() == 4:
        fake = fake.unsqueeze(1)
    psnr, ssim, lp = quality.frame_metrics(real, fake, lpips, real_norm=norm)
    return psnr, ssim, lp, fake, vq_output


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


SAVED_FORMATS = ("png", "jpeg")
_JPEG_EXTENSIONS = (".jpg", ".jpeg", ".jpe", ".jfif")


def saved_format(path) -> str:
    """The format vqgan_eval.py's Image.fromarray(...).save(path) writes (:205-220): Pillow picks it from the lower-cased
    extension of the dataset's own relative path, batch["path"].  .jpg, .jpeg, .jpe and .jfif -> "jpeg" (ImageNet's
    .JPEG, CelebA-HQ's .jpg), .png -> "png" (FFHQ); any other extension raises NotImplementedError naming it."""
    ext = os.path.splitext(os.fspath(path))[1].lower()
    if ext in _JPEG_EXTENSIONS:
        return "jpeg"
    if ext == ".png":
        return "png"
    raise NotImplementedError(f"saved_format: vqgan_eval.py would save {os.fspath(path)!r} by its extension {ext!r}; "
                              f"only PNG and JPEG are reproduced")


@torch.no_grad()
def eval_step_fid(vqgan, images: Sequence[torch.Tensor], resize: U8Resize, inception,
                  total_usage: Optional[torch.Tensor] = None, norm: U8Norm = IMAGE_NORM,
                  infer_downsample: Optional[int] = None, saved_as: str = "png"):
    """The body of vqgan_eval.py's image loop (:185-220) from the decoded ragged host images of ImageDataset, with the
    file round trip and the pytorch-fid run replaced by FID features on the device (fid.FIDInception): forward_images_u8
    for the reconstruction's bytes and vq_output, and the pool3 features of both sides.  The real side reads the
    transformed input bytes that call wrote into the encode_u8 slot (the random crop and flip are drawn once) and sees
    the bytes the script saves of the normalised input, ((x + 0.5) * 255).astype(uint8), as a per-byte map.  Returns
    (real_features, fake_features, vq_output), each features (B, 2048) fp32; no image crosses to the host.
    infer_downsample d (:207-208, :218-219): both sides' saved bytes are first resized to (h // d, h // d) with
    Image.ANTIALIAS (Pillow's LANCZOS, downsample.images_u8); the real side's byte map then comes before the resize.
    saved_as: the format the script's img.save(path) writes, saved_format(batch["path"][0]).  "png" is lossless, so
    the network sees the saved bytes themselves; with "jpeg" both sides' saved bytes (after the resize, if any) go
    through Pillow's JPEG save at its default quality 75 and reload (jpeg.roundtrip_u8), as pytorch-fid reads them.
    images may also hold JPEG files (bytes-like or paths, as ImageDataset reads them), decoded on the device byte for
    byte as Image.open(path).convert('RGB') (vqgan.forward_jpeg_u8); the results equal those of Pillow's decoded
    images, bit for bit."""
    from .metricnet import real_byte_table
    if saved_as not in SAVED_FORMATS:
        raise ValueError(f"eval_step_fid: saved_as {saved_as!r} is not one of {SAVED_FORMATS}")
    images = list(images)
    if not images:
        raise ValueError("eval_step_fid needs at least one image")
    real_byte_table(norm)                    # refuses a per-channel normalisation before the first launch
    if infer_downsample is not None or saved_as != "png":
        return _eval_step_fid_saved(vqgan, images, resize, inception, total_usage, norm, infer_downsample, saved_as)
    if hasattr(vqgan, "forward_images_u8"):
        fake, vq_output = _forward_sources(vqgan, images, resize, norm)
        if total_usage is not None and vq_output is not None:
            total_usage += vq_output["batch_usage"]
        real = vqgan.engine().encode_u8_frames(tuple(fake.shape))
    else:
        real = _host_transform(_decoded(images, inception.device), resize).to(inception.device)
        fake, vq_output = eval_step_u8(vqgan, real, total_usage, norm)
        real = real.unsqueeze(1)
    real_features = inception.features(real[:, 0], real_norm=norm).clone()
    fake_features = inception.features(fake[:, 0].contiguous()).clone()
    return real_features, fake_features, vq_output


def _forward_sources(vqgan, images, resize: U8Resize, norm: U8Norm):
    """forward_images_u8, or forward_jpeg_u8 when the list holds JPEG files (anything but a tensor)."""
    if all(isinstance(im, torch.Tensor) for im in images):
        return vqgan.forward_images_u8(images, resize, norm, EVAL_U8)
    return vqgan.forward_jpeg_u8(images, resize, norm, EVAL_U8)


def _decoded(images, device):
    """The list with its JPEG files decoded (jpeg.decode_u8 on device, brought to the host as the model's host path
    takes them)."""
    from . import jpeg
    at = [i for i, im in enumerate(images) if not isinstance(im, torch.Tensor)]
    if not at:
        return images
    out = list(images)
    for i, t in zip(at, jpeg.decode_u8([images[i] for i in at], device)):
        out[i] = t.cpu()
    return out


def _eval_step_fid_saved(vqgan, images, resize: U8Resize, inception, total_usage, norm: U8Norm, d, saved_as: str):
    """eval_step_fid on the bytes the script saves, materialised on the device: resized when d is given, then round
    tripped through JPEG when saved_as is "jpeg"."""
    from . import downsample, jpeg
    if d is not None:
        d = L.check_infer_downsample(d, "eval_step_fid")
        h, w = resize.out_size
        if h != w:
            raise ValueError(f"eval_step_fid: infer_downsample resizes square images, the transform makes {h}x{w}")
        L.eval_downsample_resize(h, d)                   # refuses a factor that leaves no pixel
    downsample.real_value_table(norm)
    if inception.device.type != "cuda":
        raise ValueError(f"eval_step_fid: the FID network is on {inception.device}, not a CUDA device")
    if hasattr(vqgan, "forward_images_u8"):
        fake, vq_output = _forward_sources(vqgan, images, resize, norm)
        if total_usage is not None and vq_output is not None:
            total_usage += vq_output["batch_usage"]
        real = vqgan.engine().encode_u8_frames(tuple(fake.shape))
    else:
        real = _host_transform(_decoded(images, inception.device), resize).to(inception.device)
        fake, vq_output = eval_step_u8(vqgan, real, total_usage, norm)
        real = real.unsqueeze(1)
    # the saved input bytes ((x + 0.5) * 255).astype(uint8): the value map at d = 1 (an identity interpolation)
    real = downsample.clips_u8(real.contiguous(), 1, real_norm=norm, what="eval_step_fid")[:, 0]
    fake = fake[:, 0].contiguous()
    if d is not None:
        real = downsample.images_u8(real, d, "eval_step_fid")
        fake = downsample.images_u8(fake, d, "eval_step_fid")
    if saved_as == "jpeg":
        real = jpeg.roundtrip_u8(real, jpeg.DEFAULT_QUALITY)
        fake = jpeg.roundtrip_u8(fake, jpeg.DEFAULT_QUALITY)
    real_features = inception.features(real).clone()
    fake_features = inception.features(fake).clone()
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


FVD_SAMPLING = ("first", "last", "center")


def fvd_external_indices(n: int, frames: int, sampling: str = "center"):
    """The frames fvd_external.py's load_videos keeps of an n-frame clip (:30-46): all when n == frames, else the first
    or last `frames`, or range(c - frames // 2, c + frames // 2), one more for odd `frames`, with c = n // 2.  Raises
    its assertion n >= frames as a ValueError."""
    if sampling not in FVD_SAMPLING:
        raise ValueError(f"fvd_external: unknown sampling {sampling!r}; expected one of {FVD_SAMPLING}")
    if frames < 1 or n < frames:
        raise ValueError(f"fvd_external: a clip of {n} frames, fewer than frames={frames}")
    if n == frames or sampling == "first":
        return range(frames)
    if sampling == "last":
        return range(n - frames, n)
    c = n // 2
    return range(c - frames // 2, c + frames // 2 + frames % 2)


def fvd_external(gt_clips_u8: Sequence[torch.Tensor], gen_clips_u8: Sequence[torch.Tensor], i3d, frames: int = 17,
                 sampling: str = "center") -> dict:
    """evaluation/fvd_external.py from decoded clips: each a uint8 (T_i, H, W, 3) tensor of any length T_i >= frames
    at the target resolution (decoding the videos with decord / ffmpeg and scaling them to --resolution is the
    caller's job).  Applies load_videos's frame selection and assertion to every clip, stacks each side on the device,
    and returns calculate_fvd(gt, gen, method="videogpt") from the bytes (i3d: fvd.load_fvd_model's network)."""
    from .quality import calculate_fvd
    sides = []
    for name, clips in (("gt", gt_clips_u8), ("gen", gen_clips_u8)):
        clips = list(clips)
        if not clips:
            raise ValueError(f"fvd_external: no {name} clips")
        for c in clips:
            _check_u8(c, (4,), f"fvd_external ({name})")
        idx = [fvd_external_indices(int(c.shape[0]), frames, sampling) for c in clips]
        sides.append(torch.stack([c[r.start:r.stop].to(i3d.device) for c, r in zip(clips, idx)]))
    return calculate_fvd(sides[0], sides[1], i3d.device, method="videogpt", i3d=i3d)
