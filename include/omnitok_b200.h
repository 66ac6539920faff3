/*
 * omnitok_b200 -- C ABI of the H100 (sm_90a) kernels behind OmniTokenizer_VQGAN.encode/decode.
 *
 * The reference (FoundationVision/OmniTokenizer) has no FFI of its own: its boundary is the
 * Python module API of OmniTokenizer_VQGAN (OmniTokenizer/omnitokenizer.py:63-413).  Each entry
 * point below replaces one group of torch library calls on that path; the reference call site
 * it stands in for is cited next to it (paths relative to /root/reference/OmniTokenizer/).
 *
 * Conventions
 *   - all pointers are DEVICE pointers owned by the caller (fp32 unless noted); nothing is
 *     allocated or retained; outputs may not alias inputs unless stated.
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*).
 *   - return 0 on success, negative on error (OMT_E_*); omt_last_error() gives the message
 *     (thread-local).  There is NO CPU fallback: a non-sm_90 device returns OMT_E_ARCH.
 *   - activations live in ONE canonical layout  X[B][T'][N][C]  (C fastest; identical to the
 *     reference's "(b t) (h w) d" tensor).  "rows" are (b,t',n) triples, M = B*T'*N.
 *   - a "row map" (seg, seg_stride, seg_off) maps logical GEMM row r to physical row
 *     (r / seg) * seg_stride + seg_off + (r % seg); seg <= 0 means identity.  It is how the
 *     first-frame / rest-frames patch matrices address the canonical buffer without a concat.
 */
#ifndef OMNITOK_B200_H_
#define OMNITOK_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OMT_ABI_VERSION 2

#define OMT_OK 0
#define OMT_E_ARG (-1)    /* bad shape / alignment / null pointer */
#define OMT_E_ARCH (-2)   /* device is not sm_90 */
#define OMT_E_CUDA (-3)   /* a CUDA runtime call failed */
#define OMT_E_UNSUPPORTED (-4)

typedef void* omt_stream_t;

int omt_abi_version(void);
const char* omt_last_error(void);
/* sm count / compute capability of the current device */
int omt_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* GEMM epilogue selectors */
#define OMT_EPI_NONE 0
#define OMT_EPI_GEGLU 1   /* packed columns (2j, 2j+1) = (value, gate): C[:, j] = gelu_erf(gate) * value */
#define OMT_EPI_QKV 2     /* dual-A forms: rope + l2norm + scale on the q / k heads (attention.py:417-437) */
#define OMT_EPI_QKV_PLANES 3   /* omt_linear_h: the same, but q / k / v leave as fp16 operand planes for omt_attn_spatial_h */

/* GEMM math selectors */
#define OMT_MATH_FP32 0      /* CUDA-core FFMA, exact fp32 (parity anchor) */
#define OMT_MATH_3XTF32 1    /* wgmma tf32, error-compensated hi/lo split, fp32 accumulate in registers */
#define OMT_MATH_F16X1 2     /* throughput mode: ONE wgmma f16 per product on the hi planes (omt_linear_h1, omt_attn_spatial_h1);
                                NOT reference-exact (about 11 significant bits per operand, like single-pass TF32) */
#define OMT_MATH_F16X3 3     /* wgmma f16 on pre-split fp16 hi / lo operand planes (omt_linear_h) */

/* C[M, N] = A[M, K] . W[N, K]^T (+ bias[N]) (+ residual[M, N]); nn.Linear everywhere on the path:
 * attention.py:411 (to_q / to_kv), :486 (to_out), :271/:288 (window qkv / proj), :164/:167 (FF),
 * omnitokenizer.py:809,819 (patch embed), :1007,1013 (to_pixels).
 * W must be allocated with rows padded up to a multiple of 128 (zero rows); K % 8 == 0 (fp32 path)
 * or K % 32 == 0 (tensor-core paths).  With OMT_EPI_GEGLU, N counts packed columns and C has N/2 columns.
 * residual may alias C (same ld): out-of-place is not required.  For OMT_MATH_3XTF32 `W` must be the
 * tf32-rounded (round-to-nearest, low 13 mantissa bits zero) high part of the weight and `W_lo` the
 * exact remainder (same shape); W_lo is ignored (may be NULL) for FP32. */
int omt_linear(const float* A, int lda, int a_seg, int a_seg_stride, int a_seg_off,
               const float* W, const float* W_lo,
               float* C, int ldc, int c_seg, int c_seg_stride, int c_seg_off,
               int M, int N, int K,
               const float* bias, const float* residual, int ldr,
               int epilogue, int math, omt_stream_t stream);

/* Dual-A form: C[:, :n_split] = A1 . W[:n_split]^T and C[:, n_split:] = A2 . W[n_split:]^T in ONE launch.
 * Attention.forward projects q from the LayerNormed input and k, v from the RAW input
 * (attention.py:407-412); stacking [Wq; Wkv] and switching the A tensor map per output tile fuses the two
 * nn.Linear calls without changing either result.  n_split % 128 == 0 (a whole output tile); same lda for A1 and A2. */
int omt_linear2(const float* A1, const float* A2, int n_split, int lda, const float* W, const float* W_lo,
                float* C, int ldc, int M, int N, int K, int math,
                /* optional fused q/k preparation (what omt_qk_prep does), q_scale == NULL disables it:
                 * columns [0, qk_cols) are heads of 64; the first half carry q (q_scale), the second k (k_scale);
                 * rope tables [tokens, 32] or NULL; the rope position of row m is m % tokens */
                const float* q_scale, const float* k_scale, const float* rope_cos, const float* rope_sin,
                int qk_cols, int tokens, omt_stream_t stream);

/* y[r,:] = (x[r,:] - mean) * rstd * w + b over C channels (C % 4 == 0, C <= 1024); b may be NULL.
 * attention.py:73-80 (LayerNorm, beta buffer), :163 (nn.LayerNorm in FeedForward), :688 (norm_out).
 * x may alias y.  (seg, seg_stride, seg_off) is a row map applied to BOTH x and y (patch embed:
 * the first-frame and rest-frames rows of X carry different LayerNorm weights, omnitokenizer.py:811,821). */
int omt_layernorm(const float* x, int ldx, float* y, int ldy, const float* w, const float* b,
                  int M, int C, float eps, int seg, int seg_stride, int seg_off, omt_stream_t stream);

/* Patch gather + LayerNorm (omnitokenizer.py:806-808 / :814-817: Rearrange + nn.LayerNorm).
 * video (B, Cin, T, H, W) fp32 contiguous, Cin >= 1.  first=1: frame 0, rows (b,h,w), features (c,p1,p2);
 * first=0: frames 1.., rows (b,t,h,w), features (c,pt,p1,p2), with pt > 0 dividing T - 1.  p > 0 is a multiple of 4
 * dividing H and W; K = Cin * (1 | pt) * p * p <= 1024.  A is [rows, K] dense.
 * ln_w == ln_b == NULL: plain patch gather (im2col of the strided Conv3d of patch_embed='cnn', omnitokenizer.py:823-838).
 * A_hi != NULL: the rows are written as fp16 hi / lo operand planes [rows, K] instead of A (A may be NULL);
 * A_rs != NULL: in the row-scaled form, inverse row scales to A_rs [rows]. */
int omt_patchify_ln(const float* video, float* A, uint16_t* A_hi, uint16_t* A_lo, float* A_rs, const float* ln_w, const float* ln_b,
                    int B, int Cin, int T, int H, int W, int p, int pt, int first, float eps,
                    omt_stream_t stream);

/* omt_patchify_ln on uint8 frames: the data pipelines' byte -> fp32 normalisation fused into the gather.
 * frames (B, T, H, W, Cin) uint8 contiguous, channels last (decord / PIL / decode_u8 layout), 4-byte aligned; 1 <= Cin <= 4.
 * Patch geometry (p > 0, pt > 0 for the rest frames, K <= 1024) as omt_patchify_ln.
 * lut: fp32 [n_tab][Cin][256], the value byte u of channel c stands for, built on the host with the pipeline's own CPU
 * expression (e.g. (u / 255 - mean_c) / std_c), so the kernel never divides and its values are the pipeline's bits.
 * sel: NULL (n_tab = 1, every sample uses table 0) or int32 [B] table index per sample, 0 or 1 (n_tab = 2; see
 * omt_u8_norm_select).  Outputs, forms and the ln_w == NULL im2col form as omt_patchify_ln; the result equals
 * omt_patchify_ln on the fp32 video the table maps the frames to, bit for bit. */
int omt_patchify_ln_u8(const uint8_t* frames, const float* lut, const int32_t* sel, float* A, uint16_t* A_hi, uint16_t* A_lo,
                       float* A_rs, const float* ln_w, const float* ln_b, int B, int Cin, int T, int H, int W, int p, int pt,
                       int first, float eps, omt_stream_t stream);

/* VideoNorm's test (OmniTokenizer/video_utils.py:33-58: `if max(clip) > 1: div_(255)`) on the device, per sample:
 * sel[b] = (max byte of the per_sample bytes of sample b > 1) ? 0 : 1.  Writes every sel[b] (no prior reset needed,
 * no host sync): two launches, safe inside a captured CUDA graph. */
int omt_u8_norm_select(const uint8_t* frames, int B, long long per_sample, int32_t* sel, omt_stream_t stream);

/* One image of omt_resample_u8.  Offsets into tab count int32 entries. */
typedef struct {
  long long src;          /* byte offset of the image's (H, W, 3) bytes in src */
  int H, W;               /* source size */
  int rh, rw;             /* size after the resize */
  int y0, x0;             /* crop origin in the resized image (0, 0 without a crop) */
  int flip;               /* 1: the output is mirrored left-right */
  int need_h, need_v;     /* 0: that axis keeps its size and Pillow skips the pass (rw == W / rh == H) */
  int hb, hc, hk;         /* horizontal: (xmin, n) bounds [rw][2] at tab + hb, coefficients [rw][hk] at tab + hc */
  int vb, vc, vk;         /* vertical: the same over rh */
  int v_first;            /* 1: vertical pass first (Pillow's Image.resize for H > 100 W shrinking in height); needs both passes */
} omt_resample_desc;

/* Pillow's 8-bit resize (libImaging/Resample.c, horizontal then vertical int32 pass, 22-bit fixed point, clip8 after
 * each pass) of a ragged batch of (H_i, W_i, 3) uint8 images, then the loaders' RandomCrop / RandomHorizontalFlip as
 * index maps: out (B, oh, ow, 3) uint8, image b = crop(resize(image b))[y0 : y0 + oh, x0 : x0 + ow], mirrored if flip.
 * The bounds and coefficients come from the host (Resample.c precompute_coeffs + normalize_coeffs_8bpc in float64), so
 * the bytes equal Pillow's.  src: packed source bytes (src_bytes of them); desc [B]: device table; tab [tab_len] int32.
 * desc_host / tab_host: the same two tables in host memory, checked before the launch (every image inside src, every
 * table inside tab, every tap inside its source axis, the crop inside the resized image); they must equal the device
 * copies.  tab == tab_host == NULL with tab_len == 0 when no image needs a pass. */
int omt_resample_u8(const uint8_t* src, long long src_bytes, const omt_resample_desc* desc,
                    const omt_resample_desc* desc_host, const int32_t* tab, const int32_t* tab_host, long long tab_len,
                    int B, int oh, int ow, uint8_t* out, omt_stream_t stream);

/* One clip of omt_resample_clips.  Table offsets count int32 words; each table entry is 4 words. */
typedef struct {
  long long src;          /* byte offset of the clip's (F, H, W, 3) bytes in src */
  int H, W;               /* source frame size */
  int y0, x0;             /* origin of the window the resize reads, in the (flipped) source frame */
  int wh, ww;             /* window size: the input length of the vertical / horizontal table */
  int rh, rw;             /* resized size: the output length of the vertical / horizontal table */
  int cy, cx;             /* crop origin in the resized frame */
  int flip;               /* 1: the source frame is mirrored left-right before the window is taken */
  int tv, th;             /* vertical table [rh][4] at tab + tv, horizontal table [rw][4] at tab + th */
  int form;               /* 0: torch's separable bilinear kernel, 1: its channels-last four-weight kernel */
} omt_clip_desc;

/* The Latte video loaders' transform of a ragged batch of (F, H_i, W_i, 3) uint8 clips (Diffusion/Latte/datasets:
 * ToTensorVideo, RandomHorizontalFlipVideo, UCFCenterCropVideo / CenterCropResizeVideo, Normalize), torch's fp32 CPU
 * arithmetic bit for bit.  out (B, 3, F, oh, ow) fp32, channel-planar:
 *   v = lut[byte]                                                       (to_tensor: u / 255, from the host)
 *   source column of window column c: x0 + c, or W - 1 - (x0 + c) when flipped; row: y0 + r
 *   axis entries (i0, i1, l0, l1) of output indices cy + y and cx + x, x_ab = v[i_a h][i_b w]; F.interpolate bilinear:
 *     form 0: t_a = fma(x_a0, l0w, x_a1 * l1w), then fma(t_0, l0h, t_1 * l1h)
 *     form 1: w_ab = l_a h * l_b w, then fma(x_11, w_11, fma(x_10, w_10, fma(x_00, w_00, x_01 * w_01)))
 *   (value - mean_c) / std_c, true division                          (Normalize)
 * The axis tables are int32 [n_out][4] = (i0, i1, l0 bits, l1 bits), built on the host in fp32 without contraction.
 * norm: fp32 [262] on the device: the 256-entry byte table, then mean[3], then std[3].  src: packed source bytes
 * (src_bytes of them); desc [B]: device table, 8-byte aligned; tab [tab_len] int32, 16-byte aligned.  desc_host /
 * tab_host: the same tables in host memory, checked before the launch (every clip inside src, every window inside its
 * frame, every table inside tab, every index inside its axis, the crop inside the resized size); they must equal the
 * device copies.  One launch for the batch. */
int omt_resample_clips(const uint8_t* src, long long src_bytes, const omt_clip_desc* desc, const omt_clip_desc* desc_host,
                       const int32_t* tab, const int32_t* tab_host, long long tab_len, const float* norm, int B, int F,
                       int oh, int ow, float* out, omt_stream_t stream);

/* The FVD metric's preprocess (OmniTokenizer/fvd/fvd.py:18-29) of B clips of F frames: the same tables, descriptors and
 * checks as omt_resample_clips (form 0 for the multi-threaded F.interpolate, no flip, no window, no crop), but
 *   v = lut[byte]  (lut: fp32 [256], float(byte) or the value a byte map sends the byte to; with sel != NULL, lut is
 *                   fp32 [2][256] and clip b reads table sel[b], 0 or 1 -- omt_u8_norm_select writes it on the device)
 *   out = 2 * y / 255 - 1 in that order, true division,
 * written channels-last: out (B, F, oh, ow, 4) fp32, 16-byte aligned, channel 3 zero (the I3D input of omt_conv3d). */
int omt_fvd_preprocess(const uint8_t* src, long long src_bytes, const omt_clip_desc* desc, const omt_clip_desc* desc_host,
                       const int32_t* tab, const int32_t* tab_host, long long tab_len, const float* lut,
                       const int32_t* sel, int B, int F, int oh, int ow, float* out, omt_stream_t stream);

/* The FVD preprocess of evaluation/common_metrics_on_video_quality (fvd/styleganv and fvd/videogpt preprocess_single)
 * of B clips of F frames: the descriptors and axis tables of omt_resample_clips (no flip, no window; desc.form picks
 * torch's bilinear kernel), torch's fp32 CPU arithmetic bit for bit.  Each source sample is read in one of three forms:
 *   OMT_FVDS_U8:        uint8 (F, H, W, 3) clips, v = (float)byte / 255 (C == 3);
 *   OMT_FVDS_F32:       fp32 (F, C, H, W) clips, C 1 (grey, every channel reads it) or 3, v used as is (styleganv);
 *   OMT_FVDS_F32_TRUNC: the same fp32 clips through videogpt's byte round trip, v = (float)(uint8)(x * 255) / 255
 *                       (the low byte of the truncated int32, as numpy's astype on x86-64);
 *   out = (y - 0.5) * 2, two roundings,
 * written channels-last: out (B, F, oh, ow, 4) fp32, 16-byte aligned, channel 3 zero (the I3D input of omt_conv3d).
 * desc.src and src_elems count elements of src (bytes, or floats); a clip's frames follow each other from desc.src, so
 * a clip stored with more than F frames is read as its first F. */
#define OMT_FVDS_U8 0
#define OMT_FVDS_F32 1
#define OMT_FVDS_F32_TRUNC 2
int omt_fvd_suite_preprocess(const void* src, long long src_elems, int form, int C, const omt_clip_desc* desc,
                             const omt_clip_desc* desc_host, const int32_t* tab, const int32_t* tab_host,
                             long long tab_len, int B, int F, int oh, int ow, float* out, omt_stream_t stream);

/* The Inception Score's input (calculate_is.py's nn.Upsample(size=(299, 299), mode='bilinear') on the CPU, or no resize)
 * of B clips of F frames: the kernel body, descriptors, axis tables and checks of omt_fvd_suite_preprocess in two of its
 * forms, OMT_FVDS_U8 (uint8 (F, H, W, 3), v = (float)byte / 255) and OMT_FVDS_F32 (fp32 (F, 3, H, W), v as is), and
 * out = y with no affine, written channels-last: out (B, F, oh, ow, 4) fp32, 16-byte aligned, channel 3 zero.  Axis
 * tables whose entries are (i, i, 1.0, 0.0) copy the frame bit for bit (the network run at the input's own size). */
int omt_is_preprocess(const void* src, long long src_elems, int form, const omt_clip_desc* desc,
                      const omt_clip_desc* desc_host, const int32_t* tab, const int32_t* tab_host, long long tab_len,
                      int B, int F, int oh, int ow, float* out, omt_stream_t stream);

/* vqgan_eval.py's --infer_downsample (:121-136, then :147-148) of B clips of F frames, torch's fp32 CPU arithmetic bit for
 * bit: the descriptors and axis tables of omt_resample_clips (no flip, no window, no crop; desc.form picks torch's
 * bilinear kernel for the call shape and thread count).  Each source sample is read in one of two forms:
 *   OMT_DS_F32: the decoder's fp32 reconstruction 'b c t h w', (3, F, H, W) per clip from desc.src (floats),
 *               v = clamp(x + 0.5, 0, 1)   (the reconstruction side);
 *   OMT_DS_U8:  the loader's uint8 (F, H, W, 3) clips from desc.src (bytes), v = lut[byte] (lut: fp32 [256], e.g.
 *               VideoNorm(byte) + 0.5; with sel != NULL, lut is fp32 [2][256] and clip b reads table sel[b], 0 or 1 --
 *               omt_u8_norm_select writes it on the device)   (the real side);
 *   out = (uint8)(y * 255): the product truncated to int32 and its low byte kept, as .byte() does on x86-64,
 * written channels-last: out (B, F, oh, ow, 3) uint8, the frames I3D.logits reads.  lut / sel are ignored for
 * OMT_DS_F32 (NULL allowed).  src_elems counts elements of src. */
#define OMT_DS_F32 0
#define OMT_DS_U8 1
int omt_eval_downsample(const void* src, long long src_elems, int form, const omt_clip_desc* desc,
                        const omt_clip_desc* desc_host, const int32_t* tab, const int32_t* tab_host, long long tab_len,
                        const float* lut, const int32_t* sel, int B, int F, int oh, int ow, uint8_t* out,
                        omt_stream_t stream);

/* Unit3D of the FVD I3D (fvd/pytorch_i3d.py:59-131) as an implicit GEMM in 3xTF32 on sm_90a wgmma:
 *   y[m, n] = act(sum_k A[m, k] W[n, k] + bias[n]),  m = ((b To + to) Ho + ho) Wo + wo,  n < N,  act = ReLU if relu
 *   A[m, (dt, dh, dw, c)] = x[b][to st - pt + dt][ho sh - ph + dh][wo sw - pw + dw][c], zero outside the volume
 * x: fp32 channels-last [B][T][H][W][Cs], 16-byte aligned; Cs a multiple of 32, or 4 (the network input: a k-block of
 * 32 values then holds 8 taps).  K = kt kh kw Cs, rounded up to a multiple of 32 when Cs == 4.
 * w_hi / w_lo: fp32 [round_up(N, 128)][K] (hi = tf32(W), lo = W - hi, BatchNorm folded in, rows >= N zero), 16-byte
 * aligned; bias: fp32 [N].  (pt, ph, pw): the front padding (SAME: pad // 2); the back padding is implied by To, Ho, Wo.
 * y: row m at y + m * ldy, N columns written and no others (N even, ldy >= N even, 8-byte aligned), so a branch of an
 * Inception block writes its slice of the block's concat buffer in place.  The wgmma accumulator is added into an fp32
 * sum on the CUDA cores every 64 values of K, so the tensor core's accumulation error does not grow with K. */
int omt_conv3d(const float* x, int Cs, int B, int T, int H, int W, const float* w_hi, const float* w_lo, int K,
               const float* bias, int N, int kt, int kh, int kw, int st, int sh, int sw, int pt, int ph, int pw,
               int To, int Ho, int Wo, float* y, int ldy, int relu, omt_stream_t stream);

/* MaxPool3dSamePadding (fvd/pytorch_i3d.py:24-56) on channels-last fp32 [B][T][H][W][Cs] -> [B][To][Ho][Wo][Cs] (Cs a
 * multiple of 4, both 16-byte aligned): taps outside the volume are F.pad's zeros; max_pool3d's CPU rule, exact. */
int omt_maxpool3d(const float* x, int Cs, int B, int T, int H, int W, int kt, int kh, int kw, int st, int sh, int sw,
                  int pt, int ph, int pw, int To, int Ho, int Wo, float* y, omt_stream_t stream);

/* The I3D head (fvd/pytorch_i3d.py:319-365): x [B][T][7][7][Cs] fp32 -> AvgPool3d([2, 7, 7], stride 1) over the first C
 * channels -> logits[t] = W[N][C] . p[t] + bias -> out [B][N] = the mean over the T - 1 steps.  T >= 2. */
int omt_i3d_head(const float* x, int Cs, int C, int B, int T, const float* w, const float* bias, int N, float* out,
                 omt_stream_t stream);

/* pytorch-fid's InceptionV3 preprocess (inception.py:147-151, after fid_score.py's ToTensor) of B images of H x W: the
 * tables, descriptors and checks of omt_fvd_preprocess with F = 1, but the division comes before the resize:
 *   v = lut[byte]  (lut: fp32 [256], byte / 255 or the value a byte map sends the byte to; with sel != NULL, lut is
 *                   fp32 [2][256] and image b reads table sel[b])
 *   out = 2 * y - 1, two roundings,
 * written channels-last: out (B, oh, ow, 4) fp32, 16-byte aligned, channel 3 zero (the input of the first conv). */
int omt_fid_preprocess(const uint8_t* src, long long src_bytes, const omt_clip_desc* desc, const omt_clip_desc* desc_host,
                       const int32_t* tab, const int32_t* tab_host, long long tab_len, const float* lut,
                       const int32_t* sel, int B, int oh, int ow, float* out, omt_stream_t stream);

/* 2-D pooling of the FID and IS InceptionV3s on channels-last fp32 [B][H][W][Cs] -> y, output pixel p = (b Ho + ho) Wo + wo,
 * channel c < C at y[p * ldy + c] (C, Cs, ldy multiples of 4; x and y 16-byte aligned), so a pool branch writes its
 * slice of the concat buffer in place.  Window (kh, kw), stride (sh, sw), symmetric padding (ph, pw) <= half the window;
 * only taps inside the image take part, in (h, w) order, as torch's CPU kernels visit them:
 *   OMT_POOL_MAX: max_pool2d (the padding never wins; NaN propagates);
 *   OMT_POOL_AVG: avg_pool2d(count_include_pad=False): the fp32 sum, then one true division by the count of taps;
 *   OMT_POOL_AVG_PAD: avg_pool2d(count_include_pad=True): the same sum, then one true division by torch's window size
 *                     (min(h0 + kh, H + ph) - h0) (min(w0 + kw, W + pw) - w0), h0 = ho sh - ph, w0 = wo sw - pw.
 * All exact.  The global AdaptiveAvgPool2d(1) of an h x w map is OMT_POOL_AVG with an h x w window. */
#define OMT_POOL_MAX 0
#define OMT_POOL_AVG 1
#define OMT_POOL_AVG_PAD 2
int omt_pool2d(const float* x, int Cs, int C, int B, int H, int W, int kh, int kw, int sh, int sw, int ph, int pw,
               int Ho, int Wo, float* y, int ldy, int mode, omt_stream_t stream);

/* Frame-pair metrics (evaluation/common_metrics_on_video_quality, OmniTokenizer/modules/lpips.py) take P frames
 * (P, H, W, 3) channels last in one of two forms:
 *   OMT_Q_U8:  uint8, each byte standing for lut[t][byte] (fp32 [n_tab][256], or [n_tab][3][256] per channel), with
 *              t = sel[p] (int32 [P]) or 0 when sel is NULL;
 *   OMT_Q_F32: fp32 values (no tables).
 * Every reduction runs in a fixed order (no floating-point atomics): two runs give the same bits. */
#define OMT_Q_U8 0
#define OMT_Q_F32 1

/* calculate_psnr.py's img_psnr and calculate_ssim.py's calculate_ssim_function (3 channels) of pairs (a[p], b[p]):
 *   sse[p]  = sum over C H W of (a - b)^2, the fp32 values widened to fp64 (PSNR follows on the host from
 *             mse = sse / (3 H W): 100 if mse < 1e-10, else 20 log10(1 / sqrt(mse)));
 *   ssim[p] = the mean over channels, in channel order, of the mean over the valid (H - 10) x (W - 10) map of
 *             ((2 mu1 mu2 + C1)(2 s12 + C2)) / ((mu1^2 + mu2^2 + C1)(s1 + s2 + C2)), C1 = 0.01^2, C2 = 0.03^2, from
 *             the five maps mu1, mu2, E[x^2], E[y^2], E[xy] filtered with taps[11] (fp64; cv2.getGaussianKernel(11,
 *             1.5)) along w, then along h, in fp64.
 * H, W >= 11.  sse, ssim: fp64 [P]. */
int omt_psnr_ssim(const void* a, const float* lut_a, const int32_t* sel_a, const void* b, const float* lut_b,
                  const int32_t* sel_b, int form, int P, int H, int W, const double* taps, double* sse, double* ssim,
                  omt_stream_t stream);

/* LPIPS network input of P frames: calculate_lpips.py's x * 2 - 1, then ScalingLayer's (x - shift_c) / scale_c, fp32
 * rounded after every op, written as out [P][H][W][4] (16-byte aligned, channel 3 zero; the omt_conv3d input layout).
 * OMT_Q_U8: lut [n_tab][3][256] holds the whole chain per byte (built on the host), sel picks the table per frame;
 * OMT_Q_F32: shift_scale fp32 [6] = (shift_0..2, scale_0..2) on the device, lut and sel NULL. */
int omt_lpips_input(const void* x, const float* lut, const int32_t* sel, const float* shift_scale, int form, int P,
                    int H, int W, float* out, omt_stream_t stream);

/* LPIPS head at one VGG tap (lpips.py:97-108): x fp32 [2P][h][w][Cs], pair p = images p and p + P, C channels; per pair
 *   taps_out[tap * P + p] = mean over pixels of sum_c lin_w[c] (x_c / (|x| + 1e-10) - y_c / (|y| + 1e-10))^2
 * with |x| = sqrt(sum_c x_c^2) (fp32 per pixel, the pixel sum in fp64).  If total != NULL, total[p] = taps_out[0][p]
 * + ... + taps_out[tap][p], added in fp32 in that order (the earlier taps' launches must precede this one). */
int omt_lpips_head(const float* x, int Cs, int C, int P, int h, int w, const float* lin_w, int tap, float* taps_out,
                   float* total, omt_stream_t stream);

/* The per-pixel map of one LPIPS tap (the lpips package's spatial=True, before the upsample): x fp32 [2P][h][w][Cs],
 * pair p = images p and p + P, C channels; map fp32 [P][h][w] gets, per pixel, exactly the term omt_lpips_head sums:
 *   sum_c lin_w[c] (x_c / (|x| + 1e-10) - y_c / (|y| + 1e-10))^2,  |x| = sqrt(sum_c x_c^2)  (fp32). */
int omt_lpips_map(const float* x, int Cs, int C, int P, int h, int w, const float* lin_w, float* map,
                  omt_stream_t stream);

/* One tap map [P][h][w] fp32 of omt_lpips_upsample_mean (4-byte aligned). */
typedef struct {
  const float* map;
  int h, w;
} omt_lpips_tap;
#define OMT_LPIPS_MAX_TAPS 5

/* The lpips package's spatial=True tail (lpips.py upsample and `val += res[kk]`) for P pairs: per output pixel of H x W,
 *   v = 0; for k in 0 .. n_taps - 1: v += up_k,
 * up_k = nn.Upsample(size=(H, W), mode='bilinear', align_corners=False) of tap k in torch's fp32 CUDA arithmetic:
 * scale = (float)h / (float)H, src = max(fmaf(dst + 0.5f, scale, -0.5f), 0), i0 = (int)src, i1 = i0 + (i0 < h - 1),
 * l1 = src - i0, l0 = 1 - l1 (likewise along w), top = fmaf(w0, a[i0][j0], w1 a[i0][j1]), bottom likewise on row i1,
 * up = fmaf(h0, top, h1 bottom); a tap of the output's size is copied.  taps: host array of n_taps (1 .. 5) entries.
 * map_out (NULL: not written): fp32 [P][H][W] of v.  mean_out[p] = (float)(the fp64 sum of pair p's v / (H W)), summed
 * in a fixed order (no atomics: two runs give the same bits). */
int omt_lpips_upsample_mean(const omt_lpips_tap* taps, int n_taps, int P, int H, int W, float* map_out,
                            float* mean_out, omt_stream_t stream);

/* Row softmax of the Inception Score's classifier (calculate_is.py's F.softmax over dim 1), fp32: rows of N logits at
 * x + r * ldx -> y + r * ldy, per row m = max, e_j = exp(x_j - m) (the difference and exp in fp64, rounded once to fp32),
 * s = the fp32 sum of e in a fixed order, y_j = e_j / s (true division).  N >= 1, ldx, ldy >= N, 4-byte aligned. */
int omt_softmax_rows(const float* x, int ldx, int rows, int N, float* y, int ldy, omt_stream_t stream);

/* The split reduction of the Inception Score (calculate_is.py:44-55 with scipy.stats.entropy), in fp64 in a fixed order
 * (no floating-point atomics: two runs give the same bits).  p: fp32 probabilities, rows of N at p + r * ldp; split k
 * holds rows [k n, (k + 1) n).  Per split:
 *   py[k][j]  = (sum over the split's rows of p[r][j]) / n                      (col_mean: fp64 [splits][N])
 *   kl[k]     = mean over the split's rows of sum_j x_j log(x_j / y_j), x = p[r] / sum(p[r]), y = py[k] / sum(py[k]),
 *               terms with x_j == 0 contributing 0                           (kl: fp64 [splits])
 * The score of split k is exp(kl[k]); the host takes it, and the mean and standard deviation over the splits. */
int omt_inception_score(const float* p, int ldp, int N, int n, int splits, double* col_mean, double* kl,
                        omt_stream_t stream);

/* The pixels vqgan_eval.py's image loop hands pytorch-fid when it saves to a .jpg / .JPEG path (vqgan_eval.py:205-220,
 * fid_score.py:107): Pillow's img.save(f, "JPEG", quality=q) then Image.open(f).convert("RGB"), byte for byte, as
 * libjpeg-turbo computes them: baseline 4:2:0, ISLOW forward and inverse DCT, h2v2 fancy upsampling (a chroma plane at
 * most 2 samples wide is replicated 2 x 2), all in int32 (oracle/jpeg_oracle.py restates the chain).  Entropy coding is
 * lossless, so no bitstream is made.
 *   src, dst: (B, H, W, 3) uint8 RGB, contiguous, on the device; dst may not overlap src or scratch.
 *   qtables: HOST memory, uint16 [2][64] (luminance, chrominance) in natural order, every entry 1..255; copied into the
 *            launch, so the caller may reuse the array once the call returns.
 *   scratch: the decoded Y, Cb and Cr planes, B (Hp Wp + 2 (Hp / 2) (Wp / 2)) bytes with Hp = 16 ceil(H / 16) and
 *            Wp = 16 ceil(W / 16); 8-byte aligned; its contents are overwritten.
 * B >= 0 (B = 0 launches nothing), H, W >= 1, Hp Wp 3 / 2 < 2^31.  Two launches: one CTA per four MCUs, then a thread
 * per output pixel. */
int omt_jpeg_roundtrip_u8(const uint8_t* src, uint8_t* dst, int B, int H, int W, const uint16_t* qtables,
                          uint8_t* scratch, omt_stream_t stream);

/* Inverse Rearrange of to_pixels (omnitokenizer.py:1008 / :1015): P [rows, K] -> video (B,Cin,T,H,W).  Rows, features and
 * geometry as omt_patchify_ln: Cin >= 1, p > 0 a multiple of 4 dividing H and W, pt > 0 dividing T - 1 for the rest frames. */
int omt_unpatchify(const float* P, float* video, int B, int Cin, int T, int H, int W, int p, int pt,
                   int first, omt_stream_t stream);

/* Un-patchify fused with the consumers' uint8 conversion: u8 = trunc(clamp(x * mul + add, lo, hi) * post), written
 * channels-LAST (B, T, H, W, Cin).  (mul, add, lo, hi, post) = (1, .5, 0, 1, 255) is vqgan_eval.py:139,147-148
 * `(clamp(x_recons + 0.5, 0, 1) * 255).byte()` and Latte's sample_ddp.py:206; (255, 128, 0, 255, 1) is DiT's
 * sample_ddp.py:163.  Each step rounds in fp32 like the torch expression, so the bytes are identical to it.  Geometry as
 * omt_unpatchify (Cin >= 1, p > 0, pt > 0 for the rest frames). */
int omt_unpatchify_u8(const float* P, uint8_t* out, int B, int Cin, int T, int H, int W, int p, int pt,
                      int first, float mul, float add, float lo, float hi, float post, omt_stream_t stream);

/* PEG (attention.py:298-338) + residual: y[r,:] = x[r,:] + bias + sum_k w[k,:] * x[nbr[r % rows_per_b, k] , :]
 * nbr: int32 [rows_per_b, 27] canonical neighbour rows inside one batch element, -1 = zero padding
 * (the spatial stencil or the reference's literally-reshaped "scrambled" temporal one, built by the host);
 * w27: weights repacked [27, C]. */
int omt_peg(const float* x, float* y, const float* w27, const float* bias, const int32_t* nbr,
            int B, int rows_per_b, int C, omt_stream_t stream);

/* Same operation as omt_peg, tiled: the stencil is evaluated in volume space (t2,h2,w2) with a
 * shared-memory halo tile and a sliding register window (9 loads per output instead of 27).
 * temporal != 0 selects the reference's literally-reshaped '(b h w) t d' volume (attention.py:313-319),
 * causal != 0 pads t by (2,0) instead of (1,1).  x, y: canonical [B*T*h*w, C]. */
int omt_peg_volume(const float* x, float* y, const float* w27, const float* bias, int B, int T, int h, int w,
                   int C, int temporal, int causal, omt_stream_t stream);

/* Packed batch ("varlen"): samples of different lengths in one canonical buffer, every sample on the same h x w grid.
 * Sample b owns latent frames [t_off[b], t_off[b+1]) = canonical rows [t_off[b]*N, t_off[b+1]*N), N = h*w, and has
 * T'_b = t_off[b+1] - t_off[b] frames.  t_off: int32 [B+1] in DEVICE memory (read by the kernel); t_off_host: the same
 * B+1 values in HOST memory, checked before the launch (t_off[0] == 0, every T'_b in 1..17, t_off[B]*N == M rows) and
 * used to size the grid.  Each sample's output equals the uniform entry point's on that sample alone, bit for bit.
 *
 * omt_peg_volume over a packed batch, in ONE launch: zero padding at each sample's own edges (no tile reads a
 * neighbour's rows); in the temporal volume the '(b h w) t d' reshape is taken per sample with its own T'_b. */
int omt_peg_volume_varlen(const float* x, float* y, const float* w27, const float* bias, const int32_t* t_off_host,
                          const int32_t* t_off, int B, int M, int h, int w, int C, int temporal, int causal,
                          omt_stream_t stream);

/* In-place rope + l2norm + per-dim scale on q and k (attention.py:417-421, :435-437).
 * q[M, heads*64] (ld ldq), k likewise; cos/sin [N, 32] or NULL (no rope; temporal blocks);
 * the rope position of row r is r % N. */
int omt_qk_prep(float* q, int ldq, float* k, int ldk, const float* q_scale, const float* k_scale,
                const float* rope_cos, const float* rope_sin, int M, int N, int heads,
                omt_stream_t stream);

/* Full (non-causal) attention over n_seq sequences of N contiguous canonical rows, head dim 64:
 * o = softmax(scale * q k^T) v   (attention.py:451, SDPA branch: no additive bias).  N % 64 == 0.
 * All three attention cores: when o_hi != NULL the result is written as fp16 hi / lo operand planes
 * (leading dimension ldo) for the out-projection GEMM instead of fp32 o (o may then be NULL). */
int omt_attn_spatial(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                     float* o, uint16_t* o_hi, uint16_t* o_lo, int ldo, int n_seq, int N, int heads, float scale,
                     omt_stream_t stream);

/* omt_attn_spatial on the operand planes written by omt_linear_h(OMT_EPI_QKV_PLANES): wgmma f16 core, Q / K / V tiles
 * straight from TMA (V as an MN-major operand: no transpose), N % 128 == 0.
 * qk_plane_scale = q_plane_scale * k_plane_scale; vinv [heads][n_seq * N]. */
int omt_attn_spatial_h(const uint16_t* q_hi, const uint16_t* q_lo, int ldq, const uint16_t* k_hi, const uint16_t* k_lo, int ldk,
                       const uint16_t* v_hi, const uint16_t* v_lo, int ldv, const float* vinv, float qk_plane_scale,
                       float* o, uint16_t* o_hi, uint16_t* o_lo, int ldo, int n_seq, int N, int heads, float scale,
                       omt_stream_t stream);

/* f16x1 (throughput) form of omt_attn_spatial_h on the hi planes alone: S = Q_hi . K_hi^T and O += P''_hi . V_hi take ONE
 * f16 wgmma per k-step (P'' = p * vinv * 2^e rounded to fp16, as in the three-product core).  o fp32, or o_hi != NULL:
 * the hi plane of O (fp16(o)) for the f16x1 out-projection; o may then be NULL.  NOT reference-exact. */
int omt_attn_spatial_h1(const uint16_t* q_hi, int ldq, const uint16_t* k_hi, int ldk, const uint16_t* v_hi, int ldv,
                        const float* vinv, float qk_plane_scale, float* o, uint16_t* o_hi, int ldo, int n_seq, int N,
                        int heads, float scale, omt_stream_t stream);

/* 8x8 (ws x ws, ws*ws == 64) window attention with relative position bias (attention.py:254-286):
 * o = softmax(scale * q k^T + bias[head]) v within each window of the (h, w) token grid.
 * bias: [heads, 64, 64] already gathered from the 225-entry table. */
int omt_attn_window(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                    float* o, uint16_t* o_hi, uint16_t* o_lo, int ldo, const float* bias, int n_frames, int h, int w, int ws, int heads,
                    float scale, omt_stream_t stream);

/* Temporal attention: for every (b, n) a sequence over t' (rows b*T*N + t*N + n), optional causal
 * mask (attention.py:451 is_causal); 1 <= T <= 17. */
int omt_attn_temporal(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                      float* o, uint16_t* o_hi, uint16_t* o_lo, int ldo, int B, int T, int N, int heads, float scale, int causal,
                      omt_stream_t stream);

/* omt_attn_temporal over a packed batch (t_off_host / t_off / M as for omt_peg_volume_varlen), in ONE launch: pixel n of
 * sample b attends over the rows (t_off[b] + t)*N + n, t < T'_b.  The kernel is instantiated for the longest sample
 * and skips every step past T'_b, so each output goes through the same operations as the <T'_b> instance. */
int omt_attn_temporal_varlen(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv,
                             float* o, uint16_t* o_hi, uint16_t* o_lo, int ldo, const int32_t* t_off_host,
                             const int32_t* t_off, int B, int M, int N, int heads, float scale, int causal,
                             omt_stream_t stream);

/* pre_vq_conv (omnitokenizer.py:144-154) [+ F.normalize(dim=channels) :251-252]:
 * z[M, cd] = x[M, C] . Wt^T + b, cd in {8, 16}; l2 != 0 divides each row by max(||z||, 1e-12). */
int omt_pre_vq(const float* x, int ldx, const float* Wt, const float* b, float* z, int M, int C, int cd,
               int l2, omt_stream_t stream);

/* Codebook.forward nearest-neighbour search (modules/codebook.py:82-86), cd == 8:
 * d[n,k] = (sum z^2 - 2 z.E_k) + sum E_k^2 in that association, idx = first argmin.
 * e2: [n_codes] precomputed sum E^2; n_codes % 64 == 0 and n_codes <= 41856 (an eighth of the table, 36 B per code,
 * and the z rows of a 512-row block share 200 KB of shared memory; launches of few rows take 256-row blocks and accept
 * up to 43648).  Pad a smaller table with zero rows whose e2 is +inf: they never win.  Also accumulates
 * counts[n_codes] (int32, caller zeroes) -- the fixed-size replacement of torch.unique (:65).  counts may be NULL.
 * One launch, no workspace. */
int omt_vq_search(const float* z, const float* E, const float* e2, int M, int n_codes,
                  int64_t* idx, int32_t* counts, omt_stream_t stream);

/* The whole VQ lookup in ONE launch: pre_vq_conv (omnitokenizer.py:248) + F.normalize (:251-252, l2 != 0) + the search
 * above.  x [M, C] is the encoder output; z [M, 8] receives the (normalised) projection (may be NULL).  A cluster of 8
 * CTAs shares a block of 512 rows: each CTA projects 64 of them, broadcasts z through distributed shared memory and
 * searches all 512 against its eighth of the table; per-row minima meet again in the row's owner CTA. */
int omt_vq_fused(const float* x, int ldx, const float* Wt, const float* b, int C, int l2, float* z,
                 const float* E, const float* e2, int M, int n_codes, int64_t* idx, int32_t* counts,
                 omt_stream_t stream);

/* Decode-side lookup: F.embedding gather (omnitokenizer.py:270) + post_vq_conv Linear(cd, C) (:156-160).
 * If idx != NULL rows come from E[idx[r]]; else from zc[M, cd].  X[M, C] = row . Wt^T + b, C % 4 == 0, C <= 1024.
 * When z_st_from != NULL (forward(): straight-through, codebook.py:120) the row is (E[idx]-z)+z and is
 * also written to zq_out[M, cd] (may be NULL). */
int omt_post_vq(const int64_t* idx, const float* E, const float* zc, const float* z_st_from,
                float* zq_out, const float* Wt, const float* b, float* X, int M, int C, int cd,
                omt_stream_t stream);

/* ---- f16x3 path: operands as 16-bit planes ------------------------------------------------------------
 * An fp32 matrix X is carried as hi = fp16(X) (round to nearest, saturating) and lo = fp16((X - hi) * 2^11), two
 * uint16 matrices with a common leading dimension: X ~= hi + lo * 2^-11 to 2^-23 |X| for |X| < 65504.
 * Producers below write the planes directly; weights are split once on the host.
 * ROW-SCALED form: a producer that sees whole rows (LayerNorm, patch gather) multiplies the row by the power of two
 * that puts its largest magnitude in [2^14, 2^15) and stores hi = fp16(x'), lo = fp16(x' - hi) UNSCALED plus the inverse
 * scale per row; the weights carry one such scale per matrix.  The GEMM then needs ONE accumulator instead of two
 * (256-wide tiles AND double buffering).  Both A operands of a dual-A call use the same form. */
typedef struct omt_linear_h_args {
  const uint16_t* a_hi; const uint16_t* a_lo;      /* A planes [M, lda] */
  const float* a_rs; const float* a2_rs;           /* non-NULL: ROW-SCALED planes (below): inverse row scales [rows of A] */
  float w_scale;                                   /* row-scaled form: inverse of the per-matrix scale of the W planes */
  const uint16_t* a2_hi; const uint16_t* a2_lo;    /* optional second A (dual-A form, columns >= n_split), same lda / row map */
  int n_split;                                     /* multiple of 128 (a whole output tile) */
  int lda, a_seg, a_seg_stride, a_seg_off;         /* lda % 8 == 0; row map as in omt_linear (segments of 64 rows) */
  const uint16_t* w_hi; const uint16_t* w_lo;      /* W planes [N rounded up to 256, K], K % 64 == 0 */
  float* c; int ldc, c_seg, c_seg_stride, c_seg_off;   /* fp32 output (OMT_EPI_NONE / OMT_EPI_QKV); row map segments of 32 rows */
  uint16_t* u_hi; uint16_t* u_lo; int ldu;         /* OMT_EPI_GEGLU: output planes U[M, N/2] */
  int M, N, K;
  const float* bias; const float* residual; int ldr;   /* residual may alias c */
  int epilogue;
  const float* q_scale; const float* k_scale; const float* rope_cos; const float* rope_sin;   /* OMT_EPI_QKV, as omt_linear2 */
  int qk_cols, tokens;
  /* OMT_EPI_QKV_PLANES: output planes u_hi / u_lo [M, N] (ldu): q / k heads multiplied by the static powers of two
   * q_plane_scale / k_plane_scale (|q| <= max|q_scale| after l2norm, so the bound is exact), v heads scaled per
   * (row, head) with the inverse scales written to vinv [N_v / 64][M]; lo planes unscaled. */
  float q_plane_scale, k_plane_scale;
  float* vinv;
  /* statically bounded operands: a_rs_uniform > 0 (with a_rs == NULL) = row-scaled form with ONE inverse scale for all rows;
   * u_scale > 0 (OMT_EPI_GEGLU) = write the U planes in that form, multiplied by u_scale (|U| * u_scale < 65504 is the
   * caller's guarantee: |gelu(g) * a| <= |g| |a| and both are bounded through the LayerNorm in front of the GEMM). */
  float a_rs_uniform, u_scale;
} omt_linear_h_args;

/* Same contract as omt_linear / omt_linear2 (nn.Linear + the fused epilogues) on operand planes. */
int omt_linear_h(const omt_linear_h_args* args, omt_stream_t stream);

/* f16x1 (throughput) form of omt_linear_h: the same argument block, forms and epilogues, ONE f16 product A_hi . W_hi per
 * k-step with fp32 accumulation.  a_lo, a2_lo, w_lo and u_lo must be NULL (a non-NULL one is rejected), so no caller can
 * take the result for the three-product one.  Row-scaled / uniform-scaled A: the epilogue multiplies by a_rs[row] * w_scale
 * (a_rs_uniform * w_scale); the 2^11 form (a_rs == NULL, a_rs_uniform == 0): hi planes of unscaled values, no factor.
 * OMT_EPI_QKV_PLANES and OMT_EPI_GEGLU write the hi planes only (u_hi; vinv as before).  Results are NOT reference-exact:
 * expect relative errors near 2^-11 per product term. */
int omt_linear_h1(const omt_linear_h_args* args, omt_stream_t stream);

/* LayerNorm as omt_layernorm with plane outputs for the GEMM that consumes it:
 * y (fp32, may be NULL), (y_hi, y_lo) planes of the normalised row, and optionally (x_hi, x_lo) planes of the RAW
 * input row -- Attention.forward projects k, v from the un-normalised input (attention.py:407-412).  lds = leading
 * dimension of every plane (lds % 8 == 0).  The row map applies to x / y; planes are written at the LOGICAL row.
 * y_rs / x_rs != NULL: that plane pair is written in the row-scaled form and the inverse row scales go to y_rs / x_rs [M]. */
int omt_layernorm_h(const float* x, int ldx, float* y, int ldy, uint16_t* y_hi, uint16_t* y_lo, float* y_rs,
                    uint16_t* x_hi, uint16_t* x_lo, float* x_rs, int lds, const float* w, const float* b,
                    int M, int C, float eps, int seg, int seg_stride, int seg_off, omt_stream_t stream);

/* Tuning knobs (process-wide): "pdl" = 0 (default; measured 2-4 % slower when on) | 1 programmatic dependent launch;
 * "peg_kernel" = 4 (default: cp.async zero-fill halo gather + packed f32x2 FMAs) | 3 (register-staged gather; also the
 * fallback for T > 64 or w > 254); identical bits;
 * "attn_kernel" = 3 (default: wgmma 3xTF32 spatial attention core when N % 128 == 0) | 1 (CUDA-core fp32);
 * "f16_bn" = 0 (default) | 128 | 256: accepted for compatibility; omt_linear_h always runs 128 x 128 tiles on sm_90;
 * "attn_f16_ctas" = 2 (default) | 1: accepted for compatibility; omt_attn_spatial_h has one kernel shape on sm_90. */
int omt_set_option(const char* name, int value);

#ifdef __cplusplus
}
#endif
#endif /* OMNITOK_B200_H_ */
