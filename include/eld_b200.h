/* eld_b200.h - C ABI of the H100-native ELD hot path (libeld_b200.so).
 *
 * The reference (Vandermode/ELD) has no FFI layer: its seams are Python duck-typed protocols
 * (SURVEY.md 8b).  This header is what a binding for that seam would call; every entry point
 * names the reference interface it replaces (file:line relative to the reference root).
 *
 * Conventions
 *   - every function returns 0 on success or a negative ELD_E* code; eld_last_error() returns a
 *     thread-local, NUL-terminated description of the last failure on the calling thread;
 *   - the caller owns ALL buffers (device pointers normally come from torch tensors); the library
 *     never frees caller memory and never synchronises the device unless documented;
 *   - `stream` is a cudaStream_t passed as void* (so that this header needs no CUDA include);
 *   - no CPU fallback: without a CUDA device every compute entry point fails with ELD_E_CUDA.
 *   - plain pointers and sizes only - no torch types.
 */
#ifndef ELD_B200_H
#define ELD_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ELD_OK            0
#define ELD_E_ARG        -1   /* bad argument (null pointer, negative size, unsupported shape) */
#define ELD_E_CUDA       -2   /* CUDA runtime / driver error (text in eld_last_error)          */
#define ELD_E_UNSUPPORTED -3  /* valid request the library does not implement                   */
#define ELD_E_WORKSPACE  -4   /* caller workspace too small                                     */

typedef struct eld_ctx eld_ctx;

/* ABI version of this header; eld_abi_version() must return it. */
#define ELD_ABI_VERSION 1
int         eld_abi_version(void);
const char* eld_last_error(void);

/* One context per (process, device).  Holds the SM count, the TMA encode entry point and cached
 * tensor maps.  Thread-compatible: distinct ctx/stream pairs may be used concurrently. */
int  eld_ctx_create(int device, eld_ctx** out);
void eld_ctx_destroy(eld_ctx* ctx);

/* ------------------------------------------------------------------------------------------------
 * Noise formation model.  Replaces NoiseModelBase.__call__ (noise.py:149-170) + the clip in
 * SynDataset.__getitem__ (dataset/sid_dataset.py:277) + RawPacker.pack_raw_bayer (noise.py:10-20),
 * batched over frames, on the GPU.
 *
 * model_mask bits select the terms; the first three are the reference's released baselines
 * (substring match on the model string, noise.py:158-166), the rest are the paper's full model,
 * which the reference does NOT ship (README.md:41, noise.py:173) - "parity unpinned".
 */
#define ELD_NOISE_P  0x01u  /* 'P'  Poisson shot noise:            z = Poisson(x/K)*K        noise.py:158-159 */
#define ELD_NOISE_p  0x02u  /* 'p'  heteroscedastic Gaussian shot: z = x + n*sqrt(max(Kx,1e-10)) noise.py:160-161 */
#define ELD_NOISE_g  0x04u  /* 'g'  Gaussian read noise:           z += n*max(g_scale,1e-10) noise.py:165-166 */
#define ELD_NOISE_G  0x08u  /* Tukey-lambda read noise  z += TL(G_lambda)*G_scale   [paper-restated] */
#define ELD_NOISE_B  0x10u  /* colour bias              z += color_bias[c]          [paper-restated] */
#define ELD_NOISE_R  0x20u  /* row (banding) noise      z += N(0,R_scale) per SENSOR row [paper-restated] */
#define ELD_NOISE_U  0x40u  /* quantisation             z += U(-q/2, q/2)           [paper-restated] */

/* Per-frame scalars = the tuple NoiseModel._sample_params() returns (noise.py:225) extended with
 * the calibrated-but-unused fields of camera_params/release/ *.npy (SURVEY F2).  Units: DN. */
typedef struct eld_noise_params {
    float K;             /* system gain                                  */
    float g_scale;       /* Gaussian read sigma                          */
    float G_scale;       /* Tukey-lambda scale                           */
    float G_lambda;      /* Tukey-lambda shape                           */
    float R_scale;       /* row-noise sigma                              */
    float q_step;        /* quantisation step                            */
    float saturation;    /* 16383-800 = 15583 (noise.py:205)             */
    float ratio;         /* exposure ratio U(100,300) (noise.py:223)     */
    float color_bias[4]; /* per packed channel (R,G1,B,G2)               */
} eld_noise_params;      /* 48 bytes, no padding */

/* Random stream (identical in the CUDA kernel and in oracle/eld_oracle.c):
 *   Philox4x32-10, key = (seed_lo, seed_hi), counter = (a, (domain<<16)|(c<<8)|d, frame_lo, frame_hi)
 *   with frame = frame_id0 + n the GLOBAL frame id - so the synthetic stream does not depend on
 *   how frames are sharded over GPUs.  See DESIGN.md "random stream".  Normals are Box-Muller on 23-bit
 *   uniforms: |n| <= 5.77 (numpy's polar method is unbounded; the truncated tail has probability 8e-9 per draw).
 *
 * clean/noisy: packed float32 [n][4][h][w] (the layout NoiseModelBase.__call__ receives, SURVEY F3).
 * params: HOST pointer to n entries (copied into the launch; no device sync).
 * clip01 != 0 applies min(max(z,0),1) (sid_dataset.py:277).  clean == noisy (in place) is allowed. */
int eld_noise_packed(eld_ctx* ctx, const float* clean, float* noisy, int n, int h, int w,
                     const eld_noise_params* params, uint32_t model_mask,
                     uint64_t seed, uint64_t frame_id0, int clip01, void* stream);

/* Same model fed by the un-packed Bayer mosaic: fuses RawPacker.pack_raw_bayer (noise.py:10-20,
 * plane order RGBG = (0,0),(0,1),(1,1),(1,0)), the LMDB de-quantisation clip(x/65535,0,1)
 * (dataset/lmdb_dataset.py:38-39) and the noise model.  mosaic: [n][H][W], H and W even;
 * in_dtype ELD_DT_U16 or ELD_DT_F32; y = (m-black)/(white-black).  Writes noisy [n][4][H/2][W/2]
 * and, if clean_out != NULL, the packed clean frame (the training target). */
#define ELD_DT_U16 0
#define ELD_DT_F32 1
#define ELD_DT_BF16 2
int eld_noise_mosaic(eld_ctx* ctx, const void* mosaic, int in_dtype, float black, float white,
                     float* noisy, float* clean_out, int n, int H, int W,
                     const eld_noise_params* params, uint32_t model_mask,
                     uint64_t seed, uint64_t frame_id0, int clip01, void* stream);

/* The LMDB wire format as input (util/lmdb_data.py:184-228, dataset/lmdb_dataset.py:24-39): packed uint16
 * [n][4][h][w], y = clip(v * scale, 0, 1) with scale = 1/65535; only 2 bytes per pixel cross PCIe.  Writes noisy
 * and, if clean_out != NULL, the de-quantised clean frame (the training target).  w % 4 == 0. */
int eld_noise_packed_u16(eld_ctx* ctx, const uint16_t* clean_u16, float scale, float* noisy, float* clean_out,
                         int n, int h, int w, const eld_noise_params* params, uint32_t model_mask,
                         uint64_t seed, uint64_t frame_id0, int clip01, void* stream);

/* Noise fused with ELDTrainDataset's augmentation (dataset/sid_dataset.py:340-356): three independent coin flips per
 * frame - flip rows (np.flip axis 1), flip columns (axis 2), transpose (0,2,1) - applied in that order to BOTH the
 * noisy input and the clean target, then the clip.  The noise of a pixel is keyed by its SOURCE position, so
 *   noisy = aug(eld_noise_packed(clean)),  target_out = aug(clean)   bit for bit, in one pass over the frame.
 * aug_flags: HOST array, one byte per frame: bit 0 rows, bit 1 columns, bit 2 transpose (needs h == w).
 * target_out may be NULL.  Not in place.  w % 4 == 0, 16-byte aligned buffers. */
#define ELD_AUG_FLIP_H     1u
#define ELD_AUG_FLIP_W     2u
#define ELD_AUG_TRANSPOSE  4u
int eld_noise_packed_aug(eld_ctx* ctx, const float* clean, float* noisy, float* target_out, int n, int h, int w,
                         const eld_noise_params* params, uint32_t model_mask, uint64_t seed, uint64_t frame_id0,
                         int clip01, const uint8_t* aug_flags, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Per-frame parameters drawn on the GPU, and the noise kernels fed from device tables: the synthesis of a training step
 * with no host work per frame, so that it can be captured in a CUDA graph and replayed on fresh frames.
 *
 * Random stream: the Philox4x32-10 stream above, two more domains (csrc/philox.cuh has the word layout):
 *   domain 4 (parameters), counter frame word = f / burst: the frames of a burst share one tuple, as
 *     NoiseModel.frame_params(burst=k) and SynDataset (dataset/sid_dataset.py:269-275) share one _sample_params();
 *   domain 5 (augmentation flags), counter frame word = f.
 * f = the global frame id: frame_id0 + i, plus *frame_id0_dev when frame_id0_dev != NULL (a device counter, so that a
 * replayed graph draws new frames; see eld_frame_counter_add).
 *
 * The laws are NoiseModel._sample_params' (noise.py:201-225) and, full_model != 0, those of the paper-restated model
 * (eld_b200.noise.NoiseModel._sample_params_full), computed in float64 from 53-bit uniforms and rounded to the float
 * fields at the end:
 *   camera uniform over cameras[0 .. n_cameras);  log K ~ U(ln 0.1, ln 30);  log s = N(0,1) sigma + slope log K + bias
 *   for s = g_scale (and, full model, G_scale and R_scale; Box-Muller normals);  ratio ~ U(100, 300);
 *   saturation 15583;  q_step 1;  full model: one row index uniform over the camera's `rows`, shared by G_lambda =
 *   G_shape[row] and color_bias = color_bias[row].  Fields a model does not draw are 0.
 * The per-frame values differ from the host draws (numpy's RandomState) but follow the same laws. */
#define ELD_MAX_CAMERAS     5
#define ELD_MAX_CALIB_ROWS  18
typedef struct eld_camera_calib {
    double g_slope, g_bias, g_sigma;      /* Profile-1 'g_scale': log g_scale = N(0,1) g_sigma + g_slope log K + g_bias */
    double G_slope, G_bias, G_sigma;      /* Profile-1 'G_scale' (full model)                                           */
    double R_slope, R_bias, R_sigma;      /* Profile-1 'R_scale' (full model)                                           */
    int    rows;                          /* number of G_shape / color_bias rows, 1 .. ELD_MAX_CALIB_ROWS               */
    float  G_shape[ELD_MAX_CALIB_ROWS];   /* Tukey-lambda shapes                                                         */
    float  color_bias[ELD_MAX_CALIB_ROWS][4];
} eld_camera_calib;                       /* 440 bytes */

/* Draws the parameters of frames i = 0 .. n-1 into params_out[i] (DEVICE, n entries) and, if flags_out != NULL, their
 * augmentation flags into flags_out[i] (DEVICE, n bytes: bit 0 rows, 1 columns, 2 transpose, three fair coins, the
 * byte eld_noise_packed_aug takes).  cameras: HOST array of n_cameras entries, copied into the launch.  One launch.
 * ELD_E_ARG, nothing written and nothing launched: a NULL ctx or cameras, n < 0, burst < 1, n_cameras < 1 or > 5, a
 * camera's rows < 1 or > 18, a NULL params_out with n > 0.  n == 0: ELD_OK, nothing launched.
 * The caller's: device buffers of n entries, and a frame_id0_dev that stays valid until the launch has run. */
int eld_noise_sample_params(eld_ctx* ctx, const eld_camera_calib* cameras, int n_cameras, int full_model, uint64_t seed,
                            uint64_t frame_id0, const uint64_t* frame_id0_dev, int burst, int n,
                            eld_noise_params* params_out, uint8_t* flags_out, void* stream);

/* eld_noise_packed (flags_dev == NULL) and eld_noise_packed_aug (flags_dev != NULL) with the parameters and flags read
 * from DEVICE tables of n entries (eld_noise_sample_params writes them) when the kernel runs, and the first frame id
 * frame_id0 (+ *frame_id0_dev if frame_id0_dev != NULL).  Given the same values as host tables, the output is the host
 * entry points' bit for bit; every frame goes in one launch (two past 65535 frames).
 *   flags_dev == NULL: eld_noise_packed's rules (any w, in place allowed); target_out must be NULL.
 *   flags_dev != NULL: eld_noise_packed_aug's rules - h == w (the flags are not seen on the host, so any of them may
 *   transpose), w % 4 == 0, 16-byte aligned buffers, not in place; target_out (may be NULL) receives aug(clean).
 * ELD_E_ARG, nothing written and nothing launched: a NULL ctx, a negative size, unknown model_mask bits, a NULL clean,
 * noisy or params_dev with n, h, w > 0, a plane of 2^32 pixels or more, the rules above.  n, h or w == 0: ELD_OK.
 * The caller's: each table entry needs K, ratio and saturation > 0 (the sampler's entries have them; a hand-written
 * table is not checked), flag bytes below 8, and tables that stay valid until the launch has run. */
int eld_noise_packed_dev(eld_ctx* ctx, const float* clean, float* noisy, float* target_out, int n, int h, int w,
                         const eld_noise_params* params_dev, uint32_t model_mask, uint64_t seed, uint64_t frame_id0,
                         const uint64_t* frame_id0_dev, int clip01, const uint8_t* flags_dev, void* stream);

/* *counter_dev += add on `stream` (one thread): advances the device frame counter of a captured step - the same pattern
 * as the capturable Adam's step counters.  ELD_E_ARG, nothing launched: a NULL ctx or counter_dev. */
int eld_frame_counter_add(eld_ctx* ctx, uint64_t* counter_dev, uint64_t add, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Paired training frames: the per-pixel work of ELDTrainDataset.__getitem__ (dataset/sid_dataset.py:337-356) over
 * LMDBDataset.__getitem__ (dataset/lmdb_dataset.py:28-41), the path of train_real.py:44-58 and of train_syn.py:66-70's
 * offline-noise database, for a batch of n frames in one launch:
 *   input_out[f]  = clip(aug_f(deq(input[f])))      input  [n][cin][h][w],  input_out  f32 [n][cin][h][w]
 *   target_out[f] = aug_f(deq(target[f]))           target [n][cout][h][w], target_out f32 [n][cout][h][w]
 *   deq   ELD_DT_U16: v / 65535 as a correctly rounded float division (lmdb_dataset.py:38-39: the float64 quotient
 *         rounded to float is the same number for every code; the clip to [0, 1] changes nothing);
 *         ELD_DT_F32: identity, NaN and -0.0 included (LMDBDataset does not clip float databases).
 *   aug_f the coin flips of sid_dataset.py:344-352 in their order: bit 0 (ELD_AUG_FLIP_H) flips rows (np.flip axis 1),
 *         bit 1 (ELD_AUG_FLIP_W) columns (axis 2), bit 2 (ELD_AUG_TRANSPOSE) transposes (0, 2, 1); aug_flags is a HOST
 *         array of n bytes copied into the launch (no device sync), NULL for no augmentation.
 *   clip  np.maximum(np.minimum(x, 1), 0) (sid_dataset.py:354): NaN stays NaN, -0.0 becomes +0.0, +Inf 1, -Inf 0.
 * cin, cout: 3 (sRGB databases) or 4 (raw); the two dtypes are independent.  Any element offset; partial tiles masked.
 * ELD_E_ARG, nothing written and nothing launched: a NULL ctx or buffer, a negative size, a channel count other than 3
 * or 4, a dtype other than ELD_DT_U16 / ELD_DT_F32, a flag byte with bits above 2, a transpose flag with h != w, flags
 * for more than 2048 frames (the table the launch carries), either output overlapping either input or the other output.
 * n, h or w == 0: ELD_OK, nothing launched. */
int eld_pair_ingest(eld_ctx* ctx, const void* input, int in_dtype, int cin, const void* target, int tgt_dtype, int cout,
                    float* input_out, float* target_out, int n, int h, int w, const uint8_t* aug_flags, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Raw -> sRGB rendering of the `--stage_in srgb` branch (train_syn.py:55-58): replaces util/process.py:51-68
 * `process` - apply_gains (:15-19), clip, binning RGBG->RGB (:41-48), apply_ccms (:22-31), clip,
 * gamma_compression (:34-39) or camera_response_function (:71-84) with its 8-bit quantisation - and the clips of
 * ISPDataset.__getitem__ (dataset/sid_dataset.py:309,311), as one elementwise kernel.
 *   packed: device f32 [n][4][h][w] (RGBG planes)   rgb: device f32 [n][3][h][w]
 *   wb: HOST [n][4] white-balance gains   ccm: HOST [n][9] cam2rgb, row-major   gamma: 2.2 in the reference
 *   crf_len == 0: gamma curve.  crf_len >= 2: crf_E device [crf_len] (irradiance grid, ascending),
 *   crf_f device [3][crf_len] (per-channel response) - linear interpolation with torchinterp1d's formula.
 * NaN as in the reference: torch.clamp keeps it and `.int()` of NaN is INT_MIN, clamped to 0, so a NaN in any of a pixel's
 * four packed values makes all three of its outputs 0.  The exponent is the float 1/gamma, one ulp off the reference's
 * double 1/2.2 for gamma = 2.2 (an ABI limit: gamma is a float); an 8-bit output can differ by one level where that ulp
 * moves pow() across a level boundary.
 * ELD_E_ARG, nothing written: a negative size, a NULL buffer, gamma <= 0 or NaN, crf_len < 0 or 1, a CRF array NULL,
 * packed and rgb overlapping.  n, h or w == 0: ELD_OK, nothing launched. */
int eld_isp_process(eld_ctx* ctx, const float* packed, float* rgb, int n, int h, int w,
                    const float* wb, const float* ccm, float gamma,
                    const float* crf_E, const float* crf_f, int crf_len, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Metric side of ELDModelBase.eval (models/ELD_model.py:203-243), per frame f of a batch of `n` frames with
 * `per_frame` = C*H*W elements each (f32, any layout, pred and target alike):
 *   correct != 0: IlluminanceCorrect.correct (:156-169): gain = <p,s>/<p,p> over the elements where s != 1,
 *                 p = clamp(pred,0,1); corrected = gain * p (written to `out` if out != NULL)
 *   correct == 0: x = pred; a non-NULL `out` receives pred bit for bit, and gain[f] = 1
 *   psnr[f] = 10 log10(255^2 / mean((clip(255 x,0,255) - clip(255 target,0,255))^2)), x = corrected (or pred):
 *             tensor2im (:23-38, no rounding) + skimage's peak_signal_noise_ratio(data_range = 255) (util/index.py:76-79)
 * NaN as in the reference (torch.clamp, torch.dot and np.clip keep it): a NaN in a frame's prediction, or an empty
 * <p, p> (target 1 everywhere, prediction <= 0 everywhere) makes that frame's gain, corrected output and PSNR NaN;
 * pred == target gives PSNR +inf.
 * scratch: device, n * 4 doubles (zeroed here).  psnr, gain (may be NULL): device f32 [n].  No host synchronisation.
 * ELD_E_ARG, nothing written: a NULL ctx / pred / target / scratch / psnr, n == 0, n > 65535, per_frame == 0, `out`
 * overlapping target, `out` overlapping pred other than out == pred (which is allowed). */
int eld_eval_correct_psnr(eld_ctx* ctx, const float* pred, const float* target, float* out, int n, size_t per_frame,
                          int correct, double* scratch, float* psnr, float* gain, void* stream);

/* The same metric in sRGB: ELDModelBase.eval with --stage_out raw --stage_eval srgb (models/ELD_model.py:226-233), which
 * renders output, target and input with postprocess_bayer_v2 -> raw2rgb_postprocess (util/process.py:116-126) before
 * tensor2im.  Per frame f of n packed frames pred, target and input (device f32 [n][4][h][w], RGBG planes):
 *   x = gain * clamp(pred, 0, 1) with eld_eval_correct_psnr's gain (the same reduction, so the same value) if
 *       correct != 0, else x = pred; written to `out` (device f32 [n][4][h][w]) if out != NULL
 *   R(.) = eld_isp_process's render with wb[f], ccm[f] and gamma 2.2, no CRF: three 8-bit levels / 255 per position
 *   psnr[f]    = 10 log10(255^2 / mean((clip(255 R(x),0,255)   - clip(255 R(target),0,255))^2))
 *   psnr_in[f] = 10 log10(255^2 / mean((clip(255 R(input),0,255) - clip(255 R(target),0,255))^2))   (input != NULL)
 *   gain[f] (may be NULL) as eld_eval_correct_psnr writes it; the means are over the 3 h w rendered values.
 * The renders stay in registers: one pass reads pred, target and input once (48 B per packed pixel position, 16 B
 * more to write `out`, 32 B more for the gain's reduction when correct != 0).
 * NaN as in the reference, and unlike eld_eval_correct_psnr: a NaN in any of a pixel's four packed values renders all
 * three of its sRGB values 0 (eld_isp_process's rule), so a NaN prediction or a NaN gain (an empty correction mask)
 * still gives a finite PSNR, as process + tensor2im do; gain[f] is then NaN.  Equal renders give PSNR +inf.
 * wb: HOST [n][4], ccm: HOST [n][9] cam2rgb row-major (as eld_isp_process).  scratch: device, n * 4 doubles (zeroed
 * here).  psnr, psnr_in: device f32 [n].  Launches: the gain's reduction (correct != 0), one render pass per 48 frames,
 * one finalise.  No host synchronisation, no allocation.
 * ELD_E_ARG, nothing written: a NULL ctx / pred / target / wb / ccm / scratch / psnr, input and psnr_in not both given or
 * both NULL, n == 0 or n > 65535, h <= 0 or w <= 0, pred / target / input overlapping an output (out == pred is allowed),
 * two outputs overlapping. */
int eld_eval_srgb_psnr(eld_ctx* ctx, const float* pred, const float* target, const float* input, float* out,
                       int n, int h, int w, const float* wb, const float* ccm, int correct, double* scratch,
                       float* psnr, float* psnr_in, float* gain, void* stream);

/* SSIM, the other half of quality_assess (util/index.py:80): skimage's structural_similarity(Y, X, data_range=255,
 * multichannel=True) with its defaults, on the tensor2im images of frame f (Y the target, X the estimate):
 *   x = gain[f] * clamp(pred, 0, 1) if gain != NULL (device f32 [n]: the gain eld_eval_correct_psnr or
 *       eld_eval_srgb_psnr wrote, so the same value), else x = pred
 *   raw stage (wb == ccm == NULL): the c planes of x and target (c = 3 or 4), each clip(255 v, 0, 255) in f32;
 *   sRGB stage (wb, ccm both given, c = 4): eld_eval_srgb_psnr's render R(.) first (gamma 2.2, no CRF; a NaN pixel
 *       renders 0), three channels clip(255 R, 0, 255)
 *   per channel, in float64: the 7 x 7 uniform-window means ux, uy, uxx, uyy, uxy, cov_norm = 49/48,
 *   vx = cov_norm (uxx - ux^2), vy likewise, vxy = cov_norm (uxy - ux uy), C1 = (0.01 * 255)^2, C2 = (0.03 * 255)^2,
 *   S = (2 ux uy + C1)(2 vxy + C2) / ((ux^2 + uy^2 + C1)(vx + vy + C2)) at every window inside the frame (the map
 *   without its 3-pixel border); ssim[f] = the mean of S over those (h - 6)(w - 6) positions and the channels
 *   ssim_in[f] the same for input against target (input != NULL).
 * NaN: in the raw stage a NaN anywhere in a frame's x or target (a NaN gain included) makes ssim[f] NaN; in the sRGB
 * stage it renders black, and ssim[f] stays finite.  Equal images give exactly 1.
 * ssim, ssim_in: device f64 [n].  scratch: device, at least eld_eval_ssim_scratch_bytes(n, h, w) bytes, one slot per
 * map tile of 32 x 16 positions, each written by one CTA and summed in a fixed order: two calls give the same bits.
 * wb: HOST [n][4], ccm: HOST [n][9] (as eld_eval_srgb_psnr).  Launches: one stencil pass (one per 48 frames in the sRGB
 * stage), one finalise.  No host synchronisation, no allocation.
 * ELD_E_ARG, nothing written and nothing launched: a NULL ctx / pred / target / scratch / ssim, input and ssim_in not
 * both given or both NULL, wb and ccm not both given or both NULL, n < 1 or n > 65535, c other than 3 or 4 (other than 4
 * in the sRGB stage), h < 7 or w < 7 (skimage raises ValueError), scratch_bytes short, scratch / ssim / ssim_in
 * overlapping pred, target, input, gain or each other. */
size_t eld_eval_ssim_scratch_bytes(int n, int h, int w);     /* 0 for n, h, w eld_eval_ssim refuses */
int eld_eval_ssim(eld_ctx* ctx, const float* pred, const float* target, const float* input, int n, int c, int h, int w,
                  const float* gain, const float* wb, const float* ccm, double* scratch, size_t scratch_bytes,
                  double* ssim, double* ssim_in, void* stream);

/* Number of kernels the library has launched through this ctx since creation (bench.py's
 * gpu_launches evidence). */
int64_t eld_launch_count(const eld_ctx* ctx);

/* ------------------------------------------------------------------------------------------------
 * U-Net (UNetSeeInDark, models/arch/Unet.py:6-91) training step on NHWC bf16 activations with fp32
 * master weights.  Declared in eld_b200_unet.h (included below) to keep this file readable.
 */
#include "eld_b200_unet.h"

#ifdef __cplusplus
}
#endif
#endif /* ELD_B200_H */
