/* fear_b200.h -- C ABI of libfear_b200.so: the H100-native (sm_90a) FEAR-XS per-frame
 * inference hot path (backbone -> pixel-wise correlation -> cls/reg heads -> box decode).
 *
 * The reference (PinataFarms/FEARTracker) is pure Python/PyTorch and has no FFI; these entry
 * points are what a binding for its hot path replaces (file:line relative to the reference):
 *
 *   fear_get_features     FEARNet.get_features            model_training/model/fear_net.py:63-66
 *                         (= Encoder stages 0..17 + AdjustLayer, blocks.py:8-42,75-88)
 *   fear_backbone         FEARNet.feature_extractor       model_training/model/fear_net.py:58-61
 *   fear_head             FEARNet.connector / BoxTower.forward  fear_net.py:76-81, blocks.py:174-194
 *   fear_track            FEARNet.track (+ FEARTracker._postprocess / FEARBoxCoder.decode)
 *                         fear_net.py:90-96, tracker/fear_tracker.py:74-86, dataset/box_coder.py:75-107
 *   fear_forward          FEARNet.forward((template, search))   fear_net.py:83-88
 *   fear_corr_concat_f32  MobileCorrelation.forward front half (matmul + cat)  blocks.py:121-124
 *   fear_corr_nhwc_f32    same contraction on the library's internal channels-last layout
 *   fear_decode           FEARBoxCoder.decode                 dataset/box_coder.py:75-107
 *   fear_decode_smooth    FEARTracker._postprocess with smooth: true (penalty, window, size smoothing)
 *                         tracker/base_tracker.py:126-205
 *   fear_track_sized / fear_track_sized_u8 / fear_forward_sized / fear_head_sized / fear_decode_sized /
 *   fear_decode_smooth_sized   the same on search crops of side S (instance_size; score_size = S / 16)
 *   fear_pack_weights     load_from_lighting + nn.Module.load_state_dict  utils/torch.py:11-24
 *
 *   fear_head_update      BoxTower.forward(search, kernel, update)   blocks.py:174-179
 *   fear_crop_resize_u8   get_extended_crop (crop + pad + resize)    model_training/utils/utils.py:215-253
 *   fear_crop_targets_u8  get_extended_crop for N tracked targets (context box + resize tables on the device)
 *   fear_advance_targets  FEARTracker.update's rescale + clamp of the decoded box, for N targets
 *                         tracker/fear_tracker.py:63-64, base_tracker.py:83-90
 *   fear_crop_targets_view_u8 / fear_advance_targets_view   the same on frames located by FearFrameView (strided,
 *                         anywhere in device memory)
 *   fear_frame_sums_u8    np.mean(frame, axis=(0, 1)) of get_extended_crop's padding, as exact integer sums
 *   fear_crop_targets_yuv420_u8 / fear_advance_targets_yuv420 / fear_frame_sums_yuv420_u8   the same three on YUV 4:2:0
 *                         frames (NV12, I420) located by FearFrameYUV420, each pixel converted to RGB exactly as
 *                         cv2.cvtColor(COLOR_YUV2RGB_NV12 / COLOR_YUV2RGB_I420) converts it
 *   fear_crop_targets_yuv_u8 / fear_advance_targets_yuv / fear_frame_sums_yuv_u8   the same three on YUV 4:2:0 frames
 *                         located by FearFrameYUV, which also names the colour format: BT.601 / BT.709 / BT.2020
 *                         matrix, limited or full range, 8-bit or 10 / 12-bit samples in uint16 (P010, P016,
 *                         yuv420p10le)
 *   fear_crop_targets_ycbcr_u8 / fear_advance_targets_ycbcr / fear_frame_sums_ycbcr_u8   the same three on YUV 4:2:0,
 *                         4:2:2 and 4:4:4 frames located by FearFrameYCbCr (YUYV / UYVY / Y210, NV16 / P210,
 *                         yuv422p, yuv444p, NVDEC's YUV444 surfaces), in every FearFrameYUV colour format
 *   fear_crop_targets_ycbcr_v210_u8 / fear_advance_targets_ycbcr_v210 / fear_frame_sums_ycbcr_v210_u8   the same three
 *                         on FearFrameYCbCrV210 tables: FearFrameYCbCr entries and v210 surfaces (10-bit 4:2:2 packed
 *                         three codes to a 32-bit word, as SDI capture cards deliver it), unpacked inside the crop
 *   fear_crop_targets_ycbcr_hdr_u8 / fear_advance_targets_ycbcr_hdr / fear_frame_sums_ycbcr_hdr_u8   the same three on
 *                         FearFrameYCbCrHDR tables: those entries with a transfer function, PQ and HLG video
 *                         tone-mapped to SDR BT.709 (BT.2446-1 Method A) inside the crop
 *   fear_crop_targets_bayer_u8 / fear_advance_targets_bayer / fear_frame_sums_bayer_u8   the same three on raw Bayer
 *                         mosaics located by FearFrameBayer (8 to 16 bits, MIPI RAW10 / RAW12), demosaiced inside the
 *                         crop as cv2.cvtColor(COLOR_Bayer*2RGB) demosaics them
 *   fear_frame_range_mono  per-frame code range (min, max) of single-channel frames located by FearFrameMono, written
 *                         into the table for their min-max gain control (thermal cores, mono cameras)
 *   fear_crop_targets_mono_u8 / fear_advance_targets_mono / fear_frame_sums_mono_u8   the same three on FearFrameMono
 *                         tables (8 to 16 bits, MIPI RAW10 / RAW12), each tap mapped to grey (g, g, g) inside the crop
 *   fear_crop_targets_rgb_u8 / fear_advance_targets_rgb / fear_frame_sums_rgb_u8   the same three on RGB frames in any
 *                         channel order located by FearFrameRGB (BGR / BGRA / ABGR, x2rgb10, rgb48 / rgba64, planar
 *                         gbrp at 8 to 16 bits), each tap's channels read and mapped to 8 bits inside the crop
 *   fear_crop_targets_oriented_u8 / fear_advance_targets_oriented   the crop and advance of any of the eight tables
 *                         above on rotated and mirrored frames (90-degree turns, left-right flip), oriented inside
 *                         the crop
 *   fear_gather_targets / fear_scatter_targets   the selected targets' rows and templates into compact step buffers,
 *                         and their new boxes back, for a step over the targets of some streams only
 *
 * Conventions: every pointer named d_* is a DEVICE pointer owned by the caller (torch keeps
 * ownership); tensors are dense fp32 in the reference's NCHW layout unless stated; `stream`
 * is a cudaStream_t passed as void*.  Hot-path calls are asynchronous on `stream`, never synchronise
 * it and never allocate (workspace is reserved up front by fear_reserve -- the only call besides
 * fear_pack_weights / fear_free that allocates or synchronises; a batch larger than the reservation is
 * processed in chunks; fear_corr_concat_ws_f32 takes its scratch from the caller).  Return 0 on success,
 * a positive cudaError_t or a negative FEAR_E* code otherwise; fear_last_error() gives the message
 * (thread-local).  Handles are not thread-safe: one handle per host thread / stream.  A handle belongs to the
 * device that was current when it was packed; every entry point selects that device for its own duration and
 * restores the caller's current device (several devices per process are fine: call fear_init for each).
 */
#ifndef FEAR_B200_H
#define FEAR_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FEAR_ABI_VERSION 1

#define FEAR_EINVAL (-1)    /* bad argument (shape, null pointer, alignment)            */
#define FEAR_ESTATE (-2)    /* handle not initialised / weights not packed              */
#define FEAR_ENOMEM (-3)    /* workspace reservation failed                             */
#define FEAR_ENODEV (-4)    /* no sm_90 device                                          */

#define FEAR_FEAT_CH 256        /* AdjustLayer output channels                          */
#define FEAR_SCORE 16           /* score map side (256 / 16)                            */
#define FEAR_TMPL 8             /* template feature side (128 / 16)                     */
#define FEAR_CORR_CH 64         /* FEAR_TMPL^2 correlation channels                     */

/* One decoded frame (FEARBoxCoder.decode semantics: xywh in float64 like the reference,
 * which promotes to double through its float64 grid; (row, col) = unravel(argmax)). */
typedef struct FearBox {
  double x, y, w, h;
  float score;      /* sigmoid(cls)[row, col]                                           */
  int32_t row, col; /* argmax of sigmoid(cls), first maximum in row-major order         */
  int32_t flat;     /* row * 16 + col                                                   */
} FearBox;

/* Multi-target tracking loop (fear_crop_targets_u8 / fear_advance_targets).  Frames are HxWx3 uint8 RGB images packed
 * into one device buffer; a frame table lists them.  Each target's tracking state lives in device memory, so a
 * captured CUDA graph steps every target with the values of the current frame. */
typedef struct FearFrame {
  int64_t offset; /* byte offset of an HxWx3 uint8 frame in the packed buffer                */
  int32_t H, W;
} FearFrame;
/* A frame wherever it lives in device memory (FEARMultiTracker's frames, packed or the caller's own tensors): 40 bytes.
 * Pixel (y, x) channel c (R, G, B) is data[y * row_stride + x * pixel_stride + c * channel_stride]; strides in bytes,
 * >= 0.  A packed HxWx3 frame at byte `offset` of a buffer is {base + offset, 3W, 3, 1, H, W}; an RGB view of an RGBA
 * surface has pixel_stride 4, a CHW tensor seen as HWC has (W, 1, H * W).  An entry with data == NULL, H < 1 or W < 1
 * is treated like a frame index outside [0, F). */
typedef struct FearFrameView {
  const uint8_t* data;                              /* device address of pixel (0, 0), channel R        */
  int64_t row_stride, pixel_stride, channel_stride; /* bytes, >= 0                                       */
  int32_t H, W;
} FearFrameView;
/* A YUV 4:2:0 frame (8-bit BT.601 limited range, as a video decoder writes it) wherever it lives in device memory:
 * 64 bytes.  Luma of pixel (y, x) is y[y * y_row_stride + x * y_pixel_stride]; its chroma is sample (y / 2, x / 2) of
 * u (Cb) and v (Cr), at u[(y / 2) * uv_row_stride + (x / 2) * uv_pixel_stride] and likewise in v.  Strides in bytes,
 * >= 0; H, W is the luma size.  NV12 with row pitch P at address b is {b, b + H*P, b + H*P + 1, P, 1, P, 2, H, W};
 * packed I420 is {b, b + H*W, b + H*W + H*W/4, W, 1, W/2, 1, H, W}; separate planes and even-offset regions of interest
 * are the same record with other addresses.  The kernels read the frame as the RGB image
 * cv2.cvtColor(frame, COLOR_YUV2RGB_NV12 / COLOR_YUV2RGB_I420) gives, bit for bit (OpenCV 4.x's fixed-point conversion,
 * nearest chroma).  An entry with a null plane, H < 1, W < 1, or an odd H or W is treated like a frame index outside
 * [0, F). */
typedef struct FearFrameYUV420 {
  const uint8_t *y, *u, *v;                /* device addresses of luma sample (0, 0), Cb and Cr samples (0, 0) */
  int64_t y_row_stride, y_pixel_stride;    /* bytes, >= 0                                                      */
  int64_t uv_row_stride, uv_pixel_stride;  /* bytes, >= 0, shared by u and v                                   */
  int32_t H, W;                            /* luma size, both even                                             */
} FearFrameYUV420;
/* A YUV 4:2:0 frame of any of the formats below: 80 bytes.  The planes are addressed as in FearFrameYUV420, with byte
 * strides; a sample is one byte when bits == 8 and a little-endian uint16 when bits is 10 or 12, whose code is
 * (sample >> shift) & (2^bits - 1): shift 16 - bits for MSB-aligned samples (NVDEC's P010 / P016), 0 for LSB-aligned
 * ones (ffmpeg's yuv420p10le / yuv420p12le).  NV12-layout P010 with row pitch P bytes at address b is
 * {b, b + H*P, b + H*P + 2, P, 2, P, 4, H, W, matrix, full_range, 10, 6}.
 *
 * (matrix FEAR_YUV_BT601, full_range 0, bits 8) is converted exactly as FearFrameYUV420 is (cv2.cvtColor, OpenCV's
 * fixed point).  Every other format uses the inverse equations of ITU-T H.273 in float64, each step rounded on its own
 * (no FMA), with Kr, Kb = 0.299, 0.114 (BT.601), 0.2126, 0.0722 (BT.709), 0.2627, 0.0593 (BT.2020 non-constant
 * luminance), m = 2^(bits - 8):
 *   limited: yn = (Y - 16m) * (1 / (219m));  pb = (U - 128m) * (1 / (224m));  pr = (V - 128m) * (1 / (224m))
 *   full:    yn = Y * (1 / (2^bits - 1));  pb = (U - 2^(bits-1)) * (1 / (2^bits - 1));  pr likewise
 *   Kg = (1 - Kr) - Kb;  cR = 2 * (1 - Kr);  cB = 2 * (1 - Kb);  gB = 2 * Kb * (1 - Kb) / Kg;  gR = 2 * Kr * (1 - Kr) / Kg
 *   R = yn + cR * pr;  G = (yn - gB * pb) - gR * pr;  B = yn + cB * pb;  out = min(max(rint(255 * v), 0), 255)
 * evaluated left to right, rint rounding half to even.  Codes outside the nominal range are not clamped; only the 8-bit
 * result saturates.  Chroma is nearest (sample (y / 2, x / 2)).  Transfer functions (PQ, HLG) are not applied.
 *
 * An entry is treated like a frame index outside [0, F) when it has a null plane, H < 1, W < 1, an odd H or W, a matrix
 * other than the three below, full_range other than 0 or 1, bits not 8, 10 or 12, a shift other than 0 at 8 bits or
 * outside [0, 16 - bits] at 10 / 12 bits, or, at 10 / 12 bits, an odd plane address or an odd stride. */
#define FEAR_YUV_BT601 0
#define FEAR_YUV_BT709 1
#define FEAR_YUV_BT2020 2
typedef struct FearFrameYUV {              /* 80 bytes                                                          */
  const void *y, *u, *v;                   /* device addresses of luma (0, 0), Cb (0, 0), Cr (0, 0)             */
  int64_t y_row_stride, y_pixel_stride;    /* bytes, >= 0                                                       */
  int64_t uv_row_stride, uv_pixel_stride;  /* bytes, >= 0, shared by u and v                                    */
  int32_t H, W;                            /* luma size, both even                                              */
  int32_t matrix, full_range, bits, shift; /* bits 8: uint8 samples, shift 0; bits 10/12: uint16, 0 <= shift <= 16-bits */
} FearFrameYUV;
/* A YUV frame of any chroma subsampling: 88 bytes, the fields of FearFrameYUV (same meaning, same formats) followed by
 * the chroma shifts.  The chroma of pixel (y, x) is sample (y >> chroma_shift_y, x >> chroma_shift_x) of u and v.
 * (chroma_shift_x, chroma_shift_y) is (1, 1) for 4:2:0, (1, 0) for 4:2:2 and (0, 0) for 4:4:4; W must be even when
 * chroma_shift_x is 1 and H when chroma_shift_y is 1, so 4:2:2 may have an odd H and 4:4:4 any size.  For a surface
 * with row pitch P bytes at address b (fields in order; "..." is H, W, matrix, full_range, bits, shift):
 *   YUYV (YUY2)             {b, b + 1, b + 3, P, 2, P, 4, ..., 1, 0}
 *   UYVY                    {b + 1, b, b + 2, P, 2, P, 4, ..., 1, 0}
 *   YVYU                    {b, b + 3, b + 1, P, 2, P, 4, ..., 1, 0}
 *   Y210 / Y212 / Y216      {b, b + 2, b + 6, P, 4, P, 8, H, W, matrix, full_range, 10 (12), 6 (4), 1, 0}
 *                           (YUYV order in uint16, MSB-aligned)
 *   NV16 / P210             {b, b + H*P, b + H*P + 1 (P210: + 2), P, 1 (2), P, 2 (4), ..., 1, 0}
 *   I422 (yuv422p)          {b, b + H*W, b + H*W + H*W/2, W, 1, W/2, 1, ..., 1, 0} (uint16 samples: offsets and
 *                           strides x2)
 *   I444 / NVDEC YUV444     {b, b + H*P, b + 2*H*P, P, 1, P, 1, ..., 0, 0} (16-bit surfaces: P, 2, P, 2, shift
 *                           16 - bits)
 *   4:2:0                   the FearFrameYUV record, then 1, 1
 * An entry is treated like a frame index outside [0, F) when FearFrameYUV's rules refuse it (read with these shifts:
 * an odd H only matters when chroma_shift_y is 1, an odd W when chroma_shift_x is 1), or when the shift pair is not one
 * of the three above (4:4:0 is refused). */
typedef struct FearFrameYCbCr {            /* 88 bytes                                                          */
  const void *y, *u, *v;                   /* device addresses of luma (0, 0), Cb (0, 0), Cr (0, 0)             */
  int64_t y_row_stride, y_pixel_stride;    /* bytes, >= 0                                                       */
  int64_t uv_row_stride, uv_pixel_stride;  /* bytes, >= 0, shared by u and v                                    */
  int32_t H, W;                            /* luma size                                                         */
  int32_t matrix, full_range, bits, shift; /* as in FearFrameYUV                                                */
  int32_t chroma_shift_x, chroma_shift_y;  /* (1, 1) 4:2:0, (1, 0) 4:2:2, (0, 0) 4:4:4                          */
} FearFrameYCbCr;
/* A FearFrameYCbCr or a v210 surface: 96 bytes, the fields of FearFrameYCbCr followed by `v210` and a reserved int32.
 * With v210 == 0 the entry is read exactly as a FearFrameYCbCr, so v210 surfaces can share a table with every other YUV
 * frame.  With v210 == 1 the entry is a v210 surface (10-bit 4:2:2 as SDI capture cards and ffmpeg's v210 codec write
 * it): y is the address of row 0's first word, y_row_stride the row pitch in bytes; bits must be 10 and the chroma
 * shifts (1, 0); matrix and full_range are read as in FearFrameYUV; u, v, y_pixel_stride, the uv strides and shift are
 * not read.  A row is a run of 16-byte groups of four little-endian 32-bit words, each holding three 10-bit codes at
 * bits 0-9, 10-19 and 20-29 (bits 30-31 are ignored).  Group g holds pixels 6g .. 6g + 5 and chroma pairs 3g .. 3g + 2:
 *   w0 = Cb0 | Y0 << 10 | Cr0 << 20     w1 = Y1 | Cb1 << 10 | Y2 << 20
 *   w2 = Cr1 | Y3 << 10 | Cb2 << 20     w3 = Y4 | Cr2 << 10 | Y5 << 20
 * Pixel x takes chroma pair x / 2 (co-sited, nearest).  W must be even, H >= 1; a row needs 16 * ceil(W / 6) bytes, and
 * capture cards and ffmpeg pitch rows to 128 * ceil(W / 48).  A W x H v210 surface with row pitch P at address b is
 *   {b, 0, 0, P, 0, 0, 0, H, W, matrix, full_range, 10, 0, 1, 0, 1, 0}
 * and converts exactly as FearFrameYUV's H.273 inverse at 10 bits does on the unpacked codes.  A v210 entry is treated
 * like a frame index outside [0, F) when y is null or not 4-byte aligned, the pitch is not a multiple of 4 or below
 * 16 * ceil(W / 6), W is odd or < 2, H < 1, bits is not 10, the shifts are not (1, 0), or matrix / full_range is not one
 * FearFrameYUV allows; any v210 value other than 0 and 1 is too. */
typedef struct FearFrameYCbCrV210 {        /* 96 bytes                                                          */
  const void *y, *u, *v;                   /* device addresses (v210: y only, row 0's first word)               */
  int64_t y_row_stride, y_pixel_stride;    /* bytes (v210: the row pitch, a multiple of 4; the pixel stride is   */
  int64_t uv_row_stride, uv_pixel_stride;  /* not read, nor are the uv strides)                                  */
  int32_t H, W;                            /* luma size                                                         */
  int32_t matrix, full_range, bits, shift; /* as in FearFrameYUV (v210: bits 10, shift not read)                */
  int32_t chroma_shift_x, chroma_shift_y;  /* as in FearFrameYCbCr (v210: 1, 0)                                 */
  int32_t v210;                            /* 0: a FearFrameYCbCr entry; 1: a v210 surface                      */
  int32_t reserved;                        /* not read                                                          */
} FearFrameYCbCrV210;
/* A FearFrameYCbCrV210 entry with its transfer characteristics, so HDR video (PQ and HLG, as phones, UHD broadcast and
 * NVDEC's P010 / P210 surfaces deliver it) is tone-mapped to SDR inside the crop: 104 bytes, the fields of
 * FearFrameYCbCrV210 followed by `transfer` and a reserved int32.  `transfer` holds the ITU-T H.273
 * TransferCharacteristics code (ffmpeg's color_trc, NVDEC's transfer_characteristics):
 *   0                     the matrix only: the entry is read exactly as the *_ycbcr_v210 entry points read its
 *                         FearFrameYCbCrV210 fields (a planar entry or a v210 surface, SDR)
 *   FEAR_TRC_PQ (16)      SMPTE ST 2084 / BT.2100 PQ
 *   FEAR_TRC_HLG (18)     BT.2100 HLG
 * A PQ or HLG entry reads its codes as the FearFrameYCbCrV210 entry does, takes the unclamped R'G'B' of FearFrameYUV's
 * H.273 inverse (before the rounding to 8 bits), and continues in float64, each step rounded on its own (no FMA):
 *   1. E' = clamp(R'G'B', 0, 1)
 *   2. display light Fd in cd/m2 per component, BT.2020 primaries:
 *        PQ:  p = E'^(1/m2);  Fd = 10000 * (max(p - c1, 0) / (c2 - c3 * p))^(1/m1)   (m1 = 2610/16384,
 *             m2 = 2523/4096 * 128, c1 = 3424/4096, c2 = 2413/4096 * 32, c3 = 2392/4096 * 32)
 *        HLG: E = E'^2 / 3 for E' <= 1/2, else (exp((E' - c) / a) + b) / 12  (a = 0.17883277, b = 1 - 4a,
 *             c = 0.5 - a ln(4a));  Ys = 0.2627 E_R + 0.6780 E_G + 0.0593 E_B;  Fd = 1000 * Ys^0.2 * E  (Lw 1000,
 *             Lb 0, system gamma 1.2)
 *   3. L = min(Fd / 1000, 1): a fixed 1000 cd/m2 peak, PQ light above it clips
 *   4. ITU-R BT.2446-1 Method A (L_HDR 1000, L_SDR 100): R'G'B' = L^(1/2.4); Y' = 0.2627 R' + 0.6780 G' + 0.0593 B';
 *      Y'p = ln(1 + (rho_HDR - 1) Y') / ln(rho_HDR), rho_HDR = 1 + 32 (1000/10000)^(1/2.4);
 *      Y'c = 1.077 Y'p (Y'p <= 0.7399), -1.1510 Y'p^2 + 2.7811 Y'p - 0.6302 (Y'p < 0.9909), 0.5 Y'p + 0.5 (otherwise);
 *      Y'sdr = (rho_SDR^Y'c - 1) / (rho_SDR - 1), rho_SDR = 1 + 32 (100/10000)^(1/2.4);  f = Y'sdr / (1.1 Y') (0 when
 *      Y' = 0);  Cb = f (B' - Y') / 1.8814;  Cr = f (R' - Y') / 1.4746;  Y'tmo = Y'sdr - max(0.1 Cr, 0)
 *   5. R' = Y'tmo + 1.4746 Cr, B' = Y'tmo + 1.8814 Cb, G' = (Y'tmo - 0.2627 R' - 0.0593 B') / 0.6780; clamp to [0, 1],
 *      ^2.4; the linear BT.2020 -> BT.709 matrix (from the primaries and D65; BT.2087's to 4 digits); clamp to [0, 1],
 *      ^(1/2.4); out = min(max(rint(255 v), 0), 255)
 * evaluated left to right, exp, log and pow from the CUDA double library (within 2 ulp; every step is continuous but
 * for a 5.5e-4 step of Method A's 4-digit coefficients at 0.7399, so a difference from another libm can in practice
 * only move an output across a rounding boundary).  The derived constants
 * (1/m1, 1/m2, b, c, 1/2.4, rho_HDR - 1, ln rho_HDR, rho_SDR, rho_SDR - 1 and the matrix) are folded to the float64
 * values feartracker_b200.image_ops.HDR_CONSTANTS and bt2020_to_bt709_matrix() name, which restate the chain in numpy.
 * There is no peak or metadata parameter (HDR10 MaxCLL, HDR10+ and Dolby Vision are not read).
 * An entry is treated like a frame index outside [0, F) when FearFrameYCbCrV210 refuses it, when transfer is not 0,
 * 16 or 18, or when transfer is 16 or 18 and the matrix is not FEAR_YUV_BT2020 or bits is 8. */
#define FEAR_TRC_PQ 16
#define FEAR_TRC_HLG 18
typedef struct FearFrameYCbCrHDR {         /* 104 bytes                                                         */
  const void *y, *u, *v;                   /* as in FearFrameYCbCrV210                                          */
  int64_t y_row_stride, y_pixel_stride;
  int64_t uv_row_stride, uv_pixel_stride;
  int32_t H, W;
  int32_t matrix, full_range, bits, shift;
  int32_t chroma_shift_x, chroma_shift_y;
  int32_t v210;                            /* 0: planar; 1: a v210 surface                                      */
  int32_t reserved;                        /* not read                                                          */
  int32_t transfer;                        /* H.273 TransferCharacteristics: 0, FEAR_TRC_PQ or FEAR_TRC_HLG      */
  int32_t reserved_hdr;                    /* not read                                                          */
} FearFrameYCbCrHDR;
/* A raw Bayer mosaic (machine-vision cameras' PFNC BayerRG8 / BayerGR12 ..., CSI-2 sensors' SRGGB10P / SRGGB12P):
 * 40 bytes.  `pattern` names the colours of the 2 x 2 block at pixel (0, 0), row by row (OpenCV 4.x's sensor-order
 * COLOR_Bayer{RGGB,GRBG,GBRG,BGGR}2RGB).  `packing` is how a row holds its samples:
 *   FEAR_BAYER_UNPACKED  one sample per pixel: a byte at 8 bits (shift 0), a uint16 at 10, 12, 14 or 16 bits whose code
 *                        is (s >> shift) & (2^bits - 1), 0 <= shift <= 16 - bits (LSB-aligned: 0, MSB: 16 - bits); a
 *                        uint16 row needs an even address and an even row_stride
 *   FEAR_BAYER_RAW10     MIPI CSI-2 RAW10 (bits 10): 4 pixels in 5 bytes, bytes 0-3 bits 9..2 of P0..P3, byte 4
 *                        P3[1:0] << 6 | P2[1:0] << 4 | P1[1:0] << 2 | P0[1:0]; a row needs 5 * ceil(W / 4) bytes
 *   FEAR_BAYER_RAW12     MIPI CSI-2 RAW12 (bits 12): 2 pixels in 3 bytes, bytes 0-1 bits 11..4 of P0, P1, byte 2
 *                        P1[3:0] << 4 | P0[3:0]; a row needs 3 * ceil(W / 2) bytes
 * `data` is sample (0, 0) (packed: the first byte of row 0) and row_stride the row pitch in bytes (shift is not read for
 * packed rows).  Every pixel is demosaiced as cv2.cvtColor(raw, COLOR_Bayer{pattern}2RGB) does (bilinear, integer): with
 * (y, x) clamped into [1, H - 2] x [1, W - 2], the pixel's own colour is its code, and with N, S, W, E the codes next to
 * it and NW, NE, SW, SE the diagonal ones, cross = (N + S + W + E + 2) >> 2, diag = (NW + NE + SW + SE + 2) >> 2,
 * hor = (W + E + 1) >> 1, ver = (N + S + 1) >> 1: an R site takes G = cross, B = diag; a B site G = cross, R = diag; a G
 * site on an R row R = hor, B = ver; a G site on a B row B = hor, R = ver.  Above 8 bits each channel value v is mapped
 * to 8 bits as FearFrameYUV's full-range luma is: min(max(rint(255 * (v * (1 / (2^bits - 1)))), 0), 255) in float64.
 * An entry is treated like a frame index outside [0, F) when data is null, H or W is below 3 (cv2 accepts smaller
 * frames; the kernels do not), pattern is not 0..3, packing is not 0..2, an unpacked entry has bits not in {8, 10, 12, 14,
 * 16}, a shift other than 0 at 8 bits, a negative shift or shift + bits > 16, or (uint16) an odd address or row_stride,
 * a RAW10 entry has bits other than 10 or a RAW12 entry bits other than 12, or row_stride is below the bytes of a row. */
#define FEAR_BAYER_RGGB 0
#define FEAR_BAYER_GRBG 1
#define FEAR_BAYER_GBRG 2
#define FEAR_BAYER_BGGR 3
#define FEAR_BAYER_UNPACKED 0
#define FEAR_BAYER_RAW10 1
#define FEAR_BAYER_RAW12 2
typedef struct FearFrameBayer {               /* 40 bytes                                                       */
  const void* data;                           /* device address of sample (0, 0) / of row 0's first byte        */
  int64_t row_stride;                         /* bytes                                                          */
  int32_t H, W;                               /* size in pixels, both >= 3                                      */
  int32_t pattern, bits, shift, packing;      /* FEAR_BAYER_*, code depth, uint16 alignment, FEAR_BAYER_* packing */
} FearFrameBayer;
/* A single-channel frame (machine-vision cameras' PFNC Mono8 / Mono10 / Mono12 / Mono16, CSI-2 mono sensors' GREY /
 * Y10 / Y12 / Y16 / Y10P / Y12P, thermal cores' 14- or 16-bit Y16): 48 bytes.  data, row_stride, bits, shift and
 * packing are FearFrameBayer's, read the same way (FEAR_BAYER_UNPACKED, FEAR_BAYER_RAW10, FEAR_BAYER_RAW12).  Pixel
 * (y, x) is the grey triple (g, g, g) of its code v:
 *   agc 0                without gain control: g = v at 8 bits; above 8 bits v is mapped as FearFrameBayer maps a
 *                        channel, min(max(rint(255 * (v * (1 / (2^bits - 1)))), 0), 255) in float64
 *   agc FEAR_AGC_MINMAX  min-max gain control over the whole frame, cv2.normalize(codes, None, 0, 255, NORM_MINMAX,
 *                        CV_8U) of the frame's codes: with lo, hi its smallest and largest code,
 *                        scale = 255 * (hi - lo > DBL_EPSILON ? 1 / (hi - lo) : 0) and shift = 0 - lo * scale in
 *                        float64, each operation rounded; then a = (float)scale, b = (float)shift and
 *                        g = min(max(rint(fmaf((float)v, a, b)), 0), 255), the multiply-add rounded once.  A constant
 *                        frame (hi == lo) is 0 everywhere, as in cv2.  lo and hi are read from the record, where
 *                        fear_frame_range_mono writes them: the record's writer sets lo = INT32_MAX and
 *                        hi = INT32_MIN (an empty range, which maps every code to 0) and the range kernel lowers and
 *                        raises them atomically to the frame's range, so a captured graph that rewrites the table
 *                        before the range kernel sees each frame's own range.
 * An entry is treated like a frame index outside [0, F) when data is null, H or W is below 1, the bits, shift or
 * packing break FearFrameBayer's rules (bits in {8, 10, 12, 14, 16} unpacked with 0 <= shift <= 16 - bits and shift 0
 * at 8 bits; 10 for RAW10, 12 for RAW12; packing 0..2), agc is neither 0 nor FEAR_AGC_MINMAX, an unpacked uint16 entry
 * has an odd address or row_stride, or row_stride is below the bytes of a row (W, 2 W, 5 * ceil(W / 4) or
 * 3 * ceil(W / 2)).  Unlike FearFrameBayer there is no neighbourhood, so 1 x 1 frames are read. */
#define FEAR_AGC_MINMAX 1
typedef struct FearFrameMono {                /* 48 bytes                                                       */
  const void* data;                           /* device address of sample (0, 0) / of row 0's first byte        */
  int64_t row_stride;                         /* bytes                                                          */
  int32_t H, W;                               /* size in pixels, both >= 1                                      */
  int32_t bits, shift, packing;               /* code depth, uint16 alignment, FEAR_BAYER_* packing             */
  int32_t agc;                                /* 0: none; FEAR_AGC_MINMAX: min-max gain control                 */
  int32_t lo, hi;                             /* the frame's code range, written by fear_frame_range_mono       */
} FearFrameMono;
/* An RGB frame whose three channels are samples of one fixed-size little-endian container at a common row and pixel
 * stride (72 bytes): packed rgb24 / bgr24, RGBA / BGRA / ARGB / ABGR (and their X variants), rgb48le / rgba64le,
 * x2rgb10le / x2bgr10le (DRM XRGB2101010, DXGI R10G10B10A2) and planar gbrp at 8 to 16 bits.  Channel c of pixel
 * (y, x) is the container at c_ptr + y * row_stride + x * pixel_stride (c_ptr = r, g or b); its code is
 * (container value >> shift_c) & (2^bits - 1), mapped to 8 bits as the code itself at 8 bits and above 8 bits as
 * FearFrameBayer maps a channel, min(max(rint(255 * (v * (1 / (2^bits - 1)))), 0), 255) in float64.  Full range only;
 * alpha and X bytes and the spare bits of a container are never read into the result.  Readable combinations:
 *   container 1   bits 8, every shift 0, any addresses and strides (byte loads, no float64 work)
 *   container 2   bits 10, 12 or 16, each shift in [0, 16 - bits]; every channel address and both strides even
 *   container 4   bits 10, the shifts a permutation of {0, 10, 20}, r == g == b, the address and both strides
 *                 multiples of 4 (one word load per tap)
 * An entry is treated like a frame index outside [0, F) when any other combination is given, a channel address is
 * null, a stride is negative, or H or W is below 1. */
typedef struct FearFrameRGB {                 /* 72 bytes                                                       */
  const uint8_t *r, *g, *b;                   /* device address of the container holding R / G / B of (0, 0)    */
  int64_t row_stride, pixel_stride;           /* bytes, >= 0, shared by the three channels                      */
  int32_t H, W;                               /* size in pixels, both >= 1                                      */
  int32_t container;                          /* bytes per container: 1, 2 (LE uint16) or 4 (LE uint32)         */
  int32_t bits;                               /* code depth                                                     */
  int32_t shift_r, shift_g, shift_b;          /* code of channel c = (container value >> shift_c) & (2^bits - 1) */
  int32_t reserved;
} FearFrameRGB;
typedef struct FearTarget {      /* 64 bytes                                                         */
  int32_t frame;                 /* index into the frame table                                       */
  int32_t x, y, w, h;            /* current box in frame pixels (TrackingState.bbox)                 */
  int32_t cx, cy, cw, ch;        /* context box of the last crop (TrackingState.mapping)             */
  int32_t pad_r, pad_g, pad_b;   /* padding colour = saturate(rint(mean colour of the init frame))   */
  int32_t reserved[4];
} FearTarget;

typedef struct FearContext FearContext;

/* Verify `device` is sm_90, initialise the library's per-device state and make it the current device
 * (like torch's .cuda(id)).  Call once per device before packing weights on it; repeated calls are cheap. */
int fear_init(int device);
int fear_abi_version(void);
const char* fear_last_error(void);

/* ---- weights ------------------------------------------------------------------------
 * The library owns the canonical list of (BN-folded) tensors it needs; the host packs them
 * in that order into one fp32 blob.  Names look like "xif4_5.pw.w"; shapes are torch-native
 * ([Cout][Cin] for 1x1, [C][k][k] for depthwise, [16][3][3][3] for the stem). */
int fear_weight_count(void);
const char* fear_weight_name(int i);
int64_t fear_weight_numel(int i);

/* blob: HOST pointer to the packed fp32 tensors; offsets[i] = element offset of tensor i,
 * offsets[n] = total elements; n must equal fear_weight_count().  Creates *handle. */
int fear_pack_weights(const float* blob, const uint64_t* offsets, int n, FearContext** handle);
/* Reserve device workspace for batches up to max_batch search frames (default 1). */
int fear_reserve(FearContext* h, int max_batch);
void fear_free(FearContext* h);

/* ---- hot path -----------------------------------------------------------------------*/
/* img (B,3,H,W) -> feat (B,256,H/16,W/16);  H, W multiples of 16, <= 256. */
int fear_get_features(FearContext* h, const float* d_img, int B, int H, int W, float* d_feat, void* stream);

/* img (B,3,H,W) -> backbone features (B,112,H/16,W/16) before the neck
 * (FEARNet.feature_extractor, fear_net.py:58-61). */
int fear_backbone(FearContext* h, const float* d_img, int B, int H, int W, float* d_feat, void* stream);

/* zfeat (Bz,256,8,8) with Bz == B or 1 (broadcast); xfeat (B,256,16,16)
 * -> bbox (B,4,16,16) = exp(adjust*pred+bias), cls (B,1,16,16) = 0.1*pred (logits). */
int fear_head(FearContext* h, const float* d_zfeat, int Bz, const float* d_xfeat, int B,
              float* d_bbox, float* d_cls, void* stream);

/* BoxTower.forward(search, kernel, update) (blocks.py:174-179): as fear_head, but the CLASSIFICATION branch correlates
 * with the dynamic template d_zupdate (Bu,256,8,8), Bu == B or 1, while the regression branch keeps d_zfeat.
 * d_zupdate == NULL is exactly fear_head. */
int fear_head_update(FearContext* h, const float* d_zfeat, int Bz, const float* d_zupdate, int Bu, const float* d_xfeat,
                     int B, float* d_bbox, float* d_cls, void* stream);

/* search (B,3,256,256) + zfeat (Bz,256,8,8) -> maps and (if non-null) decoded boxes[B].
 * d_bbox / d_cls may be null when only boxes are wanted. */
int fear_track(FearContext* h, const float* d_search, const float* d_zfeat, int Bz, int B,
               float* d_bbox, float* d_cls, FearBox* d_boxes, void* stream);

/* Same as fear_track / fear_get_features but the image is the tracker's raw uint8 RGB crop in HWC layout
 * (B,H,W,3): the ImageNet normalisation of Tracker._preprocess_image (tracker/base_tracker.py:69-81,97-103)
 * is applied inside the stem kernel with the same float32 roundings (bit-identical to host normalisation);
 * the host->device copy is 4x smaller. */
int fear_track_u8(FearContext* h, const uint8_t* d_search_u8, const float* d_zfeat, int Bz, int B,
                  float* d_bbox, float* d_cls, FearBox* d_boxes, void* stream);
int fear_get_features_u8(FearContext* h, const uint8_t* d_img_u8, int B, int H, int W, float* d_feat, void* stream);

/* template (B,3,128,128) + search (B,3,256,256) -> maps (+ boxes). */
int fear_forward(FearContext* h, const float* d_template, const float* d_search, int B,
                 float* d_bbox, float* d_cls, FearBox* d_boxes, void* stream);

/* ---- search crops of any size -------------------------------------------------------
 * The reference sets its search crop in config (siam_tracker.yaml instance_size / score_size); the network is fully
 * convolutional.  These entry points take a square search of side S, a multiple of 16 in [16, 256] (the sizes
 * fear_get_features takes), or the score-map side s = S / 16 in [1, 16] where only maps are involved.  Maps are
 * (B,4,s,s) and (B,1,s,s); the decode grid is (i - s / 2) * 16 + S / 2 (utils/utils.py:183-199).  The template stays
 * (B,3,128,128) / (Bz,256,8,8): its 64 cells are the 64 correlation channels of the checkpoint.  The entry points
 * above are these at S = 256 (s = 16), with the same results bit for bit.  Batches larger than the reserved batch are
 * chunked as above.  FEAR_EINVAL: S or s outside its range, plus the rules of the fixed-size entry point. */
/* fear_head_update on search features xfeat (B,256,s,s); d_zupdate may be NULL (= fear_head). */
int fear_head_sized(FearContext* h, const float* d_zfeat, int Bz, const float* d_zupdate, int Bu, const float* d_xfeat,
                    int B, int s, float* d_bbox, float* d_cls, void* stream);
/* fear_track on search (B,3,S,S). */
int fear_track_sized(FearContext* h, const float* d_search, int S, const float* d_zfeat, int Bz, int B,
                     float* d_bbox, float* d_cls, FearBox* d_boxes, void* stream);
/* fear_track_u8 on raw uint8 RGB crops (B,S,S,3). */
int fear_track_sized_u8(FearContext* h, const uint8_t* d_search_u8, int S, const float* d_zfeat, int Bz, int B,
                        float* d_bbox, float* d_cls, FearBox* d_boxes, void* stream);
/* fear_forward on template (B,3,128,128) + search (B,3,S,S). */
int fear_forward_sized(FearContext* h, const float* d_template, const float* d_search, int S, int B,
                       float* d_bbox, float* d_cls, FearBox* d_boxes, void* stream);

/* Host pre-processing of the tracking loop on the device (get_extended_crop, reference
 * model_training/utils/utils.py:215-253 = context crop, constant-colour padding, cv2.resize(INTER_LINEAR) on uint8):
 * d_frame (H,W,3) uint8 RGB stays on the device; d_crop (out_size,out_size,3) uint8 is what fear_track_u8 /
 * fear_get_features_u8 consume.  Bit-identical to OpenCV's 8-bit fixed-point bilinear kernel.  d_params (device,
 * int32, 8 + 6 * out_size entries, so a captured CUDA graph sees per-frame values): [0..3] context x, y, w, h in frame
 * coordinates (may leave the frame), [4..6] padding colour R, G, B, [7] 0, then xofs, xa0, xa1, yofs, ya0, ya1
 * (out_size entries each): per-axis source offset and the two 11-bit coefficients, computed on the host exactly as
 * cv::resize computes them (feartracker_b200.image_ops.resize_tables). */
int fear_crop_resize_u8(const uint8_t* d_frame, int H, int W, const int32_t* d_params, uint8_t* d_crop, int out_size,
                        void* stream);

/* Tracking loop of N targets on the device (FEARMultiTracker; every target behaves like its own FEARTracker).
 * d_frames: packed uint8 frames; d_frame_table (F entries) locates them; d_targets (N) is read and updated in place.
 * One step of the loop is  fear_crop_targets_u8 -> fear_track_u8(B = N, Bz = N) -> fear_advance_targets;  the number
 * of launches does not depend on N.  Both calls are handle-free, never allocate and never synchronise; the
 * arithmetic is bit-identical to the host helpers named below (feartracker_b200.image_ops).
 *
 * fear_crop_targets_u8: one launch for all targets.  Per target: context = context_box(bbox, offset) (float64,
 * truncated), written back to the target's cx, cy, cw, ch; then the constant-padded, bilinearly resized crop of that
 * context (get_extended_crop, as fear_crop_resize_u8, with the cv::resize tables of resize_tables built on the device)
 * into d_crops (N, out_size, out_size, 3) uint8.  Search crops: offset = search_context, out_size 256; template crops:
 * offset = template_bbox_offset, out_size 128.  A target whose frame index is outside [0, F), or whose frame has H < 1
 * or W < 1, gets a crop of its padding colour and no frame is read.  FEAR_EINVAL: a null pointer, N < 1 or N > 65535,
 * F < 1, out_size outside [1, 256], offset negative or not finite. */
int fear_crop_targets_u8(const uint8_t* d_frames, const FearFrame* d_frame_table, int F, FearTarget* d_targets, int N,
                         double offset, int out_size, uint8_t* d_crops, void* stream);
/* fear_advance_targets: d_boxes (N) are the decoded boxes of the targets' search crops.  Each target's box becomes
 * clamp_bbox(rescale_bbox(box, context, instance_size), its frame's H, W): float64 multiply then add (no FMA),
 * round half to even, sides >= 3 and the trim / minimum-side rules of clamp_bbox.  A target whose frame index is
 * outside [0, F), or whose frame has H < 1 or W < 1, keeps its box.  FEAR_EINVAL: a null pointer, N < 1, F < 1,
 * instance_size < 1. */
int fear_advance_targets(const FearBox* d_boxes, const FearFrame* d_frame_table, int F, FearTarget* d_targets, int N,
                         int instance_size, void* stream);

/* The same pair with frames located through d_views (F FearFrameView entries in device memory) instead of a packed
 * buffer and FearFrame table, so frames can stay where a decoder or a CUDA pre-processing step left them (strided views
 * included).  Same semantics, arithmetic and FEAR_EINVAL rules as fear_crop_targets_u8 / fear_advance_targets; the
 * views are read when the kernels run, so a captured graph does not depend on frame addresses or shapes.  A target
 * whose view has data == NULL, H < 1 or W < 1 gets a padding-colour crop and keeps its box. */
int fear_crop_targets_view_u8(const FearFrameView* d_views, int F, FearTarget* d_targets, int N, double offset,
                              int out_size, uint8_t* d_crops, void* stream);
int fear_advance_targets_view(const FearBox* d_boxes, const FearFrameView* d_views, int F, FearTarget* d_targets, int N,
                              int instance_size, void* stream);
/* Exact per-channel sums of F frames: d_sums (F, 3) uint64 = sum over all H * W pixels of channel R, G, B (0 for an
 * entry with data == NULL, H < 1 or W < 1).  sums / (H * W) in float64 is numpy's mean of the uint8 frame bit for bit
 * (the padding colour of a new target).  Zeroes d_sums with cudaMemsetAsync, then one launch.  FEAR_EINVAL: a null
 * pointer, F < 1 or F > 65535. */
int fear_frame_sums_u8(const FearFrameView* d_views, int F, uint64_t* d_sums, void* stream);

/* The same three on YUV 4:2:0 frames located through d_views (F FearFrameYUV420 entries in device memory), so NV12 or
 * I420 surfaces can stay where a decoder left them and no RGB copy of the frame is made.  Every pixel a kernel reads is
 * converted as cv2.cvtColor converts it (each bilinear tap is converted, then interpolated; padding taps use the
 * target's RGB padding colour), so crops, boxes and sums equal those of the *_view entry points on the cv2-converted
 * RGB frame.  fear_frame_sums_yuv420_u8 sums the converted R, G and B.  fear_advance_targets_yuv420 reads only H and W.
 * Same semantics and FEAR_EINVAL rules as fear_crop_targets_view_u8 / fear_advance_targets_view / fear_frame_sums_u8;
 * an entry with a null plane, H < 1, W < 1 or an odd H or W gets a padding-colour crop, keeps its box and sums to 0. */
int fear_crop_targets_yuv420_u8(const FearFrameYUV420* d_views, int F, FearTarget* d_targets, int N, double offset,
                                int out_size, uint8_t* d_crops, void* stream);
int fear_advance_targets_yuv420(const FearBox* d_boxes, const FearFrameYUV420* d_views, int F, FearTarget* d_targets,
                                int N, int instance_size, void* stream);
int fear_frame_sums_yuv420_u8(const FearFrameYUV420* d_views, int F, uint64_t* d_sums, void* stream);

/* The same three on YUV 4:2:0 frames of the formats FearFrameYUV describes (F entries in device memory; formats may
 * differ between entries).  Each pixel a kernel reads is converted by the entry's format, so BT.709 NV12, P010 / P016
 * and yuv420p10le surfaces are read where the decoder left them.  A (BT.601, limited, 8-bit) entry gives exactly what
 * the *_yuv420 entry points give on the same planes.  Same semantics and FEAR_EINVAL rules as the *_yuv420 entry
 * points; the table is read when the kernels run, so an entry they cannot read (see FearFrameYUV) gets a padding-colour
 * crop, keeps its box and sums to 0. */
int fear_crop_targets_yuv_u8(const FearFrameYUV* d_views, int F, FearTarget* d_targets, int N, double offset,
                             int out_size, uint8_t* d_crops, void* stream);
int fear_advance_targets_yuv(const FearBox* d_boxes, const FearFrameYUV* d_views, int F, FearTarget* d_targets, int N,
                             int instance_size, void* stream);
int fear_frame_sums_yuv_u8(const FearFrameYUV* d_views, int F, uint64_t* d_sums, void* stream);

/* The same three on YUV frames of any subsampling FearFrameYCbCr describes (F entries in device memory; layouts,
 * subsamplings and formats may differ between entries), so YUYV webcam frames, NV16 / P210 / Y210 capture surfaces,
 * yuv422p and 4:4:4 decoder output are read where they are.  A 4:2:0 entry gives exactly what the *_yuv entry points
 * give on its FearFrameYUV fields.  Same semantics and FEAR_EINVAL rules as the *_yuv entry points; an entry the
 * kernels cannot read (see FearFrameYCbCr) gets a padding-colour crop, keeps its box and sums to 0. */
int fear_crop_targets_ycbcr_u8(const FearFrameYCbCr* d_views, int F, FearTarget* d_targets, int N, double offset,
                               int out_size, uint8_t* d_crops, void* stream);
int fear_advance_targets_ycbcr(const FearBox* d_boxes, const FearFrameYCbCr* d_views, int F, FearTarget* d_targets,
                               int N, int instance_size, void* stream);
int fear_frame_sums_ycbcr_u8(const FearFrameYCbCr* d_views, int F, uint64_t* d_sums, void* stream);

/* The same three on FearFrameYCbCrV210 tables, so v210 surfaces from SDI capture cards are unpacked and converted inside
 * the crop and read where they are, alongside any other YUV frame.  A v210 == 0 entry gives exactly what the *_ycbcr
 * entry points give on its FearFrameYCbCr fields.  Same semantics and FEAR_EINVAL rules as the *_ycbcr entry points; an
 * entry the kernels cannot read (see FearFrameYCbCrV210) gets a padding-colour crop, keeps its box and sums to 0. */
int fear_crop_targets_ycbcr_v210_u8(const FearFrameYCbCrV210* d_views, int F, FearTarget* d_targets, int N,
                                    double offset, int out_size, uint8_t* d_crops, void* stream);
int fear_advance_targets_ycbcr_v210(const FearBox* d_boxes, const FearFrameYCbCrV210* d_views, int F,
                                    FearTarget* d_targets, int N, int instance_size, void* stream);
int fear_frame_sums_ycbcr_v210_u8(const FearFrameYCbCrV210* d_views, int F, uint64_t* d_sums, void* stream);

/* The same three on FearFrameYCbCrHDR tables, so PQ and HLG video is tone-mapped to SDR BT.709 inside the crop, each tap
 * converted by the chain FearFrameYCbCrHDR states, alongside SDR YUV frames and v210 surfaces.  A transfer == 0 entry
 * gives exactly what the *_ycbcr_v210 entry points give on its FearFrameYCbCrV210 fields.  Same semantics and
 * FEAR_EINVAL rules as the *_ycbcr_v210 entry points; an entry the kernels cannot read (see FearFrameYCbCrHDR) gets a
 * padding-colour crop, keeps its box and sums to 0. */
int fear_crop_targets_ycbcr_hdr_u8(const FearFrameYCbCrHDR* d_views, int F, FearTarget* d_targets, int N,
                                   double offset, int out_size, uint8_t* d_crops, void* stream);
int fear_advance_targets_ycbcr_hdr(const FearBox* d_boxes, const FearFrameYCbCrHDR* d_views, int F,
                                   FearTarget* d_targets, int N, int instance_size, void* stream);
int fear_frame_sums_ycbcr_hdr_u8(const FearFrameYCbCrHDR* d_views, int F, uint64_t* d_sums, void* stream);

/* The same three on FearFrameBayer tables: raw Bayer mosaics read where they are, each tap demosaiced (and above 8 bits
 * mapped to 8 bits) inside the crop, so the kernels see cv2.cvtColor(raw, COLOR_Bayer{pattern}2RGB).  Same semantics
 * and FEAR_EINVAL rules as the *_ycbcr entry points; an entry the kernels cannot read (see FearFrameBayer) gets a
 * padding-colour crop, keeps its box and sums to 0. */
int fear_crop_targets_bayer_u8(const FearFrameBayer* d_views, int F, FearTarget* d_targets, int N, double offset,
                               int out_size, uint8_t* d_crops, void* stream);
int fear_advance_targets_bayer(const FearBox* d_boxes, const FearFrameBayer* d_views, int F, FearTarget* d_targets,
                               int N, int instance_size, void* stream);
int fear_frame_sums_bayer_u8(const FearFrameBayer* d_views, int F, uint64_t* d_sums, void* stream);

/* The code range of every readable FearFrameMono entry with agc != 0: lo = min(lo, smallest code) and
 * hi = max(hi, largest code), atomically, in the device table itself (codes after unpacking and the shift).  Entries
 * with agc 0 and entries the kernels cannot read (see FearFrameMono) are left untouched.  Run it after the table is
 * written and before the crop or the sums; a table written with lo = INT32_MAX, hi = INT32_MIN gets each frame's
 * exact range.  FEAR_EINVAL for a null table or F outside [1, 65535]. */
int fear_frame_range_mono(FearFrameMono* d_views, int F, void* stream);
/* The same three on FearFrameMono tables: single-channel frames read where they are, each tap mapped to grey (with or
 * without min-max gain control, see FearFrameMono) inside the crop, so the kernels see cv2.cvtColor(g, COLOR_GRAY2RGB).
 * Same semantics and FEAR_EINVAL rules as the *_bayer entry points; an entry the kernels cannot read gets a
 * padding-colour crop, keeps its box and sums to 0. */
int fear_crop_targets_mono_u8(const FearFrameMono* d_views, int F, FearTarget* d_targets, int N, double offset,
                              int out_size, uint8_t* d_crops, void* stream);
int fear_advance_targets_mono(const FearBox* d_boxes, const FearFrameMono* d_views, int F, FearTarget* d_targets,
                              int N, int instance_size, void* stream);
int fear_frame_sums_mono_u8(const FearFrameMono* d_views, int F, uint64_t* d_sums, void* stream);
/* The same three on FearFrameRGB tables: RGB frames in any channel order, 8-, 10-, 12- or 16-bit containers, packed
 * or planar, read where they are, each tap's channels fetched and mapped to 8 bits inside the crop (see FearFrameRGB).
 * Same semantics and FEAR_EINVAL rules as the *_mono entry points; an entry the kernels cannot read gets a
 * padding-colour crop, keeps its box and sums to 0. */
int fear_crop_targets_rgb_u8(const FearFrameRGB* d_views, int F, FearTarget* d_targets, int N, double offset,
                             int out_size, uint8_t* d_crops, void* stream);
int fear_advance_targets_rgb(const FearBox* d_boxes, const FearFrameRGB* d_views, int F, FearTarget* d_targets, int N,
                             int instance_size, void* stream);
int fear_frame_sums_rgb_u8(const FearFrameRGB* d_views, int F, uint64_t* d_sums, void* stream);

/* Rotated and mirrored frames (phone video's display rotation, cameras mounted upside down or mirrored): the crop and
 * advance entry points of any of the eight frame tables above, on each frame as it is shown rather than as it is
 * stored.  `table` names the table d_table holds, one of the *_view_u8, *_yuv_u8, *_ycbcr_u8, *_ycbcr_v210_u8,
 * *_ycbcr_hdr_u8, *_bayer_u8, *_mono_u8 and *_rgb_u8 families; the packed FearFrame and FearFrameYUV420 tables are not
 * covered.  d_orient holds F int32 orientation codes in device memory, read when the kernels run (a captured graph sees
 * each call's codes); a null d_orient means every code is 0, which gives exactly the table's plain entry point.
 *
 * A code in [0, 7] turns the stored H x W frame by 90 * (code & 3) degrees clockwise, after a left-right flip when
 * code & 4 (numpy: np.rot90(rgb[:, ::-1] if code & 4 else rgb, -(code & 3))).  Display pixel (y, x) reads stored pixel
 *     code & 3 = 0: (y, x)              display H x W
 *                1: (H - 1 - x, y)      display W x H
 *                2: (H - 1 - y, W - 1 - x)   display H x W
 *                3: (x, W - 1 - y)      display W x H
 * then xs = W - 1 - xs when code & 4.  Targets' boxes are in display coordinates and the advance clamps to the display
 * size.  The conversion of each table (YUV matrix, v210 unpack, HDR tone map, demosaic, mono gain, RGB container) is
 * applied at the stored pixel, so the crop equals the table's crop of the oriented converted frame bit for bit.  The
 * mean colour and the mono code range do not depend on orientation: the table's fear_frame_sums_* and
 * fear_frame_range_mono run on the stored frames unchanged.  A frame whose code is outside [0, 7] is treated like an
 * entry the kernels cannot read: a padding-colour crop, and its target keeps its box.  ffmpeg's autorotate convention:
 * a display-matrix rotation of r degrees (ffprobe's rotation=-90) is code (-r mod 360) / 90 (here 1).
 * One launch each; handle-free, never allocate, never synchronise.  FEAR_EINVAL: an unknown table, plus the rules of
 * the plain entry points. */
enum {
  FEAR_TABLE_VIEW = 0,
  FEAR_TABLE_YUV = 1,
  FEAR_TABLE_YCBCR = 2,
  FEAR_TABLE_YCBCR_V210 = 3,
  FEAR_TABLE_YCBCR_HDR = 4,
  FEAR_TABLE_BAYER = 5,
  FEAR_TABLE_MONO = 6,
  FEAR_TABLE_RGB = 7
};
int fear_crop_targets_oriented_u8(int table, const void* d_table, const int32_t* d_orient, int F,
                                  FearTarget* d_targets, int N, double offset, int out_size, uint8_t* d_crops,
                                  void* stream);
int fear_advance_targets_oriented(const FearBox* d_boxes, int table, const void* d_table, const int32_t* d_orient,
                                  int F, FearTarget* d_targets, int N, int instance_size, void* stream);

/* A step over some of the targets (FEARMultiTracker fed the frames of some streams only):
 *   fear_gather_targets -> crop (M) -> fear_track_u8 (B = M, Bz = M) -> advance (M) -> fear_scatter_targets
 * d_select (M pairs of int32 in device memory, read when the kernels run, so a captured graph sees each step's
 * selection): step row i is target row select[2 i], and select[2 i + 1] is the index of its frame in the step's frame
 * table.  d_targets (N FearTarget) and d_templates (N, 256, 8, 8) fp32 are the targets' rows and templates; the step
 * runs on the compact d_step_targets (M) and d_step_templates (M, 256, 8, 8) with the crop / advance entry points of
 * any frame table above.  Both calls are handle-free, never allocate and never synchronise.
 *
 * fear_gather_targets: one launch for all M.  Step row i = target row select[2 i] with frame = select[2 i + 1]; its
 * 64 KB template is copied with 16-byte loads and stores.  A row index outside [0, N) gives an inert step row: a zero
 * FearTarget with frame = -1 (so the crop gives a padding-colour crop and the advance keeps the box) and a zero
 * template.  FEAR_EINVAL: a null pointer, N < 1, M outside [1, 65535], a template buffer not 16-byte aligned. */
int fear_gather_targets(const FearTarget* d_targets, int N, const float* d_templates, const int32_t* d_select, int M,
                        FearTarget* d_step_targets, float* d_step_templates, void* stream);
/* fear_scatter_targets: one launch.  x, y, w, h, cx, cy, cw, ch of step row i are written to target row select[2 i];
 * frame, the padding colour and the reserved words are never written.  Rows outside [0, N) are skipped; the caller
 * guarantees the rows in [0, N) are distinct.  FEAR_EINVAL: a null pointer, N < 1, M outside [1, 65535]. */
int fear_scatter_targets(const FearTarget* d_step_targets, const int32_t* d_select, int M, FearTarget* d_targets, int N,
                         void* stream);

/* Decode maps produced elsewhere: bbox (B,4,16,16), cls logits (B,1,16,16) -> boxes[B].
 * apply_sigmoid = 0 treats cls as already-activated scores (decode(use_sigmoid=False)).
 * The argmax follows torch.argmax: the first maximum in row-major order, with NaN greater than every number (the
 * first NaN wins), so -0.0 and 0.0 tie and +inf beats every finite score. */
int fear_decode(const float* d_bbox, const float* d_cls, int B, int apply_sigmoid, FearBox* d_boxes,
                void* stream);

/* FEARTracker._postprocess with smooth: true (base_tracker.py:126-205) for B frames.  d_bbox (B,4,16,16),
 * d_cls (B,1,16,16) logits as fear_track writes them; d_prev_size (B,2) float64: TrackingState.prev_size
 * (target w, h in search-crop pixels); d_params (259) float64: penalty_k, window_influence, lr, then the
 * 16x16 window row-major.  All in device memory, so a captured graph sees per-frame values.
 * Per cell, in float64 with every step rounded (no FMA): score = sigmoid(cls) in float32 as fear_decode computes it;
 * x1, y1, x2, y2 = grid -/+ distances; penalty = exp(-(limit(r_c) * limit(s_c) - 1) * penalty_k) with
 * s_c = sq(x2 - x1, y2 - y1) / sq(pw, ph), r_c = (pw / ph) / ((x2 - x1) / (y2 - y1)), sq(w, h) = sqrt((w + p) (h + p)),
 * p = (w + h) / 2, limit(r) = max(r, 1 / r); pscore = (penalty * score) * (1 - window_influence) + window *
 * window_influence.  The argmax of pscore follows fear_decode's rules (first NaN, then first maximum).  The record
 * holds that cell's x1, y1, its float32 score and (row, col, flat); w, h are the smoothed size
 * pw * (1 - l) + l * (bw * l + pw * (1 - l)) with l = f32(f32(f32(penalty) * score) * f32(lr)), the float32
 * learning rate of the reference.  Only exp may differ from numpy (by 1 ulp).  Handle-free: it never allocates and
 * never synchronises.  FEAR_EINVAL: a null pointer or B < 1; device data is not validated. */
int fear_decode_smooth(const float* d_bbox, const float* d_cls, int B, const double* d_prev_size,
                       const double* d_params, FearBox* d_boxes, void* stream);

/* fear_decode / fear_decode_smooth on s x s maps, s in [1, 16] (a search of side S = 16 s): bbox (B,4,s,s), cls
 * (B,1,s,s); the grid is (i - s / 2) * 16 + 8 s, row = flat / s, col = flat % s; d_params (3 + s * s) float64:
 * penalty_k, window_influence, lr, then the s x s window row-major.  Same arithmetic and argmax rules; at s = 16 they
 * are fear_decode / fear_decode_smooth.  FEAR_EINVAL: s outside [1, 16], plus the rules of the fixed-size forms. */
int fear_decode_sized(const float* d_bbox, const float* d_cls, int B, int s, int apply_sigmoid, FearBox* d_boxes,
                      void* stream);
int fear_decode_smooth_sized(const float* d_bbox, const float* d_cls, int B, int s, const double* d_prev_size,
                             const double* d_params, FearBox* d_boxes, void* stream);

/* z (Bz,256,64), x (B,256,256)  [= (B,256,16,16)]  ->  out (B,320,256):
 * out[:, :256] = x ; out[b, 256+k, p] = sum_c z[b,c,k] * x[b,c,p].   (blocks.py:121-124)
 * Workspace-free compatibility form: a direct CUDA-core kernel on the reference layouts (one D2D copy + one launch). */
int fear_corr_concat_f32(const float* d_z, int Bz, const float* d_x, int B, float* d_out, void* stream);
/* Same result through the hot path's wgmma kernel (layout changes in the caller's scratch: d_workspace must be
 * 1024-byte aligned and hold fear_corr_concat_workspace_bytes(B, Bz) bytes). */
size_t fear_corr_concat_workspace_bytes(int B, int Bz);
int fear_corr_concat_ws_f32(const float* d_z, int Bz, const float* d_x, int B, float* d_out, void* d_workspace,
                            size_t workspace_bytes, void* stream);

/* Channels-last core of the same contraction (the kernel the hot path launches):
 * zt (Bz,64,256) [k][c], cat (B,256,320) [p][c'] whose first 256 channels hold x;
 * writes cat[b, p, 256+k] = sum_c zt[b,k,c] * cat[b,p,c]. */
int fear_corr_nhwc_f32(const float* d_zt, int Bz, float* d_cat, int B, void* stream);

/* ---- introspection (tests / bench) ---------------------------------------------------*/
/* Select a kernel implementation for a stage by name.  Returns FEAR_EINVAL for unknown names.
 * Default = best validated implementation; every alternative is parity-tested against it.
 *   "corr", "pw"   : "auto" | "ffma" | "wgmma"                  (correlation / 1x1 convs; ffma = CUDA-core baseline)
 *   "dw"           : "auto" | "pixel" | "strip" | "roll" | "tma"  (depthwise)
 *   "fuse_stem"    : "1" (default) stem + xif1_0 in one kernel | "0" four separate kernels
 *   "fuse_irf"     : "1" (default) xif2_0 (expand 1x1 -> depthwise 3x3 s2 -> project 1x1) in ONE wgmma kernel, the
 *                    6x expanded tensor never leaves the SM | "0" three kernels
 *   "fuse_dwpw"    : bit mask (default 15): 1 = IRF blocks on 16x16 maps, 4 = also those on 32x32 maps, 2 = head SepConvs run
 *                    their depthwise conv inside the 1x1 GEMM kernel, 8 = the expand-1 blocks (depthwise 3x3 -> 1x1 24 -> 24
 *                    -> + x) run as one CUDA-core kernel; all bit-identical to the two-kernel paths (the depthwise maps are
 *                    never written)
 *   "pdl"          : "1" (default) programmatic dependent launch (process-wide) */
int fear_set_option(FearContext* h, const char* key, const char* value);
/* Number of kernels launched by this handle since creation (for bench's gpu_launches).  A fused kernel that declines
 * a shape launches nothing and is not counted; only the kernels that run in its place are (the same holds for the
 * per-stage launch counts and event brackets of fear_profile / fear_stage_ms). */
int64_t fear_launch_count(const FearContext* h);
/* Changes whenever the handle's workspace pointers or options change (fear_reserve growth, fear_set_option):
 * a CUDA graph captured from calls on this handle is stale once the value differs from the one seen at capture. */
int64_t fear_generation(const FearContext* h);
/* When enabled, every stage of the next calls is bracketed by CUDA events on `stream`;
 * fear_stage_ms returns accumulated milliseconds and launch counts (synchronises events). */
int fear_profile(FearContext* h, int enable);
int fear_stage_count(void);
const char* fear_stage_name(int i);
int fear_stage_ms(FearContext* h, int i, float* ms, int64_t* launches);

/* Debug: run the stem + the first `nblocks` backbone blocks (0..16) on img (B,3,H,W) and return
 * that activation as NCHW; B must not exceed the reserved batch; H, W multiples of 16 in [16, 256]
 * (as fear_get_features). */
int fear_debug_backbone_prefix(FearContext* h, const float* d_img, int B, int H, int W, int nblocks,
                               float* d_out, void* stream);
/* Debug: copy a head intermediate of the last fear_head / fear_track / fear_forward call (or its _sized form) as NCHW
 * (B,C,s,s), s the score side of that call (16 for the fixed-size entry points): "search_features" | "cat_cls" | "cat_reg" (320 ch: encode output + correlation) |
 * "cls_dw" | "reg_dw" | "x_reg" | "cls_tower" (256 ch).  (BoxTower.forward's 3rd/4th outputs.) */
int fear_debug_head_tensor(FearContext* h, const char* name, int B, float* d_out, void* stream);
/* Debug: write `word` into every 32-bit word of the handle's workspace (every buffer fear_reserve allocated, the
 * padding between them included), ordered on `stream` (also while it is being captured).  Tests fill the workspace
 * with a poison pattern before a call to show that the call reads nothing it did not write.  The weights, the launch and
 * stage counts and fear_generation are unchanged.  FEAR_ESTATE: a null handle or one without a workspace. */
int fear_debug_fill_workspace(FearContext* h, uint32_t word, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FEAR_B200_H */
