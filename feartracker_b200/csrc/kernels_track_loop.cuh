// Device half of the multi-target tracking loop (FEARMultiTracker): the per-frame host math of FEARTracker for N
// targets at once, on per-target state that lives in device memory (FearTarget, include/fear_b200.h), so one
// captured CUDA graph steps every target with the values of the current frame.
//
//   crop_targets_u8_kernel   context box + cv::resize tables + padded bilinear crop   (image_ops.context_box,
//                            image_ops.resize_tables, crop_resize_u8_kernel)
//   advance_targets_kernel   decoded FearBox -> next frame-space box                  (image_ops.rescale_bbox +
//                            image_ops.clamp_bbox)
//   frame_sums_u8_kernel     exact per-channel sums of whole frames                    (np.mean of the padding colour)
//   frame_range_mono_kernel  code range of single-channel frames, for their gain       (the smin, smax of
//                                                                                       cv2.normalize(NORM_MINMAX))
//   gather_targets_kernel    selected FearTarget rows and templates -> compact step buffers (a step over the targets
//   scatter_targets_kernel   the stepped boxes and context boxes -> their FearTarget rows    of some streams only)
//
// The first three are templates over where the frames are and what they hold: a packed buffer + FearFrame table
// (PackedFrames) or a FearFrameView table of strided RGB frames anywhere in device memory (FrameViews), both read
// through TrackFrame; or a table of YUV frames, FearFrameYUV420 (YUV420Frames, 4:2:0, 8-bit BT.601 limited range),
// FearFrameYUV (YUVFrames, 4:2:0, the format named per entry) or FearFrameYCbCr (YCbCrFrames, 4:2:0, 4:2:2 or 4:4:4 and
// the format named per entry), all read through YUVFrame, which converts each pixel it reads to RGB; or a table of
// FearFrameYCbCrV210 records (YCbCrV210Frames), read through V210Frame, which also unpacks v210 surfaces; or a table of
// FearFrameYCbCrHDR records (YCbCrHDRFrames), read through HDRFrame, which also tone-maps PQ and HLG video to SDR; or a
// table of FearFrameBayer records (BayerFrames), read through BayerFrame, which demosaics raw Bayer mosaics; or a
// table of FearFrameMono records (MonoFrames), read through MonoFrame, which maps single-channel codes to grey; or a
// table of FearFrameRGB records (RGBFrames), read through RGBFrame, which fetches each channel from its own address in
// an 8-, 16- or 32-bit container (any channel order, packed or planar) and maps it to 8 bits.  A frame type gives H, W, empty() and the RGB triple of one pixel, rgb(y, x, p); the context box, resize tables,
// interpolation, sums and the colour conversion exist once.  Oriented wraps any of those sources for the crop and
// advance kernels: its OrientedFrame is the stored frame turned by a per-frame code (90-degree turns after an optional
// left-right flip), each display pixel mapped to its stored pixel before the stored frame's rgb().
//
// The crop and advance kernels reproduce the host's float64 / float32 arithmetic bit for bit.  nvcc contracts a*b+c
// into an FMA by default, which rounds once instead of twice, so every multiply-add here is spelled with the explicitly
// rounded intrinsics.
#pragma once
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>

#include "../../include/fear_b200.h"

namespace fear {

constexpr int kTrackCropMaxSize = 256;   // largest crop side the crop kernel builds tables for
constexpr int kTrackCropRows = 16;       // output rows per CTA
constexpr int kTrackCropThreads = 256;
constexpr int kFrameSumCtas = 128;       // CTAs per frame of frame_sums_u8_kernel
constexpr int kFrameSumThreads = 256;

// An RGB frame as the kernels read it: pixel (y, x) channel c is data[y * rs + x * ps + c * cs] (byte strides, int64).
// A value-initialised TrackFrame{} is empty.
struct TrackFrame {
  const uint8_t* data;
  long long rs, ps, cs;
  int H, W;
  // an entry the kernels treat like a frame index outside [0, F): no pixels, or nothing to read
  __device__ __forceinline__ bool empty() const { return data == nullptr || H < 1 || W < 1; }
  __device__ __forceinline__ void rgb(int y, int x, int p[3]) const {
    const uint8_t* q = data + (long long)y * rs + (long long)x * ps;
#pragma unroll
    for (int c = 0; c < 3; ++c) p[c] = __ldg(q + c * cs);
  }
};

// OpenCV 4.x cv::cvtColor(COLOR_YUV2RGB_NV12 / COLOR_YUV2RGB_I420) of one pixel, bit for bit: BT.601 limited range in
// 20-bit fixed point, with OpenCV's ITUR_BT_601_CY / CVR / CVG / CUG / CUB coefficients and round-half-up.  int32 is
// exact (every intermediate is below 2^30 in magnitude); >> is an arithmetic shift.
__device__ __forceinline__ void yuv_to_rgb_bt601(int Y, int U, int V, int p[3]) {
  const int yy = max(0, Y - 16) * 1220542 + (1 << 19);
  const int u = U - 128, v = V - 128;
  p[0] = min(max((yy + 1673527 * v) >> 20, 0), 255);
  p[1] = min(max((yy - 852492 * v - 409993 * u) >> 20, 0), 255);
  p[2] = min(max((yy + 2116026 * u) >> 20, 0), 255);
}

// min(max(rint(255 * v), 0), 255): one channel of the H.273 conversion (rint rounds half to even).
__device__ __forceinline__ int yuv_unit_to_u8(double v) {
  return (int)fmin(fmax(rint(__dmul_rn(255.0, v)), 0.0), 255.0);
}

// The constants of the ITU-T H.273 inverse for one format (include/fear_b200.h, FearFrameYUV): yn = (Y - y0) * ys,
// pb = (U - c0) * cs, pr = (V - c0) * cs, then R = yn + cR * pr, G = (yn - gB * pb) - gR * pr, B = yn + cB * pb.
// Derived at run time from the decimal Kr, Kb with the rounded intrinsics, step by step in the documented order, so
// neither host nor device constant folding can change a bit and image_ops.yuv420_to_rgb restates them exactly.
struct YUVCoefs {
  double y0, ys, c0, cs, cR, gB, gR, cB;
};

__device__ __forceinline__ YUVCoefs yuv_coefs(int matrix, bool full_range, int bits) {
  const double Kr = matrix == FEAR_YUV_BT709 ? 0.2126 : matrix == FEAR_YUV_BT2020 ? 0.2627 : 0.299;
  const double Kb = matrix == FEAR_YUV_BT709 ? 0.0722 : matrix == FEAR_YUV_BT2020 ? 0.0593 : 0.114;
  const double m = (double)(1 << (bits - 8));
  YUVCoefs k;
  if (full_range) {
    k.y0 = 0.0;
    k.ys = __ddiv_rn(1.0, (double)((1 << bits) - 1));
    k.c0 = (double)(1 << (bits - 1));
    k.cs = k.ys;
  } else {
    k.y0 = 16.0 * m;  // exact: small integers
    k.ys = __ddiv_rn(1.0, 219.0 * m);
    k.c0 = 128.0 * m;
    k.cs = __ddiv_rn(1.0, 224.0 * m);
  }
  const double Kg = __dsub_rn(__dsub_rn(1.0, Kr), Kb);
  k.cR = __dmul_rn(2.0, __dsub_rn(1.0, Kr));
  k.cB = __dmul_rn(2.0, __dsub_rn(1.0, Kb));
  k.gB = __ddiv_rn(__dmul_rn(__dmul_rn(2.0, Kb), __dsub_rn(1.0, Kb)), Kg);
  k.gR = __ddiv_rn(__dmul_rn(__dmul_rn(2.0, Kr), __dsub_rn(1.0, Kr)), Kg);
  return k;
}

// A YUV frame: luma (y, x) is the sample at Y + y * yrs + x * yps; its chroma is sample (y >> csy, x >> csx) of the U
// and V planes (shared strides uvrs, uvps); strides in bytes.  (csx, csy) is (1, 1) for 4:2:0, (1, 0) for 4:2:2 and
// (0, 0) for 4:4:4; a subsampled side must be even.  A sample is a byte, or when `wide` a uint16 whose code is
// (s >> shift) & (2^bits - 1).  rgb() converts the pixel with yuv_to_rgb_bt601 for the default format (BT.601,
// limited, 8-bit), so every kernel sees the RGB frame cv2.cvtColor would produce, and with the H.273 constants k when
// `h273`.  `bad` marks an entry the kernels cannot read (FearFrameYUV, FearFrameYCbCr).  A value-initialised
// YUVFrame{} is empty; its flags are those of the default format, so a source that only yields default-format frames
// (YUV420Frames) compiles to the cv2 conversion alone, and a source whose shifts are the constants (1, 1)
// (YUV420Frames, YUVFrames) compiles to the 4:2:0 indexing alone.
struct YUVFrame {
  const uint8_t *Y, *U, *V;
  long long yrs, yps, uvrs, uvps;
  int H, W;
  int csx = 1, csy = 1;  // also those of YUVFrame{}, so a source with constant (1, 1) shifts folds them everywhere
  int bits, shift;
  bool wide, h273, bad;
  YUVCoefs k;
  __device__ __forceinline__ bool empty() const {
    return bad || Y == nullptr || U == nullptr || V == nullptr || H < 1 || W < 1 || (H & csy) || (W & csx);
  }
  __device__ __forceinline__ int sample(const uint8_t* q) const {
    if (!wide) return __ldg(q);
    return (__ldg(reinterpret_cast<const uint16_t*>(q)) >> shift) & ((1 << bits) - 1);
  }
  __device__ __forceinline__ void rgb(int y, int x, int p[3]) const {
    const long long c = (long long)(y >> csy) * uvrs + (long long)(x >> csx) * uvps;
    convert(sample(Y + (long long)y * yrs + (long long)x * yps), sample(U + c), sample(V + c), p);
  }
  // the codes (Y, Cb, Cr) of pixel (y, x), as rgb() reads them
  __device__ __forceinline__ void codes(int y, int x, int c[3]) const {
    const long long o = (long long)(y >> csy) * uvrs + (long long)(x >> csx) * uvps;
    c[0] = sample(Y + (long long)y * yrs + (long long)x * yps);
    c[1] = sample(U + o);
    c[2] = sample(V + o);
  }
  // the RGB triple of the codes (Yc, Uc, Vc) in this frame's format
  __device__ __forceinline__ void convert(int Yc, int Uc, int Vc, int p[3]) const {
    if (!h273) {
      yuv_to_rgb_bt601(Yc, Uc, Vc, p);
      return;
    }
    const double yn = __dmul_rn(__dsub_rn((double)Yc, k.y0), k.ys);
    const double pb = __dmul_rn(__dsub_rn((double)Uc, k.c0), k.cs);
    const double pr = __dmul_rn(__dsub_rn((double)Vc, k.c0), k.cs);
    p[0] = yuv_unit_to_u8(__dadd_rn(yn, __dmul_rn(k.cR, pr)));
    p[1] = yuv_unit_to_u8(__dsub_rn(__dsub_rn(yn, __dmul_rn(k.gB, pb)), __dmul_rn(k.gR, pr)));
    p[2] = yuv_unit_to_u8(__dadd_rn(yn, __dmul_rn(k.cB, pb)));
  }
  // the unclamped R'G'B' of the H.273 inverse of the codes (Yc, Uc, Vc), before the rounding to 8 bits: convert()'s
  // arithmetic, kept apart so the SDR conversion compiles as it always has
  __device__ __forceinline__ void h273_rgb(int Yc, int Uc, int Vc, double e[3]) const {
    const double yn = __dmul_rn(__dsub_rn((double)Yc, k.y0), k.ys);
    const double pb = __dmul_rn(__dsub_rn((double)Uc, k.c0), k.cs);
    const double pr = __dmul_rn(__dsub_rn((double)Vc, k.c0), k.cs);
    e[0] = __dadd_rn(yn, __dmul_rn(k.cR, pr));
    e[1] = __dsub_rn(__dsub_rn(yn, __dmul_rn(k.gB, pb)), __dmul_rn(k.gR, pr));
    e[2] = __dadd_rn(yn, __dmul_rn(k.cB, pb));
  }
};

// Frame i of a packed buffer located by a FearFrame table (fear_crop_targets_u8 / fear_advance_targets).
struct PackedFrames {
  const uint8_t* base;
  const FearFrame* table;
  __device__ __forceinline__ TrackFrame operator()(int i) const {
    const FearFrame f = table[i];
    return TrackFrame{base + f.offset, 3LL * f.W, 3, 1, f.H, f.W};
  }
};

// Frame i of a FearFrameView table (the *_view entry points and fear_frame_sums_u8).
struct FrameViews {
  const FearFrameView* views;
  __device__ __forceinline__ TrackFrame operator()(int i) const {
    const FearFrameView v = views[i];
    return TrackFrame{v.data, v.row_stride, v.pixel_stride, v.channel_stride, v.H, v.W};
  }
};

// Frame i of a FearFrameYUV420 table (the *_yuv420 entry points): the default format, known at compile time, so only
// the cv2 conversion is compiled into these instantiations.
struct YUV420Frames {
  const FearFrameYUV420* views;
  __device__ __forceinline__ YUVFrame operator()(int i) const {
    const FearFrameYUV420 v = views[i];
    return YUVFrame{v.y, v.u, v.v, v.y_row_stride, v.y_pixel_stride, v.uv_row_stride, v.uv_pixel_stride, v.H, v.W,
                    1, 1, 8, 0, false, false, false, YUVCoefs{}};
  }
};

// The YUVFrame of the FearFrameYUV or FearFrameYCbCr record at p with chroma shifts (csx, csy): the format is checked
// and its H.273 constants derived once per thread.
template <class Record>
__device__ __forceinline__ YUVFrame yuv_frame_of(const Record* p, int csx, int csy) {
  const Record v = *p;
  const bool wide = v.bits == 10 || v.bits == 12;
  const bool odd = ((uintptr_t)v.y | (uintptr_t)v.u | (uintptr_t)v.v | v.y_row_stride | v.y_pixel_stride |
                    v.uv_row_stride | v.uv_pixel_stride) & 1;
  const bool ok = v.matrix >= FEAR_YUV_BT601 && v.matrix <= FEAR_YUV_BT2020 && (v.full_range == 0 || v.full_range == 1)
                  && (v.bits == 8 ? v.shift == 0 : wide && v.shift >= 0 && v.shift <= 16 - v.bits && !odd);
  const bool h273 = ok && !(v.matrix == FEAR_YUV_BT601 && v.full_range == 0 && v.bits == 8);
  return YUVFrame{static_cast<const uint8_t*>(v.y), static_cast<const uint8_t*>(v.u), static_cast<const uint8_t*>(v.v),
                  v.y_row_stride, v.y_pixel_stride, v.uv_row_stride, v.uv_pixel_stride, v.H, v.W,
                  csx, csy, v.bits, v.shift, wide, h273, !ok,
                  h273 ? yuv_coefs(v.matrix, v.full_range, v.bits) : YUVCoefs{}};
}

// Frame i of a FearFrameYUV table (the *_yuv entry points): 4:2:0, the format read with the entry.
struct YUVFrames {
  const FearFrameYUV* views;
  __device__ __forceinline__ YUVFrame operator()(int i) const {
    return yuv_frame_of(views + i, 1, 1);
  }
};

// Frame i of a FearFrameYCbCr table (the *_ycbcr entry points): 4:2:0, 4:2:2 or 4:4:4, the subsampling read with the
// entry too.  Any other shift pair (4:4:0, negative or large shifts) is an entry the kernels cannot read.
struct YCbCrFrames {
  const FearFrameYCbCr* views;
  __device__ __forceinline__ YUVFrame operator()(int i) const {
    return ycbcr_frame_of(views + i);
  }
  // also the v210 == 0 entries of a FearFrameYCbCrV210 table, whose leading fields are these
  template <class Record>
  static __device__ __forceinline__ YUVFrame ycbcr_frame_of(const Record* p) {
    const int csx = p->chroma_shift_x, csy = p->chroma_shift_y;
    YUVFrame f = yuv_frame_of(p, csx, csy);
    f.bad |= !(csx == 1 ? (csy == 0 || csy == 1) : (csx == 0 && csy == 0));
    return f;
  }
};

// A frame of a FearFrameYCbCrV210 table: a YUVFrame read as it is (v210 false), or a v210 surface (v210 true) whose row
// y starts at Y + y * yrs.  A row is a run of 16-byte groups of four little-endian 32-bit words, each word three 10-bit
// codes at bits 0, 10 and 20; the twelve codes of group g are, in order, Cb0 Y0 Cr0 Y1 Cb1 Y2 Cr1 Y3 Cb2 Y4 Cr2 Y5
// (pixels 6g .. 6g + 5, chroma pairs 3g .. 3g + 2), so pixel x's luma is code 2 (x % 6) + 1 and its chroma pair
// k = (x % 6) / 2 is codes 4k (Cb) and 4k + 2 (Cr) of group x / 6.  The codes go through convert(); H, W and empty()
// are the YUVFrame's, whose fields the source fills in for either kind.  A value-initialised V210Frame{} is empty.
struct V210Frame : YUVFrame {
  bool v210;
  // code i (0 .. 11) of the group at g
  static __device__ __forceinline__ int code(const uint8_t* g, unsigned i) {
    const unsigned w = i / 3;
    return (__ldg(reinterpret_cast<const uint32_t*>(g) + w) >> (10 * (i - 3 * w))) & 1023;
  }
  __device__ __forceinline__ void rgb(int y, int x, int p[3]) const {
    if (!v210) {
      YUVFrame::rgb(y, x, p);
      return;
    }
    int c[3];
    codes(y, x, c);
    convert(c[0], c[1], c[2], p);
  }
  // the codes (Y, Cb, Cr) of pixel (y, x), of either kind
  __device__ __forceinline__ void codes(int y, int x, int c[3]) const {
    if (!v210) {
      YUVFrame::codes(y, x, c);
      return;
    }
    const unsigned g = (unsigned)x / 6, r = (unsigned)x - 6 * g, k = r >> 1;
    const uint8_t* q = Y + (long long)y * yrs + 16LL * g;
    c[0] = code(q, 2 * r + 1);
    c[1] = code(q, 4 * k);
    c[2] = code(q, 4 * k + 2);
  }
};

// Frame i of a FearFrameYCbCrV210 table (the *_ycbcr_v210 entry points): with v210 == 0 the entry's FearFrameYCbCr
// fields, read exactly as YCbCrFrames reads them; with v210 == 1 a v210 surface at y with row pitch y_row_stride, 10-bit
// 4:2:2 in the entry's matrix and range (u, v, y_pixel_stride, the uv strides and shift are not read).  A v210 entry
// the kernels cannot read: a null or non-4-byte-aligned y, a pitch not a multiple of 4 or below 16 * ceil(W / 6), an
// odd W, bits other than 10, shifts other than (1, 0), or FearFrameYUV's matrix / range / size rules; any other v210
// value is unreadable too.
struct YCbCrV210Frames {
  const FearFrameYCbCrV210* views;
  __device__ __forceinline__ V210Frame operator()(int i) const {
    return v210_frame_of(views + i);
  }
  // also the FearFrameYCbCrV210 fields that lead a FearFrameYCbCrHDR record
  template <class Record>
  static __device__ __forceinline__ V210Frame v210_frame_of(const Record* p) {
    const int v210 = p->v210;
    if (v210 != 1) {
      V210Frame f{YCbCrFrames::ycbcr_frame_of(p), false};
      f.bad |= v210 != 0;
      return f;
    }
    const Record v = *p;
    const uint8_t* y = static_cast<const uint8_t*>(v.y);
    const long long pitch = v.y_row_stride;
    const bool ok = !(((uintptr_t)y | (uintptr_t)pitch) & 3) && pitch >= 16LL * (((long long)v.W + 5) / 6) &&
                    v.bits == 10 && v.chroma_shift_x == 1 && v.chroma_shift_y == 0 && v.matrix >= FEAR_YUV_BT601 &&
                    v.matrix <= FEAR_YUV_BT2020 && (v.full_range == 0 || v.full_range == 1);
    // U and V point at the surface too, so empty() refuses exactly a null y among the planes
    return V210Frame{{y, y, y, pitch, 0, 0, 0, v.H, v.W, 1, 0, 10, 0, true, true, !ok,
                      ok ? yuv_coefs(v.matrix, v.full_range, 10) : YUVCoefs{}},
                     true};
  }
};

// The HDR chain of FearFrameYCbCrHDR (include/fear_b200.h), restating image_ops.hdr_to_sdr step by step: every float64
// operation is a rounded intrinsic (no FMA contraction), exp / log / pow come from CUDA's double library.  The derived
// constants are folded rather than derived per thread: each is the hex literal of the float64 that
// image_ops.HDR_CONSTANTS names by the same hex string (tests/test_hdr_cpu.py checks the two agree and that each is its
// derivation), so no libm or constant folding on either side can change a bit.  The BT.2020 -> BT.709 matrix is
// image_ops.bt2020_to_bt709_matrix(), derived once in Python floats from the primaries and D65 and held here the same way.
constexpr double kPqC1 = 3424.0 / 4096.0, kPqC2 = 2413.0 / 4096.0 * 32.0, kPqC3 = 2392.0 / 4096.0 * 32.0;  // exact
constexpr double kHdrPqInvM1 = 0x1.91c0d56e7162bp+2;  // 1 / m1, m1 = 2610 / 16384
constexpr double kHdrPqInvM2 = 0x1.9f9b5860989b1p-7;  // 1 / m2, m2 = 2523 / 4096 * 128
constexpr double kHdrHlgA = 0.17883277;
constexpr double kHdrHlgB = 0x1.23803fd659be6p-2;     // 1 - 4a
constexpr double kHdrHlgC = 0x1.1eac9e800497cp-1;     // 0.5 - a ln(4a)
constexpr double kHdrInv24 = 0x1.aaaaaaaaaaaabp-2;    // 1 / 2.4
constexpr double kHdrRhoHdrM1 = 0x1.885043b97c4bap+3; // rho_HDR - 1, rho_HDR = 1 + 32 (1000 / 10000)^(1 / 2.4)
constexpr double kHdrLnRhoHdr = 0x1.4ad8a755a96c8p+1; // ln(rho_HDR)
constexpr double kHdrRhoSdr = 0x1.6c9af449393ffp+2;   // rho_SDR = 1 + 32 (100 / 10000)^(1 / 2.4)
constexpr double kHdrRhoSdrM1 = 0x1.2c9af449393ffp+2; // rho_SDR - 1
__device__ constexpr double kHdrGamut[3][3] = {       // linear BT.2020 -> linear BT.709
    {0x1.a915f0355ba58p+0, -0x1.2cdf4ca1c314bp-1, -0x1.2a649e47a1b10p-4},
    {-0x1.fe28a36c581d8p-4, 0x1.2205ba47cc3a2p+0, -0x1.119808835c29cp-7},
    {-0x1.2961d1c06ea4dp-6, -0x1.9bf89e59cb351p-4, 0x1.1e65112c9e6dep+0}};

__device__ __forceinline__ double hdr_clamp01(double v) { return fmin(fmax(v, 0.0), 1.0); }

// SMPTE ST 2084 EOTF: E' in [0, 1] -> cd/m2
__device__ __forceinline__ double hdr_pq_light(double e) {
  const double p = pow(e, kHdrPqInvM2);
  const double r = __ddiv_rn(fmax(__dsub_rn(p, kPqC1), 0.0), __dsub_rn(kPqC2, __dmul_rn(kPqC3, p)));
  return __dmul_rn(10000.0, pow(r, kHdrPqInvM1));
}

// BT.2100 HLG inverse OETF: E' in [0, 1] -> scene light in [0, 1]
__device__ __forceinline__ double hdr_hlg_scene(double e) {
  if (e <= 0.5) return __ddiv_rn(__dmul_rn(e, e), 3.0);
  return __ddiv_rn(__dadd_rn(exp(__ddiv_rn(__dsub_rn(e, kHdrHlgC), kHdrHlgA)), kHdrHlgB), 12.0);
}

// Y' = 0.2627 R' + 0.6780 G' + 0.0593 B' (also HLG's Ys), left to right
__device__ __forceinline__ double hdr_luma(const double c[3]) {
  return __dadd_rn(__dadd_rn(__dmul_rn(0.2627, c[0]), __dmul_rn(0.6780, c[1])), __dmul_rn(0.0593, c[2]));
}

// BT.2446-1 Method A's tone curve Y'p -> Y'c
__device__ __forceinline__ double hdr_method_a_curve(double yp) {
  if (yp <= 0.7399) return __dmul_rn(1.077, yp);
  if (yp < 0.9909) return __dsub_rn(__dadd_rn(__dmul_rn(-1.1510, __dmul_rn(yp, yp)), __dmul_rn(2.7811, yp)), 0.6302);
  return __dadd_rn(__dmul_rn(0.5, yp), 0.5);
}

// The 8-bit SDR BT.709 triple of the unclamped BT.2020 R'G'B' e under transfer FEAR_TRC_PQ or FEAR_TRC_HLG.
__device__ __forceinline__ void hdr_to_sdr(int transfer, const double e[3], int p[3]) {
  double c[3];
  if (transfer == FEAR_TRC_PQ) {
#pragma unroll
    for (int i = 0; i < 3; ++i) c[i] = hdr_pq_light(hdr_clamp01(e[i]));
  } else {
#pragma unroll
    for (int i = 0; i < 3; ++i) c[i] = hdr_hlg_scene(hdr_clamp01(e[i]));
    const double scale = __dmul_rn(1000.0, pow(hdr_luma(c), 0.2));
#pragma unroll
    for (int i = 0; i < 3; ++i) c[i] = __dmul_rn(scale, c[i]);
  }
  // normalise to the 1000 cd/m2 peak, then BT.2446-1 Method A on L^(1 / 2.4)
#pragma unroll
  for (int i = 0; i < 3; ++i) c[i] = pow(fmin(__ddiv_rn(c[i], 1000.0), 1.0), kHdrInv24);
  const double y = hdr_luma(c);
  const double yp = __ddiv_rn(log(__dadd_rn(1.0, __dmul_rn(kHdrRhoHdrM1, y))), kHdrLnRhoHdr);
  const double ysdr = __ddiv_rn(__dsub_rn(pow(kHdrRhoSdr, hdr_method_a_curve(yp)), 1.0), kHdrRhoSdrM1);
  const double f = y == 0.0 ? 0.0 : __ddiv_rn(ysdr, __dmul_rn(1.1, y));
  const double cb = __ddiv_rn(__dmul_rn(f, __dsub_rn(c[2], y)), 1.8814);
  const double cr = __ddiv_rn(__dmul_rn(f, __dsub_rn(c[0], y)), 1.4746);
  const double ytmo = __dsub_rn(ysdr, fmax(__dmul_rn(0.1, cr), 0.0));
  // the BT.2020 inverse, back to linear light, the gamut matrix, then BT.709 R'G'B'
  const double r2 = __dadd_rn(ytmo, __dmul_rn(1.4746, cr));
  const double b2 = __dadd_rn(ytmo, __dmul_rn(1.8814, cb));
  const double g2 = __ddiv_rn(__dsub_rn(__dsub_rn(ytmo, __dmul_rn(0.2627, r2)), __dmul_rn(0.0593, b2)), 0.6780);
  const double lin[3] = {pow(hdr_clamp01(r2), 2.4), pow(hdr_clamp01(g2), 2.4), pow(hdr_clamp01(b2), 2.4)};
  // one output channel at a time: fully unrolled, the frame-sums instantiation spills a register around the library
  // calls (ptxas -v)
#pragma unroll 1
  for (int i = 0; i < 3; ++i) {
    const double v = __dadd_rn(__dadd_rn(__dmul_rn(kHdrGamut[i][0], lin[0]), __dmul_rn(kHdrGamut[i][1], lin[1])),
                               __dmul_rn(kHdrGamut[i][2], lin[2]));
    p[i] = yuv_unit_to_u8(pow(hdr_clamp01(v), kHdrInv24));
  }
}

// A frame of a FearFrameYCbCrHDR table: a V210Frame read as it is (transfer 0), or its codes through the H.273 inverse
// and the HDR chain (transfer FEAR_TRC_PQ or FEAR_TRC_HLG).  A value-initialised HDRFrame{} is empty.
struct HDRFrame : V210Frame {
  int transfer;
  __device__ __forceinline__ void rgb(int y, int x, int p[3]) const {
    if (transfer == 0) {
      V210Frame::rgb(y, x, p);
      return;
    }
    int c[3];
    double e[3];
    codes(y, x, c);
    h273_rgb(c[0], c[1], c[2], e);
    hdr_to_sdr(transfer, e, p);
  }
};

// Frame i of a FearFrameYCbCrHDR table (the *_ycbcr_hdr entry points): its FearFrameYCbCrV210 fields read exactly as
// YCbCrV210Frames reads them, and the transfer.  Unreadable besides: a transfer other than 0, FEAR_TRC_PQ and
// FEAR_TRC_HLG, or an HDR transfer with a matrix other than BT.2020 or 8-bit samples.
struct YCbCrHDRFrames {
  const FearFrameYCbCrHDR* views;
  __device__ __forceinline__ HDRFrame operator()(int i) const {
    const FearFrameYCbCrHDR* p = views + i;
    const int t = p->transfer;
    HDRFrame f{YCbCrV210Frames::v210_frame_of(p), t};
    const bool hdr = (t == FEAR_TRC_PQ || t == FEAR_TRC_HLG) && p->matrix == FEAR_YUV_BT2020 && p->bits != 8;
    f.bad |= !(t == 0 || hdr);
    return f;
  }
};

// The code of pixel (y, x) of a frame of raw samples f (BayerFrame, MonoFrame: data, rs, packing, bits, shift, the
// fields of FearFrameBayer / FearFrameMono): a byte, a masked uint16, or a MIPI RAW10 / RAW12 group's high byte and
// low bits.
template <class Raw>
__device__ __forceinline__ int raw_code(const Raw& f, int y, int x) {
  const uint8_t* row = f.data + (long long)y * f.rs;
  if (f.packing == FEAR_BAYER_RAW10) {
    const uint8_t* g = row + 5LL * (x >> 2);
    const int i = x & 3;
    return (__ldg(g + i) << 2) | ((__ldg(g + 4) >> (2 * i)) & 3);
  }
  if (f.packing == FEAR_BAYER_RAW12) {
    const uint8_t* g = row + 3LL * (x >> 1);
    const int i = x & 1;
    return (__ldg(g + i) << 4) | ((__ldg(g + 2) >> (4 * i)) & 15);
  }
  if (f.bits == 8) return __ldg(row + x);
  return (__ldg(reinterpret_cast<const uint16_t*>(row) + x) >> f.shift) & ((1 << f.bits) - 1);
}

// A raw Bayer mosaic (FearFrameBayer): rgb(y, x) demosaics the pixel as cv2.cvtColor(COLOR_Bayer*2RGB) does, from the
// codes of its 3 x 3 neighbourhood in int32, with (y, x) clamped into [1, H - 2] x [1, W - 2] (cv2 copies the second and
// second-last rows and columns over the border ones).  (ry, rx) is the R site of the 2 x 2 block at (0, 0), so pixel
// (y, x) is on an R row when (y ^ ry) is even and in an R column when (x ^ rx) is; R and B sites read all nine codes, G
// sites five.  Codes above 8 bits are mapped to 8 bits per channel with ys = 1 / (2^bits - 1), the full-range luma step
// of YUVFrame.  `bad` marks an entry the kernels cannot read.  A value-initialised BayerFrame{} is empty.
struct BayerFrame {
  const uint8_t* data;
  long long rs;
  int H, W;
  int ry, rx, packing, bits, shift;
  bool bad;
  double ys;
  __device__ __forceinline__ bool empty() const { return bad || data == nullptr || H < 3 || W < 3; }
  // the code of pixel (y, x) in the entry's container
  __device__ __forceinline__ int code(int y, int x) const {
    return raw_code(*this, y, x);
  }
  __device__ __forceinline__ int to_u8(int v) const {
    return bits == 8 ? v : yuv_unit_to_u8(__dmul_rn((double)v, ys));
  }
  __device__ __forceinline__ void rgb(int y, int x, int p[3]) const {
    y = min(max(y, 1), H - 2);
    x = min(max(x, 1), W - 2);
    const int c = code(y, x), n = code(y - 1, x), s = code(y + 1, x), w = code(y, x - 1), e = code(y, x + 1);
    const bool r_row = !((y ^ ry) & 1), r_col = !((x ^ rx) & 1);
    int r, g, b;
    if (r_row == r_col) {  // an R site (both) or a B site (neither)
      const int cross = (n + s + w + e + 2) >> 2;
      const int diag = (code(y - 1, x - 1) + code(y - 1, x + 1) + code(y + 1, x - 1) + code(y + 1, x + 1) + 2) >> 2;
      r = r_row ? c : diag;
      g = cross;
      b = r_row ? diag : c;
    } else {  // a G site: its row's other colour is horizontal, its column's vertical
      const int hor = (w + e + 1) >> 1, ver = (n + s + 1) >> 1;
      r = r_row ? hor : ver;
      g = c;
      b = r_row ? ver : hor;
    }
    p[0] = to_u8(r);
    p[1] = to_u8(g);
    p[2] = to_u8(b);
  }
};

// Frame i of a FearFrameBayer table (the *_bayer entry points), checked per entry against FearFrameBayer's rules.
struct BayerFrames {
  const FearFrameBayer* views;
  __device__ __forceinline__ BayerFrame operator()(int i) const {
    const FearFrameBayer v = views[i];
    const long long W = v.W;
    const bool wide = v.packing == FEAR_BAYER_UNPACKED && v.bits != 8;
    const long long row_bytes = v.packing == FEAR_BAYER_RAW10   ? 5 * ((W + 3) / 4)
                                : v.packing == FEAR_BAYER_RAW12 ? 3 * ((W + 1) / 2)
                                                                : (wide ? 2 : 1) * W;
    bool ok;
    if (v.packing == FEAR_BAYER_RAW10) ok = v.bits == 10;
    else if (v.packing == FEAR_BAYER_RAW12) ok = v.bits == 12;
    else if (v.packing == FEAR_BAYER_UNPACKED)
      ok = v.bits == 8 ? v.shift == 0
                       : (v.bits == 10 || v.bits == 12 || v.bits == 14 || v.bits == 16) && v.shift >= 0 &&
                             v.shift <= 16 - v.bits && !(((uintptr_t)v.data | (uintptr_t)v.row_stride) & 1);
    else ok = false;
    ok = ok && v.pattern >= FEAR_BAYER_RGGB && v.pattern <= FEAR_BAYER_BGGR && v.row_stride >= row_bytes;
    return BayerFrame{static_cast<const uint8_t*>(v.data), v.row_stride, v.H, v.W, v.pattern >> 1, v.pattern & 1,
                      v.packing, v.bits, v.shift, !ok,
                      ok && v.bits != 8 ? __ddiv_rn(1.0, (double)((1 << v.bits) - 1)) : 0.0};
  }
};

// A single-channel frame (FearFrameMono): rgb(y, x) is the grey triple (g, g, g) of the pixel's code, read as
// BayerFrame reads one (raw_code).  Without gain control g is the code at 8 bits and above it the code mapped as
// BayerFrame maps a channel; with `agc` it is cv2.normalize(NORM_MINMAX, CV_8U)'s rint(fma(v, a, b)) with the float32
// gain a and offset b that MonoFrames derives from the frame's range.  `bad` marks an entry the kernels cannot read.
// A value-initialised MonoFrame{} is empty.
struct MonoFrame {
  const uint8_t* data;
  long long rs;
  int H, W;
  int packing, bits, shift;
  bool bad, agc;
  double ys;
  float a, b;
  __device__ __forceinline__ bool empty() const { return bad || data == nullptr || H < 1 || W < 1; }
  __device__ __forceinline__ int code(int y, int x) const {
    return raw_code(*this, y, x);
  }
  __device__ __forceinline__ void rgb(int y, int x, int p[3]) const {
    const int v = code(y, x);
    int g;
    if (agc) g = min(max(__float2int_rn(__fmaf_rn(__int2float_rn(v), a, b)), 0), 255);
    else g = bits == 8 ? v : yuv_unit_to_u8(__dmul_rn((double)v, ys));
    p[0] = p[1] = p[2] = g;
  }
};

// Frame i of a FearFrameMono table (the *_mono entry points), checked per entry against FearFrameMono's rules, with
// the gain of its lo / hi when agc is set: scale = 255 * (1 / (hi - lo)) (0 unless hi > lo) and shift = 0 - lo * scale
// in float64, rounded to float32, as cv2.normalize(NORM_MINMAX) derives them for convertTo.
struct MonoFrames {
  const FearFrameMono* views;
  // the entry without its gain (the range kernel, which writes lo and hi, reads only these fields); the container
  // rules are FearFrameBayer's, restated from BayerFrames (whose kernels are left to compile as they do)
  static __device__ __forceinline__ MonoFrame unscaled(const FearFrameMono* p) {
    const void* data = p->data;
    const long long rs = p->row_stride;
    const int H = p->H, W = p->W, bits = p->bits, shift = p->shift, packing = p->packing, agc = p->agc;
    const long long w = W;
    const bool wide = packing == FEAR_BAYER_UNPACKED && bits != 8;
    const long long row_bytes = packing == FEAR_BAYER_RAW10   ? 5 * ((w + 3) / 4)
                                : packing == FEAR_BAYER_RAW12 ? 3 * ((w + 1) / 2)
                                                              : (wide ? 2 : 1) * w;
    bool ok;
    if (packing == FEAR_BAYER_RAW10) ok = bits == 10;
    else if (packing == FEAR_BAYER_RAW12) ok = bits == 12;
    else if (packing == FEAR_BAYER_UNPACKED)
      ok = bits == 8 ? shift == 0
                     : (bits == 10 || bits == 12 || bits == 14 || bits == 16) && shift >= 0 && shift <= 16 - bits &&
                           !(((uintptr_t)data | (uintptr_t)rs) & 1);
    else ok = false;
    ok = ok && (agc == 0 || agc == FEAR_AGC_MINMAX) && rs >= row_bytes;
    return MonoFrame{static_cast<const uint8_t*>(data), rs, H, W, packing, bits, shift, !ok, agc != 0,
                     ok && bits != 8 ? __ddiv_rn(1.0, (double)((1 << bits) - 1)) : 0.0, 0.f, 0.f};
  }
  __device__ __forceinline__ MonoFrame operator()(int i) const {
    MonoFrame f = unscaled(views + i);
    if (f.agc && !f.bad) {
      const double lo = (double)views[i].lo, hi = (double)views[i].hi;
      const double d = __dsub_rn(hi, lo);
      const double scale = __dmul_rn(255.0, d > 0x1p-52 ? __ddiv_rn(1.0, d) : 0.0);
      const double shift = __dsub_rn(0.0, __dmul_rn(lo, scale));
      f.a = __double2float_rn(scale);
      f.b = __double2float_rn(shift);
    }
    return f;
  }
};

// An RGB frame (FearFrameRGB): channel c of pixel (y, x) is the container at c_ptr + y * rs + x * ps, its code
// (value >> shift_c) & (2^bits - 1), mapped to 8 bits as BayerFrame maps a channel (the code itself at 8 bits).  A byte
// container is read with three byte loads and no float64 work; a 32-bit container (x2rgb10: r == g == b) with one word
// load.  `bad` marks an entry the kernels cannot read.  A value-initialised RGBFrame{} is empty.
struct RGBFrame {
  const uint8_t *r, *g, *b;
  long long rs, ps;
  int H, W;
  int container, bits;
  int sr, sg, sb;
  bool bad;
  double ys;
  __device__ __forceinline__ bool empty() const { return bad || r == nullptr || H < 1 || W < 1; }
  __device__ __forceinline__ int to_u8(int v) const { return yuv_unit_to_u8(__dmul_rn((double)v, ys)); }
  __device__ __forceinline__ void rgb(int y, int x, int p[3]) const {
    const long long o = (long long)y * rs + (long long)x * ps;
    if (container == 1) {
      p[0] = __ldg(r + o);
      p[1] = __ldg(g + o);
      p[2] = __ldg(b + o);
      return;
    }
    const int m = (1 << bits) - 1;
    int v[3];
    if (container == 4) {
      const unsigned w = __ldg(reinterpret_cast<const unsigned*>(r + o));
      v[0] = (int)(w >> sr) & m;
      v[1] = (int)(w >> sg) & m;
      v[2] = (int)(w >> sb) & m;
    } else {
      v[0] = (__ldg(reinterpret_cast<const uint16_t*>(r + o)) >> sr) & m;
      v[1] = (__ldg(reinterpret_cast<const uint16_t*>(g + o)) >> sg) & m;
      v[2] = (__ldg(reinterpret_cast<const uint16_t*>(b + o)) >> sb) & m;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) p[c] = to_u8(v[c]);
  }
};

// Frame i of a FearFrameRGB table (the *_rgb entry points), checked per entry against FearFrameRGB's rules.
struct RGBFrames {
  const FearFrameRGB* views;
  __device__ __forceinline__ RGBFrame operator()(int i) const {
    const FearFrameRGB v = views[i];
    const int bits = v.bits, sr = v.shift_r, sg = v.shift_g, sb = v.shift_b;
    const uintptr_t addr = (uintptr_t)v.r | (uintptr_t)v.g | (uintptr_t)v.b | (uintptr_t)v.row_stride |
                           (uintptr_t)v.pixel_stride;
    bool ok;
    if (v.container == 1) {
      ok = bits == 8 && (sr | sg | sb) == 0;
    } else if (v.container == 2) {
      const int top = 16 - bits;
      ok = (bits == 10 || bits == 12 || bits == 16) && sr >= 0 && sr <= top && sg >= 0 && sg <= top && sb >= 0 &&
           sb <= top && !(addr & 1);
    } else if (v.container == 4) {
      // with every shift in [0, 20], the three bits are set at 0, 10 and 20 only for a permutation of {0, 10, 20}
      ok = bits == 10 && v.r == v.g && v.r == v.b && sr >= 0 && sr <= 20 && sg >= 0 && sg <= 20 && sb >= 0 &&
           sb <= 20 && ((1 << sr) | (1 << sg) | (1 << sb)) == ((1 << 0) | (1 << 10) | (1 << 20)) && !(addr & 3);
    } else {
      ok = false;
    }
    ok = ok && v.g != nullptr && v.b != nullptr && v.row_stride >= 0 && v.pixel_stride >= 0;
    return RGBFrame{v.r, v.g, v.b, v.row_stride, v.pixel_stride, v.H, v.W, v.container, bits, sr, sg, sb, !ok,
                    ok && bits != 8 ? __ddiv_rn(1.0, (double)((1 << bits) - 1)) : 0.0};
  }
};

// A frame as it is shown: the stored frame f turned by orientation code `code` (include/fear_b200.h,
// fear_crop_targets_oriented_u8): 90 * (code & 3) degrees clockwise, after a left-right flip when code & 4.  H, W are
// the display sizes (f's swapped for odd codes) and rgb(y, x) is f.rgb at the stored pixel of display pixel (y, x):
//   code & 3:   0 (y, x)   1 (Hs - 1 - x, y)   2 (Hs - 1 - y, Ws - 1 - x)   3 (x, Ws - 1 - y)
// then xs = Ws - 1 - xs when mirrored.  Every conversion behind f.rgb is a function of the stored pixel and its stored
// neighbours, so orienting the coordinates equals orienting the converted frame, bit for bit.  A code outside [0, 7]
// is empty, as is an empty f; a value-initialised OrientedFrame{} is empty.
template <class Frame>
struct OrientedFrame {
  Frame f;
  int code;
  int H, W;
  __device__ __forceinline__ bool empty() const { return code < 0 || code > 7 || f.empty(); }
  __device__ __forceinline__ void rgb(int y, int x, int p[3]) const {
    const int r = code & 3;
    int ys = r == 0 ? y : r == 1 ? f.H - 1 - x : r == 2 ? f.H - 1 - y : x;
    int xs = r == 0 ? x : r == 1 ? y : r == 2 ? f.W - 1 - x : f.W - 1 - y;
    if (code & 4) xs = f.W - 1 - xs;
    f.rgb(ys, xs, p);
  }
};

// Frame i of any frame source above, turned by code codes[i] (int32 in device memory, read when the kernel runs; a
// null codes gives code 0 everywhere).
template <class Frames>
struct Oriented {
  Frames frames;
  const int32_t* codes;
  __device__ __forceinline__ OrientedFrame<decltype(Frames{}(0))> operator()(int i) const {
    const auto f = frames(i);
    const int code = codes != nullptr ? __ldg(codes + i) : 0;
    const bool turned = code & 1;
    return {f, code, turned ? f.W : f.H, turned ? f.H : f.W};
  }
};

// One bilinear tap: the RGB triple of pixel (y, x) of the frame, or the padding colour when the tap lies outside it.
template <class Frame>
__device__ __forceinline__ void track_tap(const Frame& fr, bool inside, int y, int x, const int pad[3], int p[3]) {
  if (inside) {
    fr.rgb(y, x, p);
  } else {
#pragma unroll
    for (int c = 0; c < 3; ++c) p[c] = pad[c];
  }
}

// context_box(bbox, offset) of image_ops (reference utils.py get_extended_crop): float64, truncated to int32.
__device__ __forceinline__ void track_context_box(int x, int y, int w, int h, double off, int& cx, int& cy, int& cw,
                                                  int& ch) {
  const double grow = __dadd_rn(1.0, __dmul_rn(2.0, off));
  cx = (int)__dsub_rn((double)x, __dmul_rn((double)w, off));
  cy = (int)__dsub_rn((double)y, __dmul_rn((double)h, off));
  cw = (int)__dmul_rn((double)w, grow);
  ch = (int)__dmul_rn((double)h, grow);
}

// One entry of image_ops._axis_table: source offset and the two 11-bit coefficients of destination index d.
// float64 position (d + 0.5) * (src / dst) - 0.5 rounded to float32, float32 floor / fraction / rint(* 2048).
// clamp (the x axis): the offset is clamped into [0, src - 1] and the fraction zeroed there.
__device__ __forceinline__ void track_axis_entry(int d, int src, int dst, bool clamp, int& ofs, int& c0, int& c1) {
  const double scale = __ddiv_rn((double)src, (double)dst);
  const float f = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), 0.5));
  int s = (int)floorf(f);
  float fr = __fsub_rn(f, __int2float_rn(s));
  if (clamp) {
    if (s < 0) {
      s = 0;
      fr = 0.f;
    } else if (s >= src - 1) {
      s = src - 1;
      fr = 0.f;
    }
  }
  ofs = s;
  c0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, fr), 2048.f));
  c1 = __float2int_rn(__fmul_rn(fr, 2048.f));
}

// grid (ceil(S / kTrackCropRows), N), kTrackCropThreads threads.  CTA (tile, n) writes rows
// [tile * kTrackCropRows, +kTrackCropRows) of crop n (S x S x 3 uint8, HWC).  Every CTA of a target derives the
// context box from the target's bbox; the CTA of tile 0 also stores it in the target (cx, cy, cw, ch), which the
// advance kernel reads after the network has run.  The x tables (S entries) and this tile's y tables are built in
// shared memory; the pixel arithmetic is crop_resize_u8_kernel's.  A target whose frame index is outside [0, F), or
// whose frame is empty (empty()), gets a crop of its padding colour and reads no pixel.  Each tap is converted to RGB
// (rgb()) before it is interpolated, as cv2 converts a whole frame before copyMakeBorder + resize.
template <class Frames>
__global__ void __launch_bounds__(kTrackCropThreads) crop_targets_u8_kernel(Frames frames, int F,
                                                                            FearTarget* __restrict__ targets,
                                                                            double off, int S,
                                                                            uint8_t* __restrict__ crops) {
  __shared__ int sx[3][kTrackCropMaxSize];
  __shared__ int sy[3][kTrackCropRows];
  const int n = blockIdx.y;
  const int row0 = blockIdx.x * kTrackCropRows;
  const int rows = min(kTrackCropRows, S - row0);
  // only the fields this kernel does not write are read (tile 0 stores the context box concurrently)
  FearTarget* tp = targets + n;
  const int frame_idx = tp->frame;
  const int pad[3] = {tp->pad_r, tp->pad_g, tp->pad_b};
  int cx, cy, cw, ch;
  track_context_box(tp->x, tp->y, tp->w, tp->h, off, cx, cy, cw, ch);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    tp->cx = cx;
    tp->cy = cy;
    tp->cw = cw;
    tp->ch = ch;
  }
  uint8_t* out = crops + ((long long)n * S + row0) * S * 3;
  const bool in_range = frame_idx >= 0 && frame_idx < F;
  using Frame = decltype(frames(0));
  const Frame fr = in_range ? frames(frame_idx) : Frame{};
  if (fr.empty()) {
    for (int i = threadIdx.x; i < rows * S * 3; i += blockDim.x) out[i] = (uint8_t)pad[i % 3];
    return;
  }
  for (int i = threadIdx.x; i < S + rows; i += blockDim.x) {
    if (i < S) track_axis_entry(i, cw, S, true, sx[0][i], sx[1][i], sx[2][i]);
    else track_axis_entry(row0 + i - S, ch, S, false, sy[0][i - S], sy[1][i - S], sy[2][i - S]);
  }
  __syncthreads();
  const int H = fr.H, W = fr.W;
  for (int i = threadIdx.x; i < rows * S; i += blockDim.x) {
    const int r = i / S, dx = i - r * S;
    const int x0 = sx[0][dx], a0 = sx[1][dx], a1 = sx[2][dx];
    const int yo = sy[0][r], b0 = sy[1][r], b1 = sy[2][r];
    const int x1 = min(x0 + 1, cw - 1);
    const int y0 = min(max(yo, 0), ch - 1), y1 = min(max(yo + 1, 0), ch - 1);
    const int fx0 = cx + x0, fx1 = cx + x1, fy0 = cy + y0, fy1 = cy + y1;
    const bool in_x0 = fx0 >= 0 && fx0 < W, in_x1 = fx1 >= 0 && fx1 < W;
    const bool in_y0 = fy0 >= 0 && fy0 < H, in_y1 = fy1 >= 0 && fy1 < H;
    int p00[3], p01[3], p10[3], p11[3];
    track_tap(fr, in_y0 && in_x0, fy0, fx0, pad, p00);
    track_tap(fr, in_y0 && in_x1, fy0, fx1, pad, p01);
    track_tap(fr, in_y1 && in_x0, fy1, fx0, pad, p10);
    track_tap(fr, in_y1 && in_x1, fy1, fx1, pad, p11);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int s0 = p00[c] * a0 + p01[c] * a1;
      const int s1 = p10[c] * a0 + p11[c] * a1;
      const int v = (((b0 * (s0 >> 4)) >> 16) + ((b1 * (s1 >> 4)) >> 16) + 2) >> 2;
      out[(long long)i * 3 + c] = (uint8_t)min(max(v, 0), 255);
    }
  }
}

// One thread per target: image_ops.rescale_bbox then image_ops.clamp_bbox against the target's frame.
//   sx = cw / instance_size;  x = round(box.x * sx + cx);  w = max(3, round(box.w * sx))   (y, h alike)
// Python's round() is half-to-even = rint.  The values stay in float64 (they are integers there) until trim_box has
// clamped them into the frame, so no int32 overflow can differ from Python's unbounded ints.  A target whose frame
// index is outside [0, F), or whose frame is empty (empty()), keeps its box.  Of the frame, only H, W and
// empty() are used.
template <class Frames>
__global__ void __launch_bounds__(128) advance_targets_kernel(const FearBox* __restrict__ boxes, Frames frames, int F,
                                                              FearTarget* __restrict__ targets, int N,
                                                              int instance_size) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  FearTarget t = targets[n];
  if (t.frame < 0 || t.frame >= F) return;
  const auto fr = frames(t.frame);
  if (fr.empty()) return;
  const FearBox b = boxes[n];
  const double sx = __ddiv_rn((double)t.cw, (double)instance_size);
  const double sy = __ddiv_rn((double)t.ch, (double)instance_size);
  const double x = rint(__dadd_rn(__dmul_rn(b.x, sx), (double)t.cx));
  const double y = rint(__dadd_rn(__dmul_rn(b.y, sy), (double)t.cy));
  const double w = fmax(3.0, rint(__dmul_rn(b.w, sx)));
  const double h = fmax(3.0, rint(__dmul_rn(b.h, sy)));
  const double W = (double)fr.W, H = (double)fr.H;
  // trim_box
  const double x1 = fmin(fmax(0.0, x), W), y1 = fmin(fmax(0.0, y), H);
  const double x2 = fmin(fmax(0.0, __dadd_rn(x1, w)), W), y2 = fmin(fmax(0.0, __dadd_rn(y1, h)), H);
  int ox = (int)x1, oy = (int)y1, ow = (int)(x2 - x1), oh = (int)(y2 - y1);
  // clamp_bbox: minimum side 3, shifted back into the frame
  if (ow < 3) {
    ow = 3;
    ox -= max(0, ox + ow - fr.W);
  }
  if (oh < 3) {
    oh = 3;
    oy -= max(0, oy + oh - fr.H);
  }
  t.x = ox;
  t.y = oy;
  t.w = ow;
  t.h = oh;
  targets[n] = t;
}

// grid (kFrameSumCtas, F), kFrameSumThreads threads: sums[f][c] += sum of channel c over the pixels of frame f that
// CTA (g, f) visits (a grid-stride loop over the frame's H * W pixels, row-major; the (y, x) position advances by the
// stride's quotient and remainder, so the loop needs no division).  One uint64 atomicAdd per channel per CTA: integer
// sums in any order are the same, so the result is deterministic.  sums must be zero on entry; an empty frame adds 0.
// The sums are of rgb(), so a YUV frame sums its converted RGB pixels.
template <class Frames>
__global__ void __launch_bounds__(kFrameSumThreads) frame_sums_u8_kernel(Frames frames,
                                                                         unsigned long long* __restrict__ sums) {
  __shared__ unsigned long long part[3][kFrameSumThreads / 32];
  const auto fr = frames(blockIdx.y);
  if (fr.empty()) return;
  const long long W = fr.W, stride = (long long)gridDim.x * blockDim.x;
  const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long sy = stride / W, sx = stride - sy * W;
  unsigned long long acc[3] = {0, 0, 0};
  for (long long y = i0 / W, x = i0 - y * W; y < fr.H;) {
    int p[3];
    fr.rgb((int)y, (int)x, p);
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] += p[c];
    x += sx;
    y += sy;
    if (x >= W) {
      x -= W;
      ++y;
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    unsigned long long v = acc[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if (lane == 0) part[c][warp] = v;
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    unsigned long long v = 0;
#pragma unroll
    for (int w = 0; w < kFrameSumThreads / 32; ++w) v += part[threadIdx.x][w];
    atomicAdd(sums + 3LL * blockIdx.y + threadIdx.x, v);
  }
}

// grid (kFrameSumCtas, F), kFrameSumThreads threads: the code range of FearFrameMono entry f with agc set, over the
// pixels CTA (g, f) visits (frame_sums_u8_kernel's grid-stride walk), reduced per warp and per CTA, then one atomicMin
// on the entry's lo and one atomicMax on its hi.  Min and max in any order are the same, so the result is
// deterministic.  Entries without agc and entries the kernels cannot read are not touched.
__global__ void __launch_bounds__(kFrameSumThreads) frame_range_mono_kernel(FearFrameMono* views) {
  __shared__ int part[2][kFrameSumThreads / 32];
  FearFrameMono* p = views + blockIdx.y;
  const MonoFrame fr = MonoFrames::unscaled(p);
  if (fr.empty() || !fr.agc) return;
  const long long W = fr.W, stride = (long long)gridDim.x * blockDim.x;
  const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long sy = stride / W, sx = stride - sy * W;
  int lo = INT_MAX, hi = INT_MIN;
  for (long long y = i0 / W, x = i0 - y * W; y < fr.H;) {
    const int v = fr.code((int)y, (int)x);
    lo = min(lo, v);
    hi = max(hi, v);
    x += sx;
    y += sy;
    if (x >= W) {
      x -= W;
      ++y;
    }
  }
  lo = __reduce_min_sync(0xffffffffu, lo);
  hi = __reduce_max_sync(0xffffffffu, hi);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    part[0][warp] = lo;
    part[1][warp] = hi;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int w = 1; w < kFrameSumThreads / 32; ++w) {
      lo = min(lo, part[0][w]);
      hi = max(hi, part[1][w]);
    }
    if (lo <= hi) {  // a CTA that visited no pixel has nothing to add
      atomicMin(&p->lo, lo);
      atomicMax(&p->hi, hi);
    }
  }
}

constexpr int kTemplateVec4 = 256 * 8 * 8 / 4;  // float4s of one (256, 8, 8) fp32 template: 64 KB
constexpr int kGatherCtasPerRow = 4;            // CTAs copying one template
constexpr int kGatherThreads = 256;
constexpr int kGatherVec4PerThread = kTemplateVec4 / (kGatherCtasPerRow * kGatherThreads);
static_assert(kGatherVec4PerThread * kGatherCtasPerRow * kGatherThreads == kTemplateVec4, "gather tiling");

// grid (kGatherCtasPerRow, M), kGatherThreads threads.  Step row i takes target row select[2 i]: CTA (c, i) copies
// quarter c of its template with 16-byte loads and stores (all loads issued before the stores), and thread 0 of CTA
// (0, i) writes the FearTarget with frame = select[2 i + 1].  A row outside [0, N) gives an inert step row: a zero
// FearTarget with frame = -1 and a zero template.
__global__ void __launch_bounds__(kGatherThreads) gather_targets_kernel(const FearTarget* __restrict__ targets, int N,
                                                                        const float4* __restrict__ templates,
                                                                        const int32_t* __restrict__ select,
                                                                        FearTarget* __restrict__ step_targets,
                                                                        float4* __restrict__ step_templates) {
  const int i = blockIdx.y;
  const int row = __ldg(select + 2 * i);
  const bool valid = row >= 0 && row < N;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    FearTarget t = {};
    t.frame = -1;
    if (valid) {
      t = targets[row];
      t.frame = __ldg(select + 2 * i + 1);
    }
    step_targets[i] = t;
  }
  const int k0 = blockIdx.x * (kGatherThreads * kGatherVec4PerThread) + threadIdx.x;
  float4* dst = step_templates + (long long)i * kTemplateVec4 + k0;
  float4 v[kGatherVec4PerThread];
#pragma unroll
  for (int j = 0; j < kGatherVec4PerThread; ++j)
    v[j] = valid ? __ldg(templates + (long long)row * kTemplateVec4 + k0 + j * kGatherThreads)
                 : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int j = 0; j < kGatherVec4PerThread; ++j) dst[j * kGatherThreads] = v[j];
}

// One thread per step row: x, y, w, h, cx, cy, cw, ch of step row i go back to target row select[2 i]; frame, the
// padding colour and the reserved words of the target row are not written.  Rows outside [0, N) are skipped.
__global__ void __launch_bounds__(128) scatter_targets_kernel(const FearTarget* __restrict__ step_targets,
                                                              const int32_t* __restrict__ select, int M,
                                                              FearTarget* __restrict__ targets, int N) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const int row = select[2 * i];
  if (row < 0 || row >= N) return;
  const FearTarget s = step_targets[i];
  FearTarget* t = targets + row;
  t->x = s.x;
  t->y = s.y;
  t->w = s.w;
  t->h = s.h;
  t->cx = s.cx;
  t->cy = s.cy;
  t->cw = s.cw;
  t->ch = s.ch;
}

}  // namespace fear
