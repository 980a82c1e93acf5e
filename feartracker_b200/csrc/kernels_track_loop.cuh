// Device half of the multi-target tracking loop (FEARMultiTracker): the per-frame host math of FEARTracker for N
// targets at once, on per-target state that lives in device memory (FearTarget, include/fear_b200.h), so one
// captured CUDA graph steps every target with the values of the current frame.
//
//   crop_targets_u8_kernel   context box + cv::resize tables + padded bilinear crop   (image_ops.context_box,
//                            image_ops.resize_tables, crop_resize_u8_kernel)
//   advance_targets_kernel   decoded FearBox -> next frame-space box                  (image_ops.rescale_bbox +
//                            image_ops.clamp_bbox)
//   frame_sums_u8_kernel     exact per-channel sums of whole frames                    (np.mean of the padding colour)
//
// The crop and advance kernels are templates over where the frames are: a packed buffer + FearFrame table
// (PackedFrames) or a FearFrameView table of strided frames anywhere in device memory (FrameViews).  Both read a frame
// through the same TrackFrame (address, byte strides, H, W), so there is one copy of the arithmetic.
//
// The crop and advance kernels reproduce the host's float64 / float32 arithmetic bit for bit.  nvcc contracts a*b+c
// into an FMA by default, which rounds once instead of twice, so every multiply-add here is spelled with the explicitly
// rounded intrinsics.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/fear_b200.h"

namespace fear {

constexpr int kTrackCropMaxSize = 256;   // largest crop side the crop kernel builds tables for
constexpr int kTrackCropRows = 16;       // output rows per CTA
constexpr int kTrackCropThreads = 256;
constexpr int kFrameSumCtas = 128;       // CTAs per frame of frame_sums_u8_kernel
constexpr int kFrameSumThreads = 256;

// A frame as the kernels read it: pixel (y, x) channel c is data[y * rs + x * ps + c * cs] (byte strides, int64).
struct TrackFrame {
  const uint8_t* data;
  long long rs, ps, cs;
  int H, W;
};

// An entry the kernels treat like a frame index outside [0, F): no pixels, or nothing to read.
__device__ __forceinline__ bool track_frame_empty(const TrackFrame& f) {
  return f.data == nullptr || f.H < 1 || f.W < 1;
}

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
// whose frame is empty (track_frame_empty), gets a crop of its padding colour and reads no pixel.
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
  const TrackFrame fr = in_range ? frames(frame_idx) : TrackFrame{nullptr, 0, 0, 0, 0, 0};
  if (track_frame_empty(fr)) {
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
    const uint8_t* r0 = fr.data + (long long)fy0 * fr.rs;
    const uint8_t* r1 = fr.data + (long long)fy1 * fr.rs;
    const long long o0 = (long long)fx0 * fr.ps, o1 = (long long)fx1 * fr.ps;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const long long oc = c * fr.cs;
      const int p00 = (in_y0 && in_x0) ? (int)__ldg(r0 + o0 + oc) : pad[c];
      const int p01 = (in_y0 && in_x1) ? (int)__ldg(r0 + o1 + oc) : pad[c];
      const int p10 = (in_y1 && in_x0) ? (int)__ldg(r1 + o0 + oc) : pad[c];
      const int p11 = (in_y1 && in_x1) ? (int)__ldg(r1 + o1 + oc) : pad[c];
      const int s0 = p00 * a0 + p01 * a1;
      const int s1 = p10 * a0 + p11 * a1;
      const int v = (((b0 * (s0 >> 4)) >> 16) + ((b1 * (s1 >> 4)) >> 16) + 2) >> 2;
      out[(long long)i * 3 + c] = (uint8_t)min(max(v, 0), 255);
    }
  }
}

// One thread per target: image_ops.rescale_bbox then image_ops.clamp_bbox against the target's frame.
//   sx = cw / instance_size;  x = round(box.x * sx + cx);  w = max(3, round(box.w * sx))   (y, h alike)
// Python's round() is half-to-even = rint.  The values stay in float64 (they are integers there) until trim_box has
// clamped them into the frame, so no int32 overflow can differ from Python's unbounded ints.  A target whose frame
// index is outside [0, F), or whose frame is empty (track_frame_empty), keeps its box.
template <class Frames>
__global__ void __launch_bounds__(128) advance_targets_kernel(const FearBox* __restrict__ boxes, Frames frames, int F,
                                                              FearTarget* __restrict__ targets, int N,
                                                              int instance_size) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  FearTarget t = targets[n];
  if (t.frame < 0 || t.frame >= F) return;
  const TrackFrame fr = frames(t.frame);
  if (track_frame_empty(fr)) return;
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
__global__ void __launch_bounds__(kFrameSumThreads) frame_sums_u8_kernel(FrameViews frames,
                                                                         unsigned long long* __restrict__ sums) {
  __shared__ unsigned long long part[3][kFrameSumThreads / 32];
  const TrackFrame fr = frames(blockIdx.y);
  if (track_frame_empty(fr)) return;
  const long long W = fr.W, stride = (long long)gridDim.x * blockDim.x;
  const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long sy = stride / W, sx = stride - sy * W;
  unsigned long long acc[3] = {0, 0, 0};
  for (long long y = i0 / W, x = i0 - y * W; y < fr.H;) {
    const uint8_t* p = fr.data + y * fr.rs + x * fr.ps;
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] += __ldg(p + c * fr.cs);
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

}  // namespace fear
