// irf_s2_fused_kernel -- the inverted-residual block xif2_0 of fbnet_c as ONE kernel (sm_90a):
//
//     Y = W2 * relu(dw3x3_s2(relu(W1 * X + b1)) + bd) + b2          16 -> 96 -> 96 -> 24 channels, 2x down
//
// (mobile_cv IRF block pw -> dw -> pwl as restated in oracle/fbnet_c.py:95-110; call site reference
// model_training/model/blocks.py:27-35).  Unfused this block is three kernels that write and re-read the 6x
// expanded tensor E = relu(W1 X + b1) and the depthwise map; here E and the depthwise output never leave the SM.
//
// Persistent CTAs (min(tiles, SMs)), two warpgroups.  A tile is 8 x 16 output pixels (= one M = 128 tile of the
// project GEMM); CTA c walks tiles c, c + G, c + 2G, ... and its warpgroups take them in turn, each running the whole
// chain of its tile on its own buffers with per-warpgroup named barriers, so one warpgroup's depthwise (FFMA) runs
// while the other waits on its wgmma:
//
//   prologue  the packed weights image -> shared memory once per CTA (constant data: before the PDL wait).
//   load      the 17 x 33 input pixels the tile needs (halo of the stride-2 3x3 window; 561 pixels, 64 B each): one
//             4-D TMA box per tile into the warpgroup's box buffer, SWIZZLE_64B, zero outside the image.  The next
//             tile's box is issued as soon as the warpgroup's last expand has read the current one.
//   per 16-channel half-slab (c, h) of the expanded tensor:
//     expand     nine 64-row blocks of the box: D[64 x 16] = A * W1[32c + 16h, +16)^T as 3xTF32 wgmma with the A
//                fragments split in registers; + b1, ReLU, zero outside the image (the depthwise conv zero-pads E,
//                and E(0) = relu(b1) != 0) -> 561 x 16-channel fp32 half-slab in shared memory.
//     depthwise  3x3 stride 2 out of that half-slab (same FMA order as the stand-alone depthwise kernels) -> + bd,
//                ReLU -> channels [16h, 16h + 16) of the A tile of the project GEMM (SWIZZLE_128B layout).
//   after both halves of slab c:
//     project    acc2[128 x 32] += dw_c * W2[:, c]^T, accumulators kept in registers across the slabs.
//   store     Y = acc2 + b2.
//
// Every output element sees the MMAs of the three-kernel path in the same K order (wgmma gives an element the same
// result whatever the instruction's N), the same depthwise FMA order and the same epilogue additions, through the
// same tc::mma3, so the block is bit-identical to the three-kernel path (tests/test_gpu_tcgen05.py, test_gpu_irf_schedule.py).
//
// smem (bytes): weights image 41216 (W1 [hi|lo] rows, W2 [hi;lo] x 3 chunks, dw, biases) | 2 A tiles 16384 |
// 2 input boxes 36864 | 2 half-slabs 35904 | 2 mbarriers.
#pragma once
#include "tc_common.cuh"

namespace fear {
namespace tc {

constexpr int kIrfCin = 16, kIrfMid = 96, kIrfCout = 24, kIrfCoutPad = 32;
constexpr int kIrfTH = 8, kIrfTW = 16;                          // output tile
constexpr int kIrfIH = 2 * kIrfTH + 1, kIrfIW = 2 * kIrfTW + 1;  // 17 x 33 input pixels
constexpr int kIrfPix = kIrfIH * kIrfIW;                        // 561
constexpr int kIrfMB = (kIrfPix + 63) / 64;                     // 9 64-row blocks of the expand GEMM
constexpr int kIrfSlabs = kIrfMid / 32;                         // 3
constexpr int kIrfThreads = 256;                                // two warpgroups
constexpr int kIrfExpandGroup = 3;                              // 64-row expand blocks in flight per wgmma wait

// weights image (floats), copied verbatim into shared memory
constexpr int kIrfW1Floats = kIrfMid * 32;                        // [96 rows][hi 16 | lo 16], SWIZZLE_128B
constexpr int kIrfW2Floats = kIrfSlabs * 2 * kIrfCoutPad * 32;    // per chunk: [hi 32 rows ; lo 32 rows] x 32 k
constexpr int kIrfDwFloats = 9 * kIrfMid;
constexpr int kIrfImageFloats = kIrfW1Floats + kIrfW2Floats + kIrfDwFloats + kIrfMid + kIrfMid + kIrfCoutPad;

constexpr int kIrfOffImg = 0;
constexpr int kIrfOffW1 = kIrfOffImg;
constexpr int kIrfOffW2 = kIrfOffW1 + kIrfW1Floats * 4;
constexpr int kIrfOffDw = kIrfOffW2 + kIrfW2Floats * 4;
constexpr int kIrfOffB1 = kIrfOffDw + kIrfDwFloats * 4;
constexpr int kIrfOffBd = kIrfOffB1 + kIrfMid * 4;
constexpr int kIrfOffB2 = kIrfOffBd + kIrfMid * 4;
// per-warpgroup buffers (two of each)
constexpr int kIrfABytes = 128 * 128;                 // raw fp32 A tile of the project GEMM, 128 rows x 32 channels
constexpr int kIrfBoxBytes = kIrfMB * 64 * 64;        // input box: 576 rows of 64 B; TMA writes the first 561
constexpr int kIrfBoxTxBytes = kIrfPix * 64;
constexpr int kIrfHalfSlabBytes = kIrfPix * 64;       // 561 pixels x 16 channels of E
constexpr int kIrfOffA = ((kIrfOffB2 + kIrfCoutPad * 4 + 1023) / 1024) * 1024;
constexpr int kIrfOffBox = kIrfOffA + 2 * kIrfABytes;
constexpr int kIrfOffSlab = kIrfOffBox + 2 * kIrfBoxBytes;
constexpr int kIrfOffBar = kIrfOffSlab + 2 * kIrfHalfSlabBytes;
constexpr int kIrfSmemBytes = kIrfOffBar + 2 * 8 + 1024 /*alignment slack*/;
static_assert(kIrfSmemBytes <= 232448, "fused IRF kernel exceeds the 227 KB shared-memory limit");
static_assert(kIrfOffW1 % 1024 == 0 && kIrfOffW2 % 1024 == 0, "swizzled weight tiles must be 1024-byte aligned");
static_assert(kIrfOffBox % 1024 == 0 && kIrfBoxBytes % 1024 == 0, "SWIZZLE_64B boxes must be 512-byte aligned");
static_assert(kIrfMB % kIrfExpandGroup == 0, "expand groups must tile the 64-row blocks");

// Byte offset of 16-byte chunk `chunk` (channels 4 chunk .. 4 chunk + 3) of box pixel pb in a half-slab.  Pixels
// pb and pb ^ 1 trade places when bit 3 of pb is set, and the chunks of a pixel are XORed with bit 1 of pb: the
// expand epilogue's 8-byte stores (4 consecutive pixels per half warp) and the depthwise's 16-byte loads (pixels pb
// and pb + 8, 4 chunks each, per quarter warp) are then conflict free.
__device__ __forceinline__ int irf_slab_off(int pb, int chunk) {
  return (pb ^ ((pb >> 3) & 1)) * 64 + ((chunk ^ (pb & 2)) << 4);
}

struct IrfParams {
  float* Y;            // [B][H/2][W/2][24]
  const float* image;  // kIrfImageFloats packed weights (device)
  int B, H, W;         // input map
  int tiles_x, tiles_y, num_tiles;
};

// Host: build the shared-memory weights image.  w1_hi/w1_lo [96][16], w2_hi/w2_lo [24][96] (tf32-split copies the
// tensor-core path already keeps), dw [9][96] (tap-major), biases.
inline void irf_build_image(float* img, const float* w1_hi, const float* w1_lo, const float* w2_hi, const float* w2_lo,
                            const float* dw, const float* b1, const float* bd, const float* b2) {
  for (int i = 0; i < kIrfImageFloats; ++i) img[i] = 0.f;
  float* W1 = img;
  for (int r = 0; r < kIrfMid; ++r)
    for (int j = 0; j < 8; ++j) {  // logical 16-byte chunk j of row r: j < 4 -> hi[4j..], else lo[4(j-4)..]
      const float* src = (j < 4 ? w1_hi : w1_lo) + r * kIrfCin + 4 * (j & 3);
      float* dst = W1 + r * 32 + 4 * (j ^ (r & 7));
      for (int e = 0; e < 4; ++e) dst[e] = src[e];
    }
  float* W2 = img + kIrfW1Floats;
  for (int c = 0; c < kIrfSlabs; ++c)
    for (int part = 0; part < 2; ++part)
      for (int n = 0; n < kIrfCout; ++n)
        for (int j = 0; j < 8; ++j) {
          const float* src = (part == 0 ? w2_hi : w2_lo) + n * kIrfMid + 32 * c + 4 * j;
          float* dst = W2 + ((c * 2 + part) * kIrfCoutPad + n) * 32 + 4 * (j ^ (n & 7));
          for (int e = 0; e < 4; ++e) dst[e] = src[e];
        }
  float* p = img + kIrfW1Floats + kIrfW2Floats;
  for (int i = 0; i < kIrfDwFloats; ++i) p[i] = dw[i];
  p += kIrfDwFloats;
  for (int i = 0; i < kIrfMid; ++i) p[i] = b1[i];
  p += kIrfMid;
  for (int i = 0; i < kIrfMid; ++i) p[i] = bd[i];
  p += kIrfMid;
  for (int i = 0; i < kIrfCout; ++i) p[i] = b2[i];
}

__device__ __forceinline__ void irf_wg_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }

__global__ void __launch_bounds__(kIrfThreads, 1)
irf_s2_fused_kernel(const __grid_constant__ CUtensorMap tmX, const IrfParams p) {
  extern __shared__ uint8_t irf_smem_raw[];
  uint8_t* smem = irf_smem_raw + ((1024u - (smem_u32(irf_smem_raw) & 1023u)) & 1023u);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kIrfOffBar);  // one per warpgroup: its box has landed
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2, wt = threadIdx.x & 127, g = lane >> 2, t = lane & 3;
  if (threadIdx.x == 0) {
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    fence_mbar_init();
    prefetch_tmap(&tmX);
  }
  {  // weights image -> shared memory, once per CTA (constant data: may be read before the previous kernel has finished)
    const float4* src = reinterpret_cast<const float4*>(p.image);
    float4* dst = reinterpret_cast<float4*>(smem + kIrfOffImg);
    for (int i = threadIdx.x; i < kIrfImageFloats / 4; i += kIrfThreads) dst[i] = __ldg(src + i);
  }
  {  // rows 561..575 of the last expand block lie past the box: zero them once so the MMAs only ever see finite values
    constexpr int kTail = (kIrfBoxBytes - kIrfBoxTxBytes) / 16;
    for (int i = threadIdx.x; i < 2 * kTail; i += kIrfThreads)
      reinterpret_cast<float4*>(smem + kIrfOffBox + (i / kTail) * kIrfBoxBytes + kIrfBoxTxBytes)[i % kTail] =
          make_float4(0.f, 0.f, 0.f, 0.f);
  }
  fence_proxy_async_smem();  // the tensor core reads W1 / W2 through the async proxy
  __syncthreads();
  pdl_trigger();
  pdl_wait();  // X is written by the previous kernel in the stream

  // The box of `tile` -> box buffer s.  Box pixel (by, bx) is input pixel (2 oy0 - 1 + by, 2 ox0 - 1 + bx): only
  // row / column -1 can fall outside the image (H, W are multiples of 16 / 32), and TMA fills those with zeros.
  auto issue_box = [&](int tile, int s) {
    const int tx = tile % p.tiles_x, rest = tile / p.tiles_x;
    mbar_arrive_expect_tx(&full[s], kIrfBoxTxBytes);
    tma_load_4d(smem + kIrfOffBox + s * kIrfBoxBytes, &tmX, &full[s], 0, 2 * kIrfTW * tx - 1,
                2 * kIrfTH * (rest % p.tiles_y) - 1, rest / p.tiles_y);
  };
  const int stride = 2 * gridDim.x;  // a warpgroup's tiles: blockIdx.x + wg G, + 2G, ...
  if (wt == 0 && blockIdx.x + wg * gridDim.x < p.num_tiles) issue_box(blockIdx.x + wg * gridDim.x, wg);

  const uint8_t* box = smem + kIrfOffBox + wg * kIrfBoxBytes;
  uint8_t* slab = smem + kIrfOffSlab + wg * kIrfHalfSlabBytes;
  uint8_t* a2 = smem + kIrfOffA + wg * kIrfABytes;
  const int rw = (warp & 3) * 16 + g;  // this thread's first row inside a 64-row block (second: + 8)
  const int Ho = p.H >> 1, Wo = p.W >> 1;
  uint32_t phase = 0;
#pragma unroll 1
  for (int tile = blockIdx.x + wg * gridDim.x; tile < p.num_tiles; tile += stride, phase ^= 1u) {
    const int tx = tile % p.tiles_x, rest = tile / p.tiles_x;
    const int b = rest / p.tiles_y, oy0 = (rest % p.tiles_y) * kIrfTH, ox0 = tx * kIrfTW;
    const bool border = (oy0 == 0) || (ox0 == 0);  // only these tiles have box pixels outside the image
    float acc2m[2][16], acc2c[2][16];
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int i = 0; i < 16; ++i) acc2m[m][i] = acc2c[m][i] = 0.f;
    mbar_wait(&full[wg], phase);

#pragma unroll 1
    for (int c = 0; c < kIrfSlabs; ++c) {
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
        // ---- (1) expand: relu(X W1[32c + 16h, +16)^T + b1), zero outside the image -> half-slab ----
        const uint32_t brow = smem_u32(smem + kIrfOffW1) + c * 4096 + h * 2048;  // 16 rows of W1: [hi 64 B | lo 64 B]
        const float* b1 = reinterpret_cast<const float*>(smem + kIrfOffB1) + c * 32 + h * 16;
#pragma unroll 1
        for (int mb0 = 0; mb0 < kIrfMB; mb0 += kIrfExpandGroup) {
          uint32_t hi[kIrfExpandGroup][2][4], lo[kIrfExpandGroup][2][4];
          float em[kIrfExpandGroup][8], ec[kIrfExpandGroup][8];
#pragma unroll
          for (int q = 0; q < kIrfExpandGroup; ++q) {
#pragma unroll
            for (int j = 0; j < 2; ++j)
#pragma unroll
              for (int e = 0; e < 4; ++e) {  // box row r, channels 8j + 4(e >> 1) + t; SWIZZLE_64B: chunk ^ ((r >> 1) & 3)
                const int r = (mb0 + q) * 64 + rw + (e & 1) * 8;
                const float v = *reinterpret_cast<const float*>(box + r * 64 + (((2 * j + (e >> 1)) ^ ((r >> 1) & 3)) << 4) + t * 4);
                const uint32_t hv = __float_as_uint(v) & 0xFFFFE000u;
                hi[q][j][e] = hv;
                lo[q][j][e] = __float_as_uint(v - __uint_as_float(hv));
              }
#pragma unroll
            for (int i = 0; i < 8; ++i) em[q][i] = ec[q][i] = 0.f;
          }
          wg_fence();
#pragma unroll
          for (int q = 0; q < kIrfExpandGroup; ++q)
#pragma unroll
            for (int j = 0; j < 2; ++j) mma3<16>(em[q], ec[q], hi[q][j], lo[q][j], brow + j * 32, brow + 64 + j * 32);
          wg_commit();
          wg_wait();
#pragma unroll
          for (int q = 0; q < kIrfExpandGroup; ++q)
#pragma unroll
            for (int hrow = 0; hrow < 2; ++hrow) {
              const int pb = (mb0 + q) * 64 + rw + hrow * 8;
              if (pb >= kIrfPix) continue;
              const int by = pb / kIrfIW, bx = pb - by * kIrfIW;
              const bool outside = border && ((2 * oy0 - 1 + by) < 0 || (2 * ox0 - 1 + bx) < 0);
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                const int col = 8 * i + 2 * t;
                float2 o;
                o.x = fmaxf((em[q][4 * i + 2 * hrow] + ec[q][4 * i + 2 * hrow]) + b1[col], 0.f);
                o.y = fmaxf((em[q][4 * i + 2 * hrow + 1] + ec[q][4 * i + 2 * hrow + 1]) + b1[col + 1], 0.f);
                if (outside) o = make_float2(0.f, 0.f);
                *reinterpret_cast<float2*>(slab + irf_slab_off(pb, col >> 2) + (col & 3) * 4) = o;
              }
            }
        }
        irf_wg_sync(wg);  // the half-slab is complete; after the last one the box has been read by the whole warpgroup
        if (c == kIrfSlabs - 1 && h == 1 && wt == 0 && tile + stride < p.num_tiles) issue_box(tile + stride, wg);
        // ---- (2) depthwise 3x3 stride 2 + bd + ReLU -> A tile: thread = (4-channel group, 2 x 2 pixels) ----
        {
          // A quarter warp = 2 blocks x 4 channel groups; the two blocks are 4 output columns apart (A-tile rows R and
          // R + 4, box pixels pb and pb + 8), which keeps its 16-byte loads and stores conflict free.
          const int cg = wt & 3, blk = wt >> 2, k = blk & 7;
          const int oy_l = (blk >> 3) * 2, ox_l = 2 * ((k & 4) | ((k & 1) << 1) | ((k >> 1) & 1));
          const int ch4 = c * 8 + h * 4 + cg;  // float4 index of the channels among the 96
          const float4* w4 = reinterpret_cast<const float4*>(smem + kIrfOffDw) + ch4;  // tap t at + t * 24
          const float4 bias4 = reinterpret_cast<const float4*>(smem + kIrfOffBd)[ch4];
          float4 wk[3][3];
#pragma unroll
          for (int ky = 0; ky < 3; ++ky)
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) wk[ky][kx] = w4[(ky * 3 + kx) * (kIrfMid / 4)];
          float4 acc[2][2];
#pragma unroll
          for (int y = 0; y < 2; ++y)
#pragma unroll
            for (int x = 0; x < 2; ++x) acc[y][x] = bias4;
#pragma unroll
          for (int rr = 0; rr < 5; ++rr) {
            float4 v[5];
#pragma unroll
            for (int i = 0; i < 5; ++i)
              v[i] = *reinterpret_cast<const float4*>(slab + irf_slab_off((2 * oy_l + rr) * kIrfIW + 2 * ox_l + i, cg));
#pragma unroll
            for (int y = 0; y < 2; ++y) {
              const int ky = rr - 2 * y;
              if (ky >= 0 && ky < 3) {
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                  const float4 kw = wk[(ky >= 0 && ky < 3) ? ky : 0][kx];
#pragma unroll
                  for (int x = 0; x < 2; ++x) {
                    const float4 u = v[2 * x + kx];
                    acc[y][x].x = fmaf(u.x, kw.x, acc[y][x].x);
                    acc[y][x].y = fmaf(u.y, kw.y, acc[y][x].y);
                    acc[y][x].z = fmaf(u.z, kw.z, acc[y][x].z);
                    acc[y][x].w = fmaf(u.w, kw.w, acc[y][x].w);
                  }
                }
              }
            }
          }
#pragma unroll
          for (int y = 0; y < 2; ++y)
#pragma unroll
            for (int x = 0; x < 2; ++x) {
              float4 v = acc[y][x];
              v.x = fmaxf(v.x, 0.f);
              v.y = fmaxf(v.y, 0.f);
              v.z = fmaxf(v.z, 0.f);
              v.w = fmaxf(v.w, 0.f);
              const int R = (oy_l + y) * kIrfTW + ox_l + x;  // A-tile row = pixel inside the 8 x 16 tile
              *reinterpret_cast<float4*>(a2 + R * 128 + (((h * 4 + cg) ^ (R & 7)) << 4)) = v;
            }
        }
        irf_wg_sync(wg);  // the half-slab has been read (the next expand rewrites it); the A tile has these channels
      }
      // ---- (3) project: acc2 += dw_c * W2[:, c]^T over the tile's two 64-row halves ----
      const uint32_t bh = smem_u32(smem + kIrfOffW2) + c * 8192;  // [hi 32 rows ; lo 32 rows] x 128 B
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        uint32_t hi[4][4], lo[4][4];
        load_a_frags(a2, m * 64 + rw, t, hi, lo);
        wg_fence();
#pragma unroll
        for (int j = 0; j < 4; ++j) mma3<32>(acc2m[m], acc2c[m], hi[j], lo[j], bh + j * 32, bh + 4096 + j * 32);
        wg_commit();
        wg_wait();
      }
      // (the next slab's depthwise rewrites the A tile only after the next expand's warpgroup barrier)
    }

    const float* b2 = reinterpret_cast<const float*>(smem + kIrfOffB2);
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int hrow = 0; hrow < 2; ++hrow) {
        const int row = m * 64 + rw + hrow * 8;
        const int oy = oy0 + (row >> 4), ox = ox0 + (row & 15);
        float* dst = p.Y + (((long long)b * Ho + oy) * Wo + ox) * kIrfCout;
#pragma unroll
        for (int i = 0; i < kIrfCout / 8; ++i) {
          const int col = 8 * i + 2 * t;
          *reinterpret_cast<float2*>(dst + col) =
              make_float2((acc2m[m][4 * i + 2 * hrow] + acc2c[m][4 * i + 2 * hrow]) + b2[col],
                          (acc2m[m][4 * i + 2 * hrow + 1] + acc2c[m][4 * i + 2 * hrow + 1]) + b2[col + 1]);
        }
      }
  }
}

// X [B][H][W][16] -> Y [B][H/2][W/2][24] on min(tiles, num_sms) persistent CTAs.  Returns 0 on launch, 1 when the
// shape is not covered, < 0 on error.
inline int launch_irf_s2(cudaStream_t s, const float* X, float* Y, const float* image, int B, int H, int W, int num_sms) {
  if (!available()) return 1;
  const int Ho = H / 2, Wo = W / 2;
  if (H % 2 || W % 2 || Ho % kIrfTH || Wo % kIrfTW) return 1;
  if (attr_needed(reinterpret_cast<const void*>(irf_s2_fused_kernel))) {
    if (cudaFuncSetAttribute(irf_s2_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kIrfSmemBytes) != cudaSuccess)
      return -30;
  }
  CUtensorMap tmX;
  int r = make_tmap_nhwc(&tmX, X, (uint64_t)B, (uint64_t)H, (uint64_t)W, kIrfCin, kIrfCin, kIrfIW, kIrfIH,
                         CU_TENSOR_MAP_SWIZZLE_64B);
  if (r) return r;
  IrfParams p;
  p.Y = Y;
  p.image = image;
  p.B = B;
  p.H = H;
  p.W = W;
  p.tiles_x = Wo / kIrfTW;
  p.tiles_y = Ho / kIrfTH;
  p.num_tiles = B * p.tiles_x * p.tiles_y;
  const int grid = p.num_tiles < num_sms ? p.num_tiles : num_sms;
  if (launch_pdl(irf_s2_fused_kernel, dim3(grid), dim3(kIrfThreads), (size_t)kIrfSmemBytes, s, tmX, p) != cudaSuccess)
    return -31;
  return 0;
}

}  // namespace tc
}  // namespace fear
