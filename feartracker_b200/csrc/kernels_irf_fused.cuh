// irf_s2_fused_kernel -- the inverted-residual block xif2_0 of fbnet_c as ONE kernel (sm_90a):
//
//     Y = W2 * relu(dw3x3_s2(relu(W1 * X + b1)) + bd) + b2          16 -> 96 -> 96 -> 24 channels, 2x down
//
// (mobile_cv IRF block pw -> dw -> pwl as restated in oracle/fbnet_c.py:95-110; call site reference
// model_training/model/blocks.py:27-35).  Unfused this block is three kernels that write and re-read the 6x
// expanded tensor E = relu(W1 X + b1) and the depthwise map; here E and the depthwise output never leave the SM.
//
// One CTA (two warpgroups) per 8 x 16 output-pixel tile (= one M = 128 tile of the project GEMM):
//
//   load      the 17 x 33 input pixels the tile needs (halo of the stride-2 3x3 window; 561 pixels, 64 B each) go to
//             shared memory with coalesced 16-byte loads (zero outside the image), the packed weights image likewise.
//   per 32-channel slab c of the expanded tensor:
//     expand     nine 64-row blocks of the box, alternating between the warpgroups: D[64 x 32] = A * W1[c]^T as 3xTF32
//                wgmma with the A fragments split in registers; + b1, ReLU, zero outside the image (the depthwise conv
//                zero-pads E, and E(0) = relu(b1) != 0) -> 561 x 32-channel fp32 slab in shared memory.
//     depthwise  3x3 stride 2 out of that slab (same FMA order as the stand-alone depthwise kernels) -> + bd, ReLU ->
//                A tile of the project GEMM in the SWIZZLE_128B layout.
//     project    acc2[128 x 32] += dw_c * W2[:, c]^T, accumulators kept in registers across the slabs.
//   store     Y = acc2 + b2.
//
// All MMA orders / operand splits / epilogue additions replicate pw_tc_kernel (both go through tc::mma3), so the block
// is bit-identical to the three-kernel path (tests/test_gpu_tcgen05.py::test_fused_irf_block).
//
// smem: A2 16 KB | weights image 40.25 KB (W1 [hi|lo] rows, W2 [hi;lo] x 3 chunks, dw, biases) | input box 45 KB |
// slab 70.1 KB.
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
constexpr int kIrfXPitch = 20;                                  // floats per input-box row (16 + 4: conflict-free fragment loads)

// weights image (floats), copied verbatim into shared memory
constexpr int kIrfW1Floats = kIrfMid * 32;                        // [96 rows][hi 16 | lo 16], SWIZZLE_128B
constexpr int kIrfW2Floats = kIrfSlabs * 2 * kIrfCoutPad * 32;    // per chunk: [hi 32 rows ; lo 32 rows] x 32 k
constexpr int kIrfDwFloats = 9 * kIrfMid;
constexpr int kIrfImageFloats = kIrfW1Floats + kIrfW2Floats + kIrfDwFloats + kIrfMid + kIrfMid + kIrfCoutPad;

constexpr int kIrfOffA2 = 0;                                       // raw fp32 A tile of the project GEMM
constexpr int kIrfOffImg = 16384;
constexpr int kIrfOffW1 = kIrfOffImg;
constexpr int kIrfOffW2 = kIrfOffW1 + kIrfW1Floats * 4;
constexpr int kIrfOffDw = kIrfOffW2 + kIrfW2Floats * 4;
constexpr int kIrfOffB1 = kIrfOffDw + kIrfDwFloats * 4;
constexpr int kIrfOffBd = kIrfOffB1 + kIrfMid * 4;
constexpr int kIrfOffB2 = kIrfOffBd + kIrfMid * 4;
constexpr int kIrfOffX = ((kIrfOffB2 + kIrfCoutPad * 4 + 255) / 256) * 256;
constexpr int kIrfOffSlab = kIrfOffX + kIrfMB * 64 * kIrfXPitch * 4;
constexpr int kIrfSlabBytes = kIrfPix * 128;
constexpr int kIrfSmemBytes = kIrfOffSlab + kIrfSlabBytes + 1024 /*alignment slack*/;
static_assert(kIrfSmemBytes <= 232448, "fused IRF kernel exceeds the 227 KB shared-memory limit");
static_assert(kIrfOffW1 % 1024 == 0 && kIrfOffW2 % 1024 == 0, "swizzled weight tiles must be 1024-byte aligned");

struct IrfParams {
  const float* X;      // [B][H][W][16]
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

__global__ void __launch_bounds__(kIrfThreads, 1) irf_s2_fused_kernel(const IrfParams p) {
  extern __shared__ uint8_t irf_smem_raw[];
  uint8_t* smem = irf_smem_raw + ((1024u - (smem_u32(irf_smem_raw) & 1023u)) & 1023u);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  {  // weights image -> shared memory (constant data: may be read before the previous kernel has finished)
    const float4* src = reinterpret_cast<const float4*>(p.image);
    float4* dst = reinterpret_cast<float4*>(smem + kIrfOffImg);
    for (int i = threadIdx.x; i < kIrfImageFloats / 4; i += kIrfThreads) dst[i] = __ldg(src + i);
  }
  pdl_trigger();
  pdl_wait();  // X is written by the previous kernel in the stream

  const int Ho = p.H >> 1, Wo = p.W >> 1;
  const int tx = blockIdx.x % p.tiles_x, rest = blockIdx.x / p.tiles_x;
  const int b = rest / p.tiles_y, oy0 = (rest % p.tiles_y) * kIrfTH, ox0 = tx * kIrfTW;
  float* xs = reinterpret_cast<float*>(smem + kIrfOffX);
  for (int i = threadIdx.x; i < kIrfMB * 64 * 4; i += kIrfThreads) {  // (box pixel, 16-byte quarter)
    const int pb = i >> 2, j = i & 3;
    const int by = pb / kIrfIW, bx = pb - by * kIrfIW;
    const int iy = 2 * oy0 - 1 + by, ix = 2 * ox0 - 1 + bx;
    const bool ok = pb < kIrfPix && iy >= 0 && ix >= 0;
    const float4 v = ok ? __ldg(reinterpret_cast<const float4*>(p.X + (((long long)b * p.H + iy) * p.W + ix) * kIrfCin) + j)
                        : make_float4(0.f, 0.f, 0.f, 0.f);
    *reinterpret_cast<float4*>(xs + pb * kIrfXPitch + 4 * j) = v;
  }
  fence_proxy_async_smem();  // the tensor core reads W1 / W2 through the async proxy
  __syncthreads();

  const int wg = warp >> 2, g = lane >> 2, t = lane & 3;
  const int rw = (warp & 3) * 16 + g;  // this thread's first row inside a 64-row block (second: + 8)
  const bool border = (oy0 == 0) || (ox0 == 0);  // only these tiles have box pixels outside the image
  float acc2m[16], acc2c[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) acc2m[i] = acc2c[i] = 0.f;
  uint8_t* slab = smem + kIrfOffSlab;
  uint8_t* a2 = smem + kIrfOffA2;

  for (int c = 0; c < kIrfSlabs; ++c) {
    // ---- (1) expand: relu(X W1[c]^T + b1), zero outside the image -> slab ----
    // Slab layout: pixel pb = by * 33 + bx of the 17 x 33 box at byte pb * 128; the 16-byte chunk of channel group j
    // sits at position j ^ (bx & 7): a reader's chunk offset depends only on the box column.
    const uint32_t brow = smem_u32(smem + kIrfOffW1) + c * 4096;  // rows [32c, 32c + 32) of W1: [hi 64 B | lo 64 B]
    const float* b1 = reinterpret_cast<const float*>(smem + kIrfOffB1) + c * 32;
    for (int mb = wg; mb < kIrfMB; mb += 2) {
      uint32_t hi[2][4], lo[2][4];
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float v = xs[(mb * 64 + rw + (e & 1) * 8) * kIrfXPitch + 8 * j + 4 * (e >> 1) + t];
          const uint32_t h = __float_as_uint(v) & 0xFFFFE000u;
          hi[j][e] = h;
          lo[j][e] = __float_as_uint(v - __uint_as_float(h));
        }
      float em[16], ec[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) em[i] = ec[i] = 0.f;
      wg_fence();
#pragma unroll
      for (int j = 0; j < 2; ++j) mma3<32>(em, ec, hi[j], lo[j], brow + j * 32, brow + 64 + j * 32);
      wg_commit();
      wg_wait();
#pragma unroll
      for (int hrow = 0; hrow < 2; ++hrow) {
        const int pb = mb * 64 + rw + hrow * 8;
        if (pb >= kIrfPix) continue;
        const int by = pb / kIrfIW, bx = pb - by * kIrfIW;
        const bool outside = border && ((2 * oy0 - 1 + by) < 0 || (2 * ox0 - 1 + bx) < 0);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int col = 8 * i + 2 * t;
          float2 o;
          o.x = fmaxf((em[4 * i + 2 * hrow] + ec[4 * i + 2 * hrow]) + b1[col], 0.f);
          o.y = fmaxf((em[4 * i + 2 * hrow + 1] + ec[4 * i + 2 * hrow + 1]) + b1[col + 1], 0.f);
          if (outside) o = make_float2(0.f, 0.f);
          *reinterpret_cast<float2*>(slab + pb * 128 + ((((col >> 2) ^ (bx & 7))) << 4) + (col & 3) * 4) = o;
        }
      }
    }
    __syncthreads();  // the slab is complete
    // ---- (2) depthwise 3x3 stride 2 + bd + ReLU -> A tile of the project GEMM: thread = (4-channel group, 2 x 2 pixels) ----
    {
      const int cg = threadIdx.x & 7, blk = threadIdx.x >> 3;
      const int oy_l = (blk >> 3) * 2, ox_l = (blk & 7) * 2;
      const float4* w4 = reinterpret_cast<const float4*>(smem + kIrfOffDw) + c * 8 + cg;  // tap t at + t * 24
      const float4 bias4 = reinterpret_cast<const float4*>(smem + kIrfOffBd)[c * 8 + cg];
      float4 wk[3][3];
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) wk[ky][kx] = w4[(ky * 3 + kx) * (kIrfMid / 4)];
      const uint8_t* rows = slab + (2 * oy_l) * (kIrfIW * 128);
      float4 acc[2][2];
#pragma unroll
      for (int y = 0; y < 2; ++y)
#pragma unroll
        for (int x = 0; x < 2; ++x) acc[y][x] = bias4;
#pragma unroll
      for (int rr = 0; rr < 5; ++rr) {
        float4 v[5];
#pragma unroll
        for (int i = 0; i < 5; ++i) {
          const int bx = 2 * ox_l + i;
          v[i] = *reinterpret_cast<const float4*>(rows + rr * (kIrfIW * 128) + bx * 128 + ((cg ^ (bx & 7)) << 4));
        }
#pragma unroll
        for (int y = 0; y < 2; ++y) {
          const int ky = rr - 2 * y;
          if (ky >= 0 && ky < 3) {
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
              const float4 k = wk[(ky >= 0 && ky < 3) ? ky : 0][kx];
#pragma unroll
              for (int x = 0; x < 2; ++x) {
                const float4 u = v[2 * x + kx];
                acc[y][x].x = fmaf(u.x, k.x, acc[y][x].x);
                acc[y][x].y = fmaf(u.y, k.y, acc[y][x].y);
                acc[y][x].z = fmaf(u.z, k.z, acc[y][x].z);
                acc[y][x].w = fmaf(u.w, k.w, acc[y][x].w);
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
          *reinterpret_cast<float4*>(a2 + R * 128 + ((cg ^ (R & 7)) << 4)) = v;
        }
    }
    __syncthreads();  // the A tile is complete; everyone has left the slab
    // ---- (3) project: acc2 += dw_c * W2[:, c]^T ----
    {
      uint32_t hi[4][4], lo[4][4];
      load_a_frags(a2, wg * 64 + rw, t, hi, lo);
      const uint32_t bh = smem_u32(smem + kIrfOffW2) + c * 8192;  // [hi 32 rows ; lo 32 rows] x 128 B
      wg_fence();
#pragma unroll
      for (int j = 0; j < 4; ++j) mma3<32>(acc2m, acc2c, hi[j], lo[j], bh + j * 32, bh + 4096 + j * 32);
      wg_commit();
      wg_wait();
    }
    __syncthreads();  // the A tile has been read by every warp before the next slab rewrites it
  }

  const float* b2 = reinterpret_cast<const float*>(smem + kIrfOffB2);
#pragma unroll
  for (int hrow = 0; hrow < 2; ++hrow) {
    const int row = wg * 64 + rw + hrow * 8;
    const int oy = oy0 + (row >> 4), ox = ox0 + (row & 15);
    float* dst = p.Y + (((long long)b * Ho + oy) * Wo + ox) * kIrfCout;
#pragma unroll
    for (int i = 0; i < kIrfCout / 8; ++i) {
      const int col = 8 * i + 2 * t;
      *reinterpret_cast<float2*>(dst + col) = make_float2((acc2m[4 * i + 2 * hrow] + acc2c[4 * i + 2 * hrow]) + b2[col],
                                                          (acc2m[4 * i + 2 * hrow + 1] + acc2c[4 * i + 2 * hrow + 1]) + b2[col + 1]);
    }
  }
}

// X [B][H][W][16] -> Y [B][H/2][W/2][24].  Returns 0 on launch, 1 when the shape is not covered, < 0 on error.
inline int launch_irf_s2(cudaStream_t s, const float* X, float* Y, const float* image, int B, int H, int W) {
  if (!available()) return 1;
  const int Ho = H / 2, Wo = W / 2;
  if (H % 2 || W % 2 || Ho % kIrfTH || Wo % kIrfTW) return 1;
  if (attr_needed(reinterpret_cast<const void*>(irf_s2_fused_kernel))) {
    if (cudaFuncSetAttribute(irf_s2_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kIrfSmemBytes) != cudaSuccess)
      return -30;
  }
  IrfParams p;
  p.X = X;
  p.Y = Y;
  p.image = image;
  p.B = B;
  p.H = H;
  p.W = W;
  p.tiles_x = Wo / kIrfTW;
  p.tiles_y = Ho / kIrfTH;
  p.num_tiles = B * p.tiles_x * p.tiles_y;
  if (launch_pdl(irf_s2_fused_kernel, dim3(p.num_tiles), dim3(kIrfThreads), (size_t)kIrfSmemBytes, s, p) != cudaSuccess) return -31;
  return 0;
}

}  // namespace tc
}  // namespace fear
