// Fused stem + xif1_0 kernel (CUDA cores, weights in the constant bank, input patch by TMA).  sm_90a.
#pragma once
#include "kernels_ffma.cuh"
#include "tc_common.cuh"

namespace fear {

// ------------------------------------------------------------------------------------------
// Fused stem + first IRF block:  conv3x3 s2 (3 -> 16) + ReLU  ->  xif1_0 = dw3x3 + ReLU -> 1x1 (16 -> 16)
// + residual.  (fbnet_c xif0_0 + xif1_0; reference call site fear_net.py:58-61.)
//
// Unfused, these four kernels stream 1.7 GB per 256-frame step through HBM (the 128x128x16 stem map is
// written once and read three times, the depthwise map once each way).  Here a CTA owns a 16 x 32 tile of
// the block's output: it stages the 37 x 69 x 3 input patch in shared memory, computes the 18 x 34 stem
// pixels the depthwise conv needs (halo recomputed: 1.2x stem FLOPs), keeps them in shared memory, and runs
// dw + pw + residual from there, so HBM sees the image once and the block output once.
// Every accumulation is done in the order of the unfused kernels (stem_conv3x3s2_kernel, dw_conv_*_kernel,
// pw_small_kernel): the results are bit-identical.
// Each thread works on 2 horizontally adjacent pixels x 16 channels so that one weight fetch from shared
// memory feeds 32 FMAs (the loops are FMA-issue bound, not LDS bound).
// ------------------------------------------------------------------------------------------
constexpr int kFsTH = 16, kFsTW = 32;                  // output tile
constexpr int kFsSH = kFsTH + 2, kFsSW = kFsTW + 2;    // stem tile incl. the depthwise halo: 18 x 34
constexpr int kFsPH = 2 * kFsSH + 1;                   // input patch rows: 37
constexpr int kFsPW = 2 * kFsSW + 1;                   // input patch cols: 69
constexpr int kFsPP = 72;                              // patch row pitch (floats; 16-byte aligned rows)
constexpr int kFsPitch = 20;                           // floats per stem pixel in smem (16 + 4 pad)
// Stem tile addressing.  A thread owns two horizontally adjacent pixels, so the lanes of a quarter warp touch pixels q, q + 2,
// ... q + 14: with a 5-quad pixel pitch the 16-byte chunk c of those pixels falls on bank quads (2 j + c) mod 8 -- lanes j and
// j + 4 collide (ncu: 2 wavefronts per ideal wavefront on every STS.128 / LDS.128 of the tile, L1/TEX 74 % busy).  Storing
// chunk c of pixel q at slot c ^ ((q >> 3) & 1) separates them: conflict free for writes and reads.  Even chunks sit at
// base + 16 s + 16 c, odd chunks at base - 16 s + 16 c (s = the swizzle bit), i.e. two base pointers per pixel.
struct FsPix {
  const float* e;  // base for chunks 0, 2
  const float* o;  // base for chunks 1, 3
};
__device__ __forceinline__ FsPix fs_pix(const float* stem, int q) {
  const int s4 = ((q >> 3) & 1) << 2;  // swizzle offset in floats
  const float* b = stem + q * kFsPitch;
  return {b + s4, b - s4};
}
__device__ __forceinline__ float4 fs_ld(const FsPix& p, int c4) {
  return *reinterpret_cast<const float4*>(((c4 & 1) ? p.o : p.e) + 4 * c4);
}
__device__ __forceinline__ void fs_st(const FsPix& p, int c4, float4 v) {
  *reinterpret_cast<float4*>(const_cast<float*>(((c4 & 1) ? p.o : p.e) + 4 * c4)) = v;
}
constexpr int kFsThreads = 320;
// All weights of the fused kernel (3.4 KB), passed BY VALUE as a __grid_constant__ kernel parameter: they live in
// the constant bank, every index below is a compile-time constant after unrolling, so each FFMA takes its weight
// as a c[0][imm] operand -- no shared-memory broadcast (an LDS costs one LSU wavefront per 4 bytes even when all
// lanes read the same address, which made the smem-weight version LSU-bound at ~25 % of the FMA rate), no registers.
struct FsWeights {
  float sw[27 * 16];  // stem [tap][c]
  float sb[16];
  float dw[9 * 16];   // xif1_0 depthwise [tap][c]
  float db[16];
  float pw[16 * 16];  // xif1_0 project, transposed to [k][o]
  float pb[16];
};
constexpr int kFsSmemBytes = 4 * (3 * kFsPH * kFsPP + kFsSH * kFsSW * kFsPitch) + 128;

constexpr int kFsRawPitch = 224;  // bytes per uint8 patch row: 4 lead-in bytes + 70 pixels x 3 channels, rounded up to 16

template <bool U8>
__global__ void __launch_bounds__(kFsThreads, 2)
stem_xif1_fused_kernel(const __grid_constant__ CUtensorMap tmImg, float* __restrict__ out, int H, int W, StemNorm nrm,
                       const __grid_constant__ FsWeights wts) {
  extern __shared__ uint8_t fs_smem_raw[];
  __shared__ uint64_t bar;
  float* patch = reinterpret_cast<float*>(fs_smem_raw + ((128u - (tc::smem_u32(fs_smem_raw) & 127u)) & 127u));  // [3][37][72]
  float* stem = patch + 3 * kFsPH * kFsPP;                                                                 // [18*34][20]
  uint8_t* raw = reinterpret_cast<uint8_t*>(stem) + 32;  // uint8 landing zone [37][208] (128-byte aligned), dead before phase 2

  const int Hs = H >> 1, Ws = W >> 1;
  const int tiles_x = Ws / kFsTW, tiles_y = Hs / kFsTH;
  int t = blockIdx.x;
  const int tx = t % tiles_x;
  t /= tiles_x;
  const int ty = t % tiles_y;
  const int b = t / tiles_y;
  const int oy0 = ty * kFsTH, ox0 = tx * kFsTW;  // tile origin at stem resolution
  // patch origin in the image.  The conv needs columns from 2*ox0 - 3; the box starts one column earlier so that the
  // innermost TMA coordinate is 16-byte aligned (floats: column % 4 == 0; uint8: byte 6*ox0 - 16).
  const int py0 = 2 * oy0 - 3, px0 = 2 * ox0 - 4;

  // ---- phase 1: one TMA box brings the input patch in; everything outside the image is zero-filled by the TMA
  //      unit (= the stem conv's padding).  (The first version gathered the patch with ~24 scalar loads per
  //      thread and spent 58 % of its stall samples waiting on them.)
  if (threadIdx.x == 0) {
    tc::mbar_init(&bar, 1);
    tc::fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (U8) {
      tc::mbar_arrive_expect_tx(&bar, kFsPH * kFsRawPitch);
      tc::tma_load_3d(raw, &tmImg, &bar, 6 * ox0 - 16, py0, b);
    } else {
      tc::mbar_arrive_expect_tx(&bar, 3 * kFsPH * kFsPP * 4);
      tc::tma_load_3d(patch, &tmImg, &bar, px0, py0, b * 3);
    }
  }
  tc::mbar_wait(&bar, 0);
  if (U8) {
    // uint8 HWC bytes -> normalised float planes; pixels outside the image stay exactly 0 (not (0 - mean) / std).
    // One (row, 4-pixel group) per thread and iteration: the group's 12 bytes are three aligned 32-bit loads, a byte becomes
    // a float without I2F (2^23 | b, minus 2^23: exact), and each channel's 4 values leave as one STS.128.  (The first
    // version -- one pixel per iteration, LDS.U8 + I2F -- took a third of this kernel: ncu put 74 % of its stall samples here.)
    constexpr int kGroups = (kFsPW + 1 + 3) / 4;  // 18 groups cover patch columns 0..71 (70, 71 are padding)
    for (int it = threadIdx.x; it < kFsPH * kGroups; it += kFsThreads) {
      const int pr = it / kGroups, g = it - pr * kGroups;
      const int iy = py0 + pr;
      const bool row_ok = iy >= 0 && iy < H;
      const uint32_t* src = reinterpret_cast<const uint32_t*>(raw + pr * kFsRawPitch + 4 + 12 * g);
      const uint32_t w[3] = {src[0], src[1], src[2]};
      float v[3][4];
#pragma unroll
      for (int px = 0; px < 4; ++px) {
        const int ix = px0 + 4 * g + px;
        const bool ok = row_ok && ix >= 0 && ix < W;
#pragma unroll
        for (int ci = 0; ci < 3; ++ci) {
          const int idx = 3 * px + ci;  // byte inside the 12-byte group
          const uint32_t byte = (w[idx >> 2] >> (8 * (idx & 3))) & 0xffu;
          const float f = __fsub_rn(__uint_as_float(0x4B000000u | byte), 8388608.0f);  // == (float)byte
          v[ci][px] = ok ? __fmul_rn(__fsub_rn(f, nrm.mean[ci]), nrm.inv[ci]) : 0.f;
        }
      }
#pragma unroll
      for (int ci = 0; ci < 3; ++ci)
        *reinterpret_cast<float4*>(patch + (ci * kFsPH + pr) * kFsPP + 4 * g) = make_float4(v[ci][0], v[ci][1], v[ci][2], v[ci][3]);
    }
    __syncthreads();
  }

  // ---- phase 2: stem conv for the 18 x 34 pixels (2 per thread), ReLU, zero outside the map ----
  if (threadIdx.x < kFsSH * (kFsSW / 2)) {
    const int sy = threadIdx.x / (kFsSW / 2), j = threadIdx.x % (kFsSW / 2);
    float a0[16], a1[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) a0[c] = a1[c] = wts.sb[c];
#pragma unroll
    for (int ci = 0; ci < 3; ++ci) {
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
        const float* row = patch + (ci * kFsPH + 2 * sy + ky) * kFsPP + 4 * j;
        const float4 q = *reinterpret_cast<const float4*>(row);  // patch columns 4j .. 4j+3 (the taps start at 4j+1)
        const float2 e = *reinterpret_cast<const float2*>(row + 4);
        const float v0[3] = {q.y, q.z, q.w};
        const float v1[3] = {q.w, e.x, e.y};
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
#pragma unroll
          for (int c = 0; c < 16; ++c) {
            const float wv = wts.sw[(ci * 9 + ky * 3 + kx) * 16 + c];
            a0[c] = fmaf(v0[kx], wv, a0[c]);
            a1[c] = fmaf(v1[kx], wv, a1[c]);
          }
        }
      }
    }
    const int gy = oy0 - 1 + sy;
    const int gx = ox0 - 1 + 2 * j;
    const bool in_y = gy >= 0 && gy < Hs;
    const bool in0 = in_y && gx >= 0 && gx < Ws, in1 = in_y && gx + 1 >= 0 && gx + 1 < Ws;
    const FsPix d0 = fs_pix(stem, sy * kFsSW + 2 * j), d1 = fs_pix(stem, sy * kFsSW + 2 * j + 1);
#pragma unroll
    for (int c4 = 0; c4 < 4; ++c4) {
      fs_st(d0, c4,
            in0 ? make_float4(fmaxf(a0[4 * c4], 0.f), fmaxf(a0[4 * c4 + 1], 0.f), fmaxf(a0[4 * c4 + 2], 0.f),
                              fmaxf(a0[4 * c4 + 3], 0.f))
                : make_float4(0.f, 0.f, 0.f, 0.f));
      fs_st(d1, c4,
            in1 ? make_float4(fmaxf(a1[4 * c4], 0.f), fmaxf(a1[4 * c4 + 1], 0.f), fmaxf(a1[4 * c4 + 2], 0.f),
                              fmaxf(a1[4 * c4 + 3], 0.f))
                : make_float4(0.f, 0.f, 0.f, 0.f));
    }
  }
  __syncthreads();

  // ---- phase 3: depthwise 3x3 + ReLU, 1x1 16 -> 16, + residual; 2 output pixels per thread ----
  if (threadIdx.x < kFsTH * (kFsTW / 2)) {
    const int oy = threadIdx.x / (kFsTW / 2), j = threadIdx.x % (kFsTW / 2);
    float d0[16], d1[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) d0[c] = d1[c] = wts.db[c];
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
      float4 x[4][4];  // 4 stem columns x 16 channels of this row
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const FsPix px = fs_pix(stem, (oy + ky) * kFsSW + 2 * j + i);
#pragma unroll
        for (int c4 = 0; c4 < 4; ++c4) x[i][c4] = fs_ld(px, c4);
      }
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
#pragma unroll
        for (int c4 = 0; c4 < 4; ++c4) {
          const float* k = wts.dw + (ky * 3 + kx) * 16 + 4 * c4;
          d0[4 * c4] = fmaf(x[kx][c4].x, k[0], d0[4 * c4]);
          d0[4 * c4 + 1] = fmaf(x[kx][c4].y, k[1], d0[4 * c4 + 1]);
          d0[4 * c4 + 2] = fmaf(x[kx][c4].z, k[2], d0[4 * c4 + 2]);
          d0[4 * c4 + 3] = fmaf(x[kx][c4].w, k[3], d0[4 * c4 + 3]);
          d1[4 * c4] = fmaf(x[kx + 1][c4].x, k[0], d1[4 * c4]);
          d1[4 * c4 + 1] = fmaf(x[kx + 1][c4].y, k[1], d1[4 * c4 + 1]);
          d1[4 * c4 + 2] = fmaf(x[kx + 1][c4].z, k[2], d1[4 * c4 + 2]);
          d1[4 * c4 + 3] = fmaf(x[kx + 1][c4].w, k[3], d1[4 * c4 + 3]);
        }
      }
    }
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      d0[c] = fmaxf(d0[c], 0.f);
      d1[c] = fmaxf(d1[c], 0.f);
    }
    float p0[16], p1[16];
#pragma unroll
    for (int o = 0; o < 16; ++o) p0[o] = p1[o] = wts.pb[o];
#pragma unroll
    for (int k = 0; k < 16; ++k) {
#pragma unroll
      for (int o = 0; o < 16; ++o) {
        const float wv = wts.pw[k * 16 + o];
        p0[o] = fmaf(d0[k], wv, p0[o]);
        p1[o] = fmaf(d1[k], wv, p1[o]);
      }
    }
    const FsPix r0 = fs_pix(stem, (oy + 1) * kFsSW + 2 * j + 1), r1 = fs_pix(stem, (oy + 1) * kFsSW + 2 * j + 2);
    float4* o0 = reinterpret_cast<float4*>(out + (((long long)b * Hs + oy0 + oy) * Ws + ox0 + 2 * j) * 16);
#pragma unroll
    for (int o4 = 0; o4 < 4; ++o4) {
      const float4 q0 = fs_ld(r0, o4), q1 = fs_ld(r1, o4);
      o0[o4] = make_float4(p0[4 * o4] + q0.x, p0[4 * o4 + 1] + q0.y, p0[4 * o4 + 2] + q0.z, p0[4 * o4 + 3] + q0.w);
      o0[4 + o4] = make_float4(p1[4 * o4] + q1.x, p1[4 * o4 + 1] + q1.y, p1[4 * o4 + 2] + q1.z, p1[4 * o4 + 3] + q1.w);
    }
  }
}

}  // namespace fear
