// wgmma / TMA kernels of the FEAR-XS hot path (sm_90a only).
//
// corr_tc_kernel -- the pixel-wise template (x) search correlation (MobileCorrelation.forward's matmul,
// reference model_training/model/blocks.py:123) on the Hopper tensor cores:
//
//     s[b, p, k] = sum_c x[b, p, c] * z[b, k, c]        p in 256 search cells, k in 64 template cells, c in 256
//
// Channels-last operands are K-major GEMM operands as they lie in HBM: x = first 256 channels of the
// 320-channel concat buffer [B*256][320] (written there by the encode 1x1 conv), z = [Bz*64][256].
// The result goes straight into channels [256,320) of the same buffer, so the "torch.cat" of the
// reference costs nothing and the kernel moves exactly the algorithmic bytes (z + x in, s out).
//
// fp32 fidelity: tf32 keeps 11 significand bits, which fails the 1e-3 parity bar (SURVEY.md
// section 7.4), so each operand is split on the fly into tf32 (hi, lo) pairs and three products
// (hi*hi + hi*lo + lo*hi) accumulate in fp32 registers -- error ~1e-6, still far above the FFMA rate.
//
// pw_tc_kernel -- every 1x1 convolution as a 3xTF32 GEMM on the same pipeline (optionally with the preceding
// depthwise conv computed by its consumer warps).
//
// Common shape of the kernels: one CTA per 128-row tile = two consumer warpgroups of 64 rows each plus one TMA
// producer warp; K streamed in 32-channel chunks (one 128-byte swizzled row) through an mbarrier ring.  The A
// operand of every wgmma comes from REGISTERS: a consumer thread reads its fragment of the raw fp32 tile from
// shared memory once, splits it into (hi, lo) in registers and issues the three products against the weight tiles
// in shared memory, so no lo tile of the activations is ever written.
#pragma once
#include <cuda_runtime.h>
#include <stdlib.h>

#include <initializer_list>

#include "tc_common.cuh"

namespace fear {
namespace tc {

constexpr int kCorrChunk = 32;                 // channels per stage = one 128-byte swizzled row
constexpr int kCorrABytes = 128 * 128;         // [128 pixels][32 ch] fp32
constexpr int kCorrBBytes = 64 * 128;          // [64 template cells][32 ch] fp32
constexpr int kTcThreads = 288;                // 2 consumer warpgroups + the TMA producer warp
constexpr int kTcConsumers = 256;

// named barrier over the consumer warps (the producer warp never joins)
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// ------------------------------------------------------------------------------------------
// corr_tc_kernel: tile = half a frame (128 search cells) x 64 template cells, K = 256 in 8 chunks.  The template
// tile is an MMA operand in shared memory and is not pre-split: the consumers rewrite each landed tile as hi
// (low mantissa bits cleared, in place) and write lo right behind it.
// ------------------------------------------------------------------------------------------
constexpr int kCorrStages = 3;
constexpr int kCorrStageBytes = kCorrABytes + 2 * kCorrBBytes;  // x raw | z hi | z lo
constexpr int kCorrSmemBytes = kCorrStages * kCorrStageBytes + 1024 /*align*/ + 256 /*barriers*/;

__global__ void __launch_bounds__(kTcThreads, 1)
corr_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               float* __restrict__ cat, int z_mod) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kCorrStages * kCorrStageBytes);  // [stages] TMA landed
  uint64_t* empty = full + kCorrStages;                                                // [stages] 8 consumer warps done
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int kChunks = 256 / kCorrChunk;
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    for (int s = 0; s < kCorrStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_trigger();
  pdl_wait();
  const int frame = blockIdx.x >> 1, half = blockIdx.x & 1;
  const int arow = frame * 256 + half * 128;
  auto st_x = [&](int s) { return smem + s * kCorrStageBytes; };
  auto st_z = [&](int s) { return smem + s * kCorrStageBytes + kCorrABytes; };

  if (warp == 8) {
    if (lane == 0) {
      const int brow = z_mod ? (frame % z_mod) * 64 : 0;
      for (int c = 0; c < kChunks; ++c) {
        const int stage = c % kCorrStages;
        mbar_wait_backoff(&empty[stage], (uint32_t)(((c / kCorrStages) & 1) ^ 1));
        mbar_arrive_expect_tx(&full[stage], kCorrABytes + kCorrBBytes);
        tma_load_2d(st_x(stage), &tmA, &full[stage], c * kCorrChunk, arow);
        tma_load_2d(st_z(stage), &tmB, &full[stage], c * kCorrChunk, brow);
      }
    }
    return;
  }
  const int wg = warp >> 2, r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), t = lane & 3;
  float accm[32], accc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) accm[i] = accc[i] = 0.f;
  for (int c = 0; c < kChunks; ++c) {
    const int stage = c % kCorrStages;
    mbar_wait(&full[stage], (uint32_t)((c / kCorrStages) & 1));
    float4* zh = reinterpret_cast<float4*>(st_z(stage));
    float4* zl = reinterpret_cast<float4*>(st_z(stage) + kCorrBBytes);
#pragma unroll
    for (int i = 0; i < kCorrBBytes / 16 / kTcConsumers; ++i) {  // index-identical copy: the swizzle carries over
      const float4 v = zh[threadIdx.x + i * kTcConsumers];
      float4 h, l;
      split_tf32_trunc(v.x, h.x, l.x);
      split_tf32_trunc(v.y, h.y, l.y);
      split_tf32_trunc(v.z, h.z, l.z);
      split_tf32_trunc(v.w, h.w, l.w);
      zh[threadIdx.x + i * kTcConsumers] = h;
      zl[threadIdx.x + i * kTcConsumers] = l;
    }
    fence_proxy_async_smem();  // generic-proxy writes -> visible to the tensor core (async proxy)
    consumer_sync();
    uint32_t hi[4][4], lo[4][4];
    load_a_frags(st_x(stage), r0, t, hi, lo);
    const uint32_t bh = smem_u32(zh), bl = smem_u32(zl);
    wg_fence();
#pragma unroll
    for (int j = 0; j < 4; ++j) mma3<64>(accm, accc, hi[j], lo[j], bh + j * 32, bl + j * 32);
    wg_commit();
    wg_wait();
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[stage]);
  }
  float* out = cat + (long long)(arow + r0) * 320 + 256 + 2 * t;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    *reinterpret_cast<float2*>(out + 8 * i) = make_float2(accm[4 * i] + accc[4 * i], accm[4 * i + 1] + accc[4 * i + 1]);
    *reinterpret_cast<float2*>(out + 8 * 320 + 8 * i) =
        make_float2(accm[4 * i + 2] + accc[4 * i + 2], accm[4 * i + 3] + accc[4 * i + 3]);
  }
}

// ------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------
inline int init_pw();

// Per-device initialisation (called by fear_init with the device selected).
inline int init() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  cudaDeviceProp p;
  if (cudaGetDeviceProperties(&p, dev) != cudaSuccess) return -1;
  DeviceState& st = dev_state();
  st.num_sms = p.multiProcessorCount;
  st.inited = true;
  if (resolve_driver()) return 0;  // tensor-core / TMA path stays unavailable; the FFMA path still works
  if (cudaFuncSetAttribute(corr_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kCorrSmemBytes) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  if (init_pw()) return 0;
  st.tc_ready = true;
  return 0;
}

// cat holds `groups` consecutive [B][256][320] buffers (the cls and reg branches of the head): frame f of
// every group correlates with template f (or template 0 when Bz == 1).  One launch covers all groups.
inline int launch_corr(cudaStream_t s, const float* zt, int Bz, float* cat, int B, int groups) {
  if (!available()) return -20;
  CUtensorMap tmA, tmB;
  const int frames = B * groups;
  int r;
  r = make_tmap_2d(&tmA, cat, (uint64_t)frames * 256, 320, 320, 128, kCorrChunk);
  if (r) return r;
  r = make_tmap_2d(&tmB, zt, (uint64_t)Bz * 64, 256, 256, 64, kCorrChunk);
  if (r) return r;
  if (launch_pdl(corr_tc_kernel, dim3(frames * 2), dim3(kTcThreads), kCorrSmemBytes, s, tmA, tmB, cat, Bz == 1 ? 0 : B) !=
      cudaSuccess)
    return -23;
  return 0;
}

// ------------------------------------------------------------------------------------------
// pw_tc_kernel -- 1x1 convolution as a GEMM on wgmma:  C[M][N] = act(A[M][K] * W[N][K]^T + bias (+ R))
// A = channels-last activations (rows = pixels), W = BN-folded torch-native [Cout][Cin] weights,
// pre-split on the host into tf32 (hi, lo) copies; A is split in registers.  One CTA per (m_tile, n_tile) pair,
// n fastest; tile = 128 pixels x NT output channels.  TMA zero-fills the K tail (Cin not a multiple of 32),
// rows >= M and weight rows >= N; the epilogue clips the M / N tails.
// ------------------------------------------------------------------------------------------
struct PwParams {
  const float* bias;  // [N] or null
  const float* R;     // residual [M][ldr] or null
  float* C;
  int ldr, ldc;
  int M, N, num_n_tiles, num_chunks, last_ksteps, relu, stages, stage_bytes;
  // --- fused depthwise producer (DWK = 3 | 5): the A operand is dw(X) computed on the fly ---
  int dw_relu, dw_bias;  // ReLU / bias of the depthwise stage
  int box_bytes;         // bytes of one (tile rows + DWK - 1) x (map width + DWK - 1) x 32-channel input box
};

// DWK = 0: plain 1x1 conv.  DWK = 3 | 5 (option "fuse_dwpw", on by default; MW x MW maps with MW = 16 | 32, stride 1): the
// layer's input is the output of a DWK x DWK depthwise conv that is never materialised -- the producer TMA-loads the
// depthwise INPUT box of each (128-pixel tile, 32-channel chunk) with its zero-filled halo (tmA is then the 4-D NHWC
// map of X), the consumer warps run the depthwise conv out of shared memory (same FMA order as dw_tma_kernel => same
// fp32 values as the unfused pair of kernels) and write the A tile in the SWIZZLE_128B layout the fragment loads expect.
template <int NT, int DWK, int MW = 16>
__global__ void __launch_bounds__(kTcThreads, 1)
pw_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmWh,
             const __grid_constant__ CUtensorMap tmWl, const __grid_constant__ CUtensorMap tmDW,
             const __grid_constant__ CUtensorMap tmDB, const PwParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int S = p.stages;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + S * p.stage_bytes);
  uint64_t* empty = full + S;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int w_bytes = NT * 128;
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmWh);
    prefetch_tmap(&tmWl);
    for (int s = 0; s < S; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_trigger();  // the next kernel may start its prologue on SMs we have left
  pdl_wait();     // everything above overlapped the previous kernel's tail; its results are visible from here on

  const int mt = blockIdx.x / p.num_n_tiles, nt = blockIdx.x - mt * p.num_n_tiles;
  // stage: [A tile 16 KB][w_hi][w_lo] (+ fused depthwise: [input box][dw weights DWK*DWK x 32][dw bias 32])
  auto a_tile = [&](int s) { return smem + s * p.stage_bytes; };
  auto w_hi = [&](int s) { return smem + s * p.stage_bytes + kCorrABytes; };
  auto w_lo = [&](int s) { return w_hi(s) + w_bytes; };
  auto dw_box = [&](int s) { return w_lo(s) + w_bytes; };
  auto dw_wts = [&](int s) { return dw_box(s) + p.box_bytes; };
  auto dw_bia = [&](int s) { return dw_wts(s) + DWK * DWK * 128; };

  if (warp == 8) {
    if (lane == 0) {
      constexpr int th = 128 / MW, tpf = MW / th;  // tile rows, tiles per frame
      for (int c = 0; c < p.num_chunks; ++c) {
        const int stage = c % S;
        mbar_wait_backoff(&empty[stage], (uint32_t)(((c / S) & 1) ^ 1));
        if constexpr (DWK > 0) {
          mbar_arrive_expect_tx(&full[stage], 2 * w_bytes + p.box_bytes + DWK * DWK * 128 + (p.dw_bias ? 128 : 0));
          tma_load_4d(dw_box(stage), &tmA, &full[stage], c * 32, -(DWK / 2), (mt % tpf) * th - DWK / 2, mt / tpf);
          tma_load_2d(dw_wts(stage), &tmDW, &full[stage], c * 32, 0);
          if (p.dw_bias) tma_load_2d(dw_bia(stage), &tmDB, &full[stage], c * 32, 0);
        } else {
          mbar_arrive_expect_tx(&full[stage], kCorrABytes + 2 * w_bytes);
          tma_load_2d(a_tile(stage), &tmA, &full[stage], c * 32, mt * 128);
        }
        tma_load_2d(w_hi(stage), &tmWh, &full[stage], c * 32, nt * NT);
        tma_load_2d(w_lo(stage), &tmWl, &full[stage], c * 32, nt * NT);
      }
    }
    return;
  }

  const int wg = warp >> 2, r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), t = lane & 3;
  float accm[NT / 2], accc[NT / 2];
#pragma unroll
  for (int i = 0; i < NT / 2; ++i) accm[i] = accc[i] = 0.f;
  for (int c = 0; c < p.num_chunks; ++c) {
    const int stage = c % S;
    mbar_wait(&full[stage], (uint32_t)((c / S) & 1));
    if constexpr (DWK > 0) {
      // thread = (2-channel pair, 1 x 8 pixel strip); 16 strips cover the 128-pixel tile
      constexpr int K = DWK, TX = 8, NIN = TX + K - 1, IW = MW + K - 1, PXN = MW / TX;
      typedef unsigned long long U2;  // two packed fp32 channels
      const int c2 = threadIdx.x & 15, pos = threadIdx.x >> 4;
      const int x0 = (pos % PXN) * TX, y0 = pos / PXN;
      const U2* in2 = reinterpret_cast<const U2*>(dw_box(stage)) + (y0 * IW + x0) * 16 + c2;
      const U2* w2 = reinterpret_cast<const U2*>(dw_wts(stage)) + c2;
      const U2 bias2 = p.dw_bias ? reinterpret_cast<const U2*>(dw_bia(stage))[c2] : 0ull;
      U2 acc[TX];
#pragma unroll
      for (int i = 0; i < TX; ++i) acc[i] = bias2;
#pragma unroll
      for (int ky = 0; ky < K; ++ky) {
        U2 v[NIN];
#pragma unroll
        for (int i = 0; i < NIN; ++i) v[i] = in2[(ky * IW + i) * 16];
#pragma unroll
        for (int kx = 0; kx < K; ++kx) {
          const U2 k = w2[(ky * K + kx) * 16];
#pragma unroll
          for (int i = 0; i < TX; ++i) ffma2(acc[i], v[i + kx], k);
        }
      }
      uint8_t* at = a_tile(stage);
#pragma unroll
      for (int i = 0; i < TX; ++i) {
        float2 v = make_float2(__uint_as_float((uint32_t)acc[i]), __uint_as_float((uint32_t)(acc[i] >> 32)));
        if (p.dw_relu) {
          v.x = fmaxf(v.x, 0.f);
          v.y = fmaxf(v.y, 0.f);
        }
        const int R = y0 * MW + x0 + i;  // A-tile row = pixel inside the tile
        *reinterpret_cast<float2*>(at + R * 128 + (((c2 >> 1) ^ (R & 7)) << 4) + ((c2 & 1) << 3)) = v;
      }
      consumer_sync();  // the A tile of this chunk is complete (and every warp has left the previous chunk's)
    }
    uint32_t hi[4][4], lo[4][4];
    load_a_frags(a_tile(stage), r0, t, hi, lo);
    const uint32_t bh = smem_u32(w_hi(stage)), bl = smem_u32(w_lo(stage));
    const int ksteps = (c == p.num_chunks - 1) ? p.last_ksteps : 4;  // K tail: skip all-zero K-steps
    wg_fence();
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (j < ksteps) mma3<NT>(accm, accc, hi[j], lo[j], bh + j * 32, bl + j * 32);
    wg_commit();
    wg_wait();
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[stage]);
  }

  // epilogue: (main + corr) + bias (+ residual), ReLU, 8-byte stores (4 lanes cover one 32-byte sector)
  const int n0 = nt * NT + 2 * t;
#pragma unroll
  for (int hrow = 0; hrow < 2; ++hrow) {
    const long long grow = (long long)mt * 128 + r0 + hrow * 8;
    if (grow >= p.M) continue;
#pragma unroll
    for (int i = 0; i < NT / 8; ++i) {
      const int col = n0 + 8 * i;
      if (col >= p.N) continue;
      float2 o = make_float2(accm[4 * i + 2 * hrow] + accc[4 * i + 2 * hrow], accm[4 * i + 2 * hrow + 1] + accc[4 * i + 2 * hrow + 1]);
      float2 b = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + col)) : make_float2(0.f, 0.f);
      if (p.R) {
        const float2 rr = __ldg(reinterpret_cast<const float2*>(p.R + grow * p.ldr + col));
        b.x += rr.x;
        b.y += rr.y;
      }
      o.x += b.x;
      o.y += b.y;
      if (p.relu) {
        o.x = fmaxf(o.x, 0.f);
        o.y = fmaxf(o.y, 0.f);
      }
      *reinterpret_cast<float2*>(p.C + grow * p.ldc + col) = o;
    }
  }
}

constexpr int kPwMaxSmem = 232448 - 1024;  // 227 KB opt-in limit minus static/driver slack
constexpr int kPwMaxStages = 3;

// Output-channel tile for a layer: the layer is cut into the fewest tiles of <= 128 columns (two accumulators of
// NT / 2 registers per thread), each the narrowest instantiated width that covers its share; the last tile may hang
// over N (weight rows >= N are zero-filled by TMA, the store is clipped).
inline int pw_tile_n(int N) {
  const int Np = (N + 15) & ~15;
  const int tiles = (Np + 127) / 128;
  const int need = (Np + tiles - 1) / tiles;
  for (int nt : {16, 32, 48, 64, 96, 112, 128})
    if (nt >= need) return nt;
  return 0;
}

inline bool pw_supported(int cin, int cout) { return available() && cin % 8 == 0 && cout % 8 == 0; }

#define FEAR_PW_FOR_NT(X) X(16) X(32) X(48) X(64) X(96) X(112) X(128)

inline int init_pw() {
  cudaError_t e = cudaSuccess;
#define FEAR_PW_ATTR(NT_)                                                                                                  \
  if (e == cudaSuccess) e = cudaFuncSetAttribute(pw_tc_kernel<NT_, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPwMaxSmem);     \
  if (e == cudaSuccess) e = cudaFuncSetAttribute(pw_tc_kernel<NT_, 3, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPwMaxSmem); \
  if (e == cudaSuccess) e = cudaFuncSetAttribute(pw_tc_kernel<NT_, 5, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPwMaxSmem); \
  if (e == cudaSuccess) e = cudaFuncSetAttribute(pw_tc_kernel<NT_, 3, 32>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPwMaxSmem); \
  if (e == cudaSuccess) e = cudaFuncSetAttribute(pw_tc_kernel<NT_, 5, 32>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPwMaxSmem);
  FEAR_PW_FOR_NT(FEAR_PW_ATTR)
#undef FEAR_PW_ATTR
  if (e != cudaSuccess) {
    cudaGetLastError();
    return -1;
  }
  return 0;
}

// w_hi / w_lo: tf32-split copies of the [N][K] weights (device).
inline int launch_pw(cudaStream_t s, const float* A, int lda, const float* w_hi, const float* w_lo, const float* bias,
                     const float* R, int ldr, float* C, int ldc, int M, int N, int K, int relu) {
  if (!available()) return -20;
  PwParams p;
  p.bias = bias;
  p.R = R;
  p.C = C;
  p.ldr = ldr;
  p.ldc = ldc;
  p.M = M;
  p.N = N;
  p.num_chunks = (K + 31) / 32;
  const int NT = pw_tile_n(N);
  if (!NT) return -21;
  p.num_n_tiles = (((N + 15) & ~15) + NT - 1) / NT;
  p.last_ksteps = ((K - 32 * (p.num_chunks - 1)) + 7) / 8;
  p.relu = relu;
  p.dw_relu = p.dw_bias = p.box_bytes = 0;
  p.stage_bytes = kCorrABytes + 2 * NT * 128;
  p.stages = p.num_chunks < kPwMaxStages ? p.num_chunks : kPwMaxStages;
  CUtensorMap tmA, tmWh, tmWl;
  int r = make_tmap_2d(&tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, 128, 32);
  if (r) return r;
  r = make_tmap_2d(&tmWh, w_hi, (uint64_t)N, (uint64_t)K, (uint64_t)K, NT, 32);
  if (r) return r;
  r = make_tmap_2d(&tmWl, w_lo, (uint64_t)N, (uint64_t)K, (uint64_t)K, NT, 32);
  if (r) return r;
  const int tiles = ((M + 127) / 128) * p.num_n_tiles;
  const size_t smem_bytes = (size_t)p.stages * p.stage_bytes + 1024 + 256;
  cudaError_t e = cudaErrorInvalidValue;
  switch (NT) {
#define FEAR_PW_CASE(NT_)                                                                                                     \
  case NT_:                                                                                                                   \
    e = launch_pdl(pw_tc_kernel<NT_, 0>, dim3(tiles), dim3(kTcThreads), smem_bytes, s, tmA, tmWh, tmWl, tmA, tmA, p); \
    break;
    FEAR_PW_FOR_NT(FEAR_PW_CASE)
#undef FEAR_PW_CASE
  }
  return e == cudaSuccess ? 0 : -23;
}

// Depthwise-fused GEMM (option "fuse_dwpw", default on; tests/test_gpu_parity.py): 1x1 conv whose input is dw_k x dw_k depthwise(X)
// (+bias, ReLU), X = [B][map_w][map_w][K] channels-last, stride 1.  out = act(dw(X) * W^T + bias (+R)).
// Returns 1 when the shape is not covered (caller runs the two kernels separately).
inline int launch_pw_dw(cudaStream_t s, const float* X, int B, int dw_k, const float* dw_w, const float* dw_b, int dw_relu,
                        const float* w_hi, const float* w_lo, const float* bias, const float* R, int ldr, float* C,
                        int ldc, int N, int K, int relu, int map_w = 16) {
  if (!available()) return -20;
  if ((dw_k != 3 && dw_k != 5) || K % 4 || (map_w != 16 && map_w != 32)) return 1;
  PwParams p;
  const int M = B * map_w * map_w;
  p.bias = bias;
  p.R = R;
  p.C = C;
  p.ldr = ldr;
  p.ldc = ldc;
  p.M = M;
  p.N = N;
  p.num_chunks = (K + 31) / 32;
  const int NT = pw_tile_n(N);
  if (!NT) return 1;
  p.num_n_tiles = (((N + 15) & ~15) + NT - 1) / NT;
  p.last_ksteps = ((K - 32 * (p.num_chunks - 1)) + 7) / 8;
  p.relu = relu;
  p.dw_relu = dw_relu;
  p.dw_bias = dw_b != nullptr;
  const int ih = 128 / map_w + dw_k - 1, iw = map_w + dw_k - 1;
  p.box_bytes = ih * iw * 128;
  p.stage_bytes = (kCorrABytes + 2 * NT * 128 + p.box_bytes + dw_k * dw_k * 128 + 128 + 1023) & ~1023;
  p.stages = p.num_chunks < 2 ? 1 : 2;
  const size_t smem_bytes = (size_t)p.stages * p.stage_bytes + 1024 + 256;
  if ((int)smem_bytes > kPwMaxSmem) return 1;
  CUtensorMap tmX, tmWh, tmWl, tmDW, tmDB;
  int r = make_tmap_nhwc(&tmX, X, (uint64_t)B, (uint64_t)map_w, (uint64_t)map_w, (uint64_t)K, 32, iw, ih);
  if (r) return r;
  r = make_tmap_2d(&tmWh, w_hi, (uint64_t)N, (uint64_t)K, (uint64_t)K, NT, 32);
  if (r) return r;
  r = make_tmap_2d(&tmWl, w_lo, (uint64_t)N, (uint64_t)K, (uint64_t)K, NT, 32);
  if (r) return r;
  r = make_tmap_2d_plain(&tmDW, dw_w, (uint64_t)dw_k * dw_k, (uint64_t)K, dw_k * dw_k, 32);
  if (r) return r;
  if (dw_b) {
    r = make_tmap_2d_plain(&tmDB, dw_b, 1, (uint64_t)K, 1, 32);
    if (r) return r;
  } else {
    tmDB = tmDW;
  }
  const int tiles = (M / 128) * p.num_n_tiles;
  cudaError_t e = cudaErrorInvalidValue;
#define FEAR_PW_DW_LAUNCH(NT_, K_, MW_) \
  e = launch_pdl(pw_tc_kernel<NT_, K_, MW_>, dim3(tiles), dim3(kTcThreads), smem_bytes, s, tmX, tmWh, tmWl, tmDW, tmDB, p)
  switch (NT) {
#define FEAR_PW_CASE(NT_)                                \
  case NT_:                                              \
    if (map_w == 16) {                                   \
      if (dw_k == 5) FEAR_PW_DW_LAUNCH(NT_, 5, 16);      \
      else FEAR_PW_DW_LAUNCH(NT_, 3, 16);                \
    } else {                                             \
      if (dw_k == 5) FEAR_PW_DW_LAUNCH(NT_, 5, 32);      \
      else FEAR_PW_DW_LAUNCH(NT_, 3, 32);                \
    }                                                    \
    break;
    FEAR_PW_FOR_NT(FEAR_PW_CASE)
#undef FEAR_PW_CASE
  }
#undef FEAR_PW_DW_LAUNCH
  return e == cudaSuccess ? 0 : -23;
}

}  // namespace tc
}  // namespace fear
