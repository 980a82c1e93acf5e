// wgmma / TMA kernels of the FEAR-XS hot path (sm_90a only).
//
// corr_tc_kernel -- the pixel-wise template (x) search correlation (MobileCorrelation.forward's matmul,
// reference model_training/model/blocks.py:123) on the Hopper tensor cores:
//
//     s[b, p, k] = sum_c x[b, p, c] * z[b, k, c]        p in P search cells, k in 64 template cells, c in 256
//
// P = s * s is the score map (s = 16 for 256 x 256 searches, any s in [1, 16] for searches of side 16 s).
// Channels-last operands are K-major GEMM operands as they lie in HBM: x = first 256 channels of the
// 320-channel concat buffer [B*P][320] (written there by the encode 1x1 conv), z = [Bz*64][256].
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
// corr_tc_kernel: tile = 128 search cells of one frame x 64 template cells, K = 256 in 8 chunks; ceil(P / 128) tiles
// per frame (two at P = 256), so a tile never straddles two frames.  The search operand is read through a 3-D map
// (channel, cell, frame): TMA zero-fills the cells >= P of a frame's last tile and the epilogue does not store them.
// The template tile is an MMA operand in shared memory and is not pre-split: the consumers rewrite each landed tile as
// hi (low mantissa bits cleared, in place) and write lo right behind it.
// ------------------------------------------------------------------------------------------
constexpr int kCorrStages = 3;
constexpr int kCorrStageBytes = kCorrABytes + 2 * kCorrBBytes;  // x raw | z hi | z lo
constexpr int kCorrSmemBytes = kCorrStages * kCorrStageBytes + 1024 /*align*/ + 256 /*barriers*/;

__global__ void __launch_bounds__(kTcThreads, 1)
corr_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               float* __restrict__ cat, int z_mod, int P) {
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
  const int tiles = (P + 127) >> 7;
  const int frame = blockIdx.x / tiles, cell0 = (blockIdx.x - frame * tiles) * 128;
  auto st_x = [&](int s) { return smem + s * kCorrStageBytes; };
  auto st_z = [&](int s) { return smem + s * kCorrStageBytes + kCorrABytes; };

  if (warp == 8) {
    if (lane == 0) {
      const int brow = z_mod ? (frame % z_mod) * 64 : 0;
      for (int c = 0; c < kChunks; ++c) {
        const int stage = c % kCorrStages;
        mbar_wait_backoff(&empty[stage], (uint32_t)(((c / kCorrStages) & 1) ^ 1));
        mbar_arrive_expect_tx(&full[stage], kCorrABytes + kCorrBBytes);
        tma_load_3d(st_x(stage), &tmA, &full[stage], c * kCorrChunk, cell0, frame);
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
  const int cell = cell0 + r0;  // this thread's rows: cell and cell + 8
  float* out = cat + ((long long)frame * P + cell) * 320 + 256 + 2 * t;
  if (cell < P) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      *reinterpret_cast<float2*>(out + 8 * i) = make_float2(accm[4 * i] + accc[4 * i], accm[4 * i + 1] + accc[4 * i + 1]);
  }
  if (cell + 8 < P) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
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

// cat holds `groups` consecutive [B][P][320] buffers (the cls and reg branches of the head): frame f of
// every group correlates with template f (or template 0 when Bz == 1).  One launch covers all groups.
inline int launch_corr(cudaStream_t s, const float* zt, int Bz, float* cat, int B, int groups, int P) {
  if (!available()) return -20;
  if (P < 1 || P > 256) return -21;
  CUtensorMap tmA, tmB;
  const int frames = B * groups;
  int r;
  r = make_tmap_3d(&tmA, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, cat, 320, (uint64_t)P, (uint64_t)frames, 320 * 4,
                   (uint64_t)P * 320 * 4, kCorrChunk, 128, 1, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
  if (r) return r;
  r = make_tmap_2d(&tmB, zt, (uint64_t)Bz * 64, 256, 256, 64, kCorrChunk);
  if (r) return r;
  if (launch_pdl(corr_tc_kernel, dim3(frames * ((P + 127) / 128)), dim3(kTcThreads), kCorrSmemBytes, s, tmA, tmB, cat,
                 Bz == 1 ? 0 : B, P) != cudaSuccess)
    return -23;
  return 0;
}

// ------------------------------------------------------------------------------------------
// pw_tc_kernel -- 1x1 convolution as a GEMM on wgmma:  C[M][N] = act(A[M][K] * W[N][K]^T + bias (+ R))
// A = channels-last activations (rows = pixels), W = BN-folded torch-native [Cout][Cin] weights,
// pre-split on the host into tf32 (hi, lo) copies; A is split in registers.  Tile = 128 pixels x NT output channels;
// tile index = m_tile * num_n_tiles + n_tile (n fastest: the n-tiles of one m-tile run together and share A in L2).
// TMA zero-fills the K tail (Cin not a multiple of 32), rows >= M and weight rows >= N; the epilogue clips the M / N tails.
// ------------------------------------------------------------------------------------------
struct PwParams {
  const float* bias;  // [N] or null
  const float* R;     // residual [M][ldr] or null
  float* C;
  int ldr, ldc;
  int M, N, num_n_tiles, num_tiles, num_chunks, last_ksteps, relu, stages, stage_bytes;
  // --- fused depthwise producer (DWK = 3 | 5): the A operand is dw(X) computed on the fly ---
  int dw_relu, dw_bias;  // ReLU / bias of the depthwise stage
  int box_bytes;         // bytes of one (tile rows + DWK - 1) x (map width + DWK - 1) x 32-channel input box
  int tma_store;         // pw_tc_kernel stores C by TMA (tmC); 0 when C or ldc is not 16-byte aligned
};

// Warp-specialised CTA: warpgroup 0 is the TMA producer and keeps kPwProducerRegs registers per thread, warpgroups 1-2
// are the consumers and take the rest: 128 * 40 + 256 * 232 = 64 512 of the SM's 65 536.  The consumers' budget holds
// 128 accumulators (NT = 128) plus the A fragments of two chunks whose MMA groups are in flight at once.
constexpr int kPwThreads = 384;
constexpr int kPwProducerRegs = 40, kPwConsumerRegs = 232;

// The 3xTF32 products of one 32-channel chunk, KS K steps in K order (KS < 4 only for the K tail, whose all-zero
// K steps are skipped).  One straight-line issue sequence per KS: no wgmma sits behind a per-step branch.
template <int NT, int KS>
__device__ __forceinline__ void mma3_chunk(float* accm, float* accc, const uint32_t (&hi)[4][4], const uint32_t (&lo)[4][4],
                                           uint32_t bh, uint32_t bl) {
#pragma unroll
  for (int j = 0; j < KS; ++j) mma3<NT>(accm, accc, hi[j], lo[j], bh + j * 32, bl + j * 32);
}

// Depthwise K x K conv (stride 1, MW x MW map) of one 32-channel chunk of a 128-pixel tile, from the landed input box
// (halo included) into the A tile in the SWIZZLE_128B layout the fragment loads expect.  ct = consumer thread (0..255)
// = (2-channel pair, 1 x 8 pixel strip); 16 strips cover the tile.  Same FMA order as dw_tma_kernel.
template <int K, int MW>
__device__ __forceinline__ void dw_chunk(const uint8_t* box, const uint8_t* wts, const uint8_t* bia, uint8_t* at, int ct,
                                         int dw_bias, int dw_relu) {
  constexpr int TX = 8, NIN = TX + K - 1, IW = MW + K - 1, PXN = MW / TX;
  typedef unsigned long long U2;  // two packed fp32 channels
  const int c2 = ct & 15, pos = ct >> 4;
  const int x0 = (pos % PXN) * TX, y0 = pos / PXN;
  const U2* in2 = reinterpret_cast<const U2*>(box) + (y0 * IW + x0) * 16 + c2;
  const U2* w2 = reinterpret_cast<const U2*>(wts) + c2;
  const U2 bias2 = dw_bias ? reinterpret_cast<const U2*>(bia)[c2] : 0ull;
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
#pragma unroll
  for (int i = 0; i < TX; ++i) {
    float2 v = make_float2(__uint_as_float((uint32_t)acc[i]), __uint_as_float((uint32_t)(acc[i] >> 32)));
    if (dw_relu) {
      v.x = fmaxf(v.x, 0.f);
      v.y = fmaxf(v.y, 0.f);
    }
    const int R = y0 * MW + x0 + i;  // A-tile row = pixel inside the tile
    *reinterpret_cast<float2*>(at + R * 128 + (((c2 >> 1) ^ (R & 7)) << 4) + ((c2 & 1) << 3)) = v;
  }
}

// Epilogue of one tile: (main + corr) + bias (+ residual), ReLU, 8-byte stores straight from the accumulator registers
// (4 lanes cover one 32-byte sector).
template <int NT>
__device__ __forceinline__ void pw_epilogue(const PwParams& p, const float* accm, const float* accc, int mt, int nt, int r0,
                                            int t) {
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

// Epilogue of one consumer warpgroup's 64 rows through shared memory, for pw_tc_kernel.  First the same arithmetic as
// pw_epilogue, in place in accm, so every bias and residual load is issued before the first barrier.  Then slabs of 32
// columns (two [64 rows][16 columns] boxes, SWIZZLE_64B, so the 8-byte writes of a warp take the minimum two wavefronts),
// each stored by TMA from one elected thread.  Slabs alternate between two buffers and the tile's last slab goes to
// `last`; a buffer is rewritten only once the store issued from it two slabs ago has read it (wait_group.read 1).
// Nothing waits for the global writes: the warpgroup goes on to the next tile's MMAs.  TMA clips the M and N tails at
// the tensor's bounds.
constexpr int kPwSlabBytes = 64 * 128;  // one warpgroup's 64 rows x 32 columns
constexpr int kPwBoxBytes = 64 * 64;    // one TMA store box: 64 rows x 16 columns
template <int NT>
__host__ __device__ constexpr int pw_slabs() { return (NT + 31) / 32; }  // staging slabs per tile

// Named barrier of one consumer warpgroup (ids 2 and 3; consumer_sync is id 1).
__device__ __forceinline__ void wg_sync(int wgc) { asm volatile("bar.sync %0, 128;" ::"r"(2 + wgc) : "memory"); }

template <int NT>
__device__ __forceinline__ void pw_epilogue_tma(const PwParams& p, const CUtensorMap* tmC, float* accm, const float* accc,
                                                int mt, int nt, int wgc, int wr, int t, uint8_t* last, uint8_t* other,
                                                bool leader) {
  const long long row0 = (long long)mt * 128 + wgc * 64;  // first output row of this warpgroup
#pragma unroll
  for (int i = 0; i < NT / 8; ++i) {
    const int col = nt * NT + 8 * i + 2 * t;
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
      const long long grow = row0 + wr + hrow * 8;
      float2 o = make_float2(accm[4 * i + 2 * hrow] + accc[4 * i + 2 * hrow], accm[4 * i + 2 * hrow + 1] + accc[4 * i + 2 * hrow + 1]);
      if (grow < p.M && col < p.N) {  // TMA drops what lies outside C; bias and R are not read there
        float2 b = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + col)) : make_float2(0.f, 0.f);
        if (p.R) {
          const float2 rr = __ldg(reinterpret_cast<const float2*>(p.R + grow * p.ldr + col));
          b.x += rr.x;
          b.y += rr.y;
        }
        o.x += b.x;
        o.y += b.y;
      }
      if (p.relu) {
        o.x = fmaxf(o.x, 0.f);
        o.y = fmaxf(o.y, 0.f);
      }
      accm[4 * i + 2 * hrow] = o.x;
      accm[4 * i + 2 * hrow + 1] = o.y;
    }
  }
#pragma unroll
  for (int s = 0; s < pw_slabs<NT>(); ++s) {
    uint8_t* buf = (pw_slabs<NT>() - 1 - s) & 1 ? other : last;
    if (leader) tma_store_wait_read<1>();
    wg_sync(wgc);
#pragma unroll
    for (int i = 4 * s; i < 4 * s + 4 && i < NT / 8; ++i) {
      const int cc = 8 * (i & 1) + 2 * t;  // column inside the 16-column box
#pragma unroll
      for (int hrow = 0; hrow < 2; ++hrow) {
        const int r = wr + hrow * 8;
        *reinterpret_cast<float2*>(buf + ((i >> 1) & 1) * kPwBoxBytes + r * 64 + (((cc >> 2) ^ ((r >> 1) & 3)) << 4) +
                                   (cc & 3) * 4) = make_float2(accm[4 * i + 2 * hrow], accm[4 * i + 2 * hrow + 1]);
      }
    }
    fence_proxy_async_smem();  // generic-proxy writes -> visible to the TMA engine
    wg_sync(wgc);
    if (leader) {
#pragma unroll
      for (int b = 0; b < 2 && 32 * s + 16 * b < NT; ++b) {
        const int col0 = nt * NT + 32 * s + 16 * b;
        if (col0 < p.N && row0 < p.M) tma_store_2d(tmC, buf + b * kPwBoxBytes, col0, (int)row0);
      }
      tma_store_commit();
    }
  }
}

// DWK = 0: plain 1x1 conv.  DWK = 3 | 5 (option "fuse_dwpw", on by default; MW x MW maps with MW = 16 | 32, stride 1): the
// layer's input is the output of a DWK x DWK depthwise conv that is never materialised -- the producer TMA-loads the
// depthwise INPUT box of each (128-pixel tile, 32-channel chunk) with its zero-filled halo (tmA is then the 4-D NHWC
// map of X), the consumer warps run the depthwise conv out of shared memory (dw_chunk) and write the A tile.
//
// Persistent: min(tiles, SMs) CTAs, CTA c walks tiles c, c + G, c + 2G, ...  The producer streams the CTA's whole
// chunk sequence through the mbarrier ring without regard to tile boundaries, so the next tile's first chunks land while
// the consumers finish and store the current one; stage and parity advance over that sequence.  Both consumer
// warpgroups share each tile (64 rows each, weights fetched once per 128 rows).  A consumer issues chunk c's MMA group
// and then waits only for chunk c - 1's (wgmma.wait_group 1), which frees c - 1's stage and A fragments; in the fused
// forms chunk c + 1's depthwise conv runs while chunk c's group is in flight.  wait_group 0 only before the epilogue.
// Each consumer warpgroup then stores its 64 rows by TMA from shared memory (pw_epilogue_tma) and goes straight on to
// the next tile; with p.tma_store == 0 it stores from registers (pw_epilogue).
template <int NT, int DWK, int MW = 16>
__global__ void __launch_bounds__(kPwThreads, 1)
pw_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmWh,
             const __grid_constant__ CUtensorMap tmWl, const __grid_constant__ CUtensorMap tmDW,
             const __grid_constant__ CUtensorMap tmDB, const __grid_constant__ CUtensorMap tmC, const PwParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int S = p.stages;
  // two 16 KB buffers after the ring: the epilogue's staging slabs and, in the fused forms, the A tiles
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + S * p.stage_bytes + 2 * kCorrABytes);  // [stages] TMA landed
  uint64_t* empty = full + S;  // [stages] 8 consumer warps done
  constexpr int w_bytes = NT * 128;
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmWh);
    prefetch_tmap(&tmWl);
    if (p.tma_store) prefetch_tmap(&tmC);
    for (int s = 0; s < S; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_trigger();  // the next kernel may start its prologue on SMs we have left
  pdl_wait();     // everything above overlapped the previous kernel's tail; its results are visible from here on

  // plain stage: [A tile 16 KB][w_hi][w_lo]; fused stage: [w_hi][w_lo][input box][dw weights DWK*DWK x 32][dw bias 32],
  // then two 16 KB buffers after the ring.  Each holds one staging slab of each consumer warpgroup (warpgroup w's 8 KB
  // at offset 8 KB * w).  In the fused forms the buffers are also the A tiles: an A tile is free once every consumer has
  // loaded its fragments, long before the stage's weights are (their MMAs still run), so two of them serve any ring
  // depth and the room they leave buys the ring a third stage.  A warpgroup stages only its own rows of an A tile,
  // which only it reads, once its last MMA group is done.  The tile's last slab goes to the last chunk's A tile, so the
  // next tile's first depthwise conv, which writes the other A tile, waits only for the slabs before it (wait_group.read
  // 1, then consumer_sync), and the last slab need only be read before the barrier that follows that conv.
  auto a_tile = [&](int s) { return smem + s * p.stage_bytes; };
  auto a_buf = [&](int b) { return smem + S * p.stage_bytes + b * kCorrABytes; };
  auto w_hi = [&](int s) { return smem + s * p.stage_bytes + (DWK > 0 ? 0 : kCorrABytes); };
  auto w_lo = [&](int s) { return w_hi(s) + w_bytes; };
  auto dw_box = [&](int s) { return w_lo(s) + w_bytes; };
  auto dw_wts = [&](int s) { return dw_box(s) + p.box_bytes; };
  auto dw_bia = [&](int s) { return dw_wts(s) + DWK * DWK * 128; };

  // Warpgroup index broadcast from lane 0: the compiler can prove it uniform, so no wgmma below is on a divergent path.
  const int wg = __shfl_sync(0xffffffffu, (int)threadIdx.x / 128, 0);
  if (wg == 0) {
    setmaxnreg_dec<kPwProducerRegs>();
    if (threadIdx.x == 0) {
      constexpr int th = 128 / MW, tpf = MW / th;  // tile rows, tiles per frame
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int mt = tile / p.num_n_tiles, nt = tile - mt * p.num_n_tiles;
        for (int c = 0; c < p.num_chunks; ++c) {
          mbar_wait_backoff(&empty[stage], phase ^ 1);
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
          if (++stage == S) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    return;
  }
  setmaxnreg_inc<kPwConsumerRegs>();

  const int ct = threadIdx.x - 128, warp = ct >> 5, lane = ct & 31;  // consumer thread / warp (0..255 / 0..7)
  const int wgc = warp >> 2, wr = (warp & 3) * 16 + (lane >> 2), t = lane & 3;  // consumer warpgroup, row inside it
  const int r0 = wgc * 64 + wr;
  const bool leader = (ct & 127) == 0;  // issues the warpgroup's TMA stores
  int stage = 0, ab = 0;  // ring stage, fused A buffer of the current chunk
  uint32_t phase = 0;
  int slab = 0;  // staging slabs written so far (plain form: the buffers alternate over the CTA's slabs)
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const int mt = tile / p.num_n_tiles, nt = tile - mt * p.num_n_tiles;
    float accm[NT / 2], accc[NT / 2];
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) accm[i] = accc[i] = 0.f;
    if constexpr (DWK > 0) {
      const bool drain = p.tma_store && tile != blockIdx.x;  // the previous tile's slabs lie in the A tiles
      if (drain) {
        if (leader) tma_store_wait_read<1>();
        consumer_sync();
      }
      mbar_wait(&full[stage], phase);
      dw_chunk<DWK, MW>(dw_box(stage), dw_wts(stage), dw_bia(stage), a_buf(ab), ct, p.dw_bias, p.dw_relu);
      if (drain && leader) tma_store_wait_read<0>();  // before the next depthwise conv writes the last slab's A tile
      consumer_sync();  // the A tile of this chunk is complete
    }
    int prev = 0;
    for (int c = 0; c < p.num_chunks; ++c) {
      if constexpr (DWK == 0) mbar_wait(&full[stage], phase);
      uint32_t hi[4][4], lo[4][4];
      load_a_frags(DWK > 0 ? a_buf(ab) : a_tile(stage), r0, t, hi, lo);
      const uint32_t bh = smem_u32(w_hi(stage)), bl = smem_u32(w_lo(stage));
      const int ksteps = (c == p.num_chunks - 1) ? p.last_ksteps : 4;
      wg_fence();
      if (ksteps == 4) mma3_chunk<NT, 4>(accm, accc, hi, lo, bh, bl);
      else if (ksteps == 3) mma3_chunk<NT, 3>(accm, accc, hi, lo, bh, bl);
      else if (ksteps == 2) mma3_chunk<NT, 2>(accm, accc, hi, lo, bh, bl);
      else mma3_chunk<NT, 1>(accm, accc, hi, lo, bh, bl);
      wg_commit();
      if (c > 0) {  // chunk c - 1's group is done: its stage may be refilled
        wg_wait_n<1>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[prev]);
      }
      prev = stage;
      if (++stage == S) {
        stage = 0;
        phase ^= 1;
      }
      if constexpr (DWK > 0) {
        ab ^= 1;  // its last reader loaded chunk c - 1's fragments before the previous consumer_sync
        if (c + 1 < p.num_chunks) {  // the next chunk's depthwise conv, while this chunk's MMAs run
          mbar_wait(&full[stage], phase);
          dw_chunk<DWK, MW>(dw_box(stage), dw_wts(stage), dw_bia(stage), a_buf(ab), ct, p.dw_bias, p.dw_relu);
          consumer_sync();
        }
      }
    }
    wg_wait_n<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[prev]);
    if (p.tma_store) {
      const int lb = DWK > 0 ? ab ^ 1 : (slab + pw_slabs<NT>() - 1) & 1;  // fused: the last chunk's A tile
      slab += pw_slabs<NT>();
      pw_epilogue_tma<NT>(p, &tmC, accm, accc, mt, nt, wgc, wr, t, a_buf(lb) + wgc * kPwSlabBytes,
                          a_buf(lb ^ 1) + wgc * kPwSlabBytes, leader);
    } else
      pw_epilogue<NT>(p, accm, accc, mt, nt, r0, t);
  }
  if (leader && p.tma_store) tma_store_wait<0>();  // the stores are complete before the CTA exits
}

// One-chunk GEMMs (K <= 32) on narrow tiles: one CTA per tile, 288 threads (two consumer warpgroups and one TMA
// producer warp), no persistence.  Such a CTA loads its A and W tiles, issues one group of MMAs and stores its tile;
// at NT <= 32 it needs 68 registers per thread, three CTAs share an SM and one CTA's loads and stores overlap another's
// MMAs, which the persistent kernel (one CTA per SM, its consumers' epilogue between two tiles' MMAs) does not match at
// these shapes.  Same mma3 sequence per output element and same epilogue as pw_tc_kernel.
template <int NT>
__global__ void __launch_bounds__(kTcThreads, 1)
pw_tc_narrow_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmWh,
                    const __grid_constant__ CUtensorMap tmWl, const PwParams p) {
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
  pdl_trigger();
  pdl_wait();

  const int mt = blockIdx.x / p.num_n_tiles, nt = blockIdx.x - mt * p.num_n_tiles;
  auto a_tile = [&](int s) { return smem + s * p.stage_bytes; };
  auto w_hi = [&](int s) { return smem + s * p.stage_bytes + kCorrABytes; };
  auto w_lo = [&](int s) { return w_hi(s) + w_bytes; };

  if (warp == 8) {
    if (lane == 0) {
      for (int c = 0; c < p.num_chunks; ++c) {
        const int stage = c % S;
        mbar_wait_backoff(&empty[stage], (uint32_t)(((c / S) & 1) ^ 1));
        mbar_arrive_expect_tx(&full[stage], kCorrABytes + 2 * w_bytes);
        tma_load_2d(a_tile(stage), &tmA, &full[stage], c * 32, mt * 128);
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
  pw_epilogue<NT>(p, accm, accc, mt, nt, r0, t);
}

constexpr int kPwMaxSmem = 232448 - 1024;  // 227 KB opt-in limit minus static/driver slack
constexpr int kPwMaxStages = 4;
constexpr int kPwSmemExtra = 1024 /*align*/ + 256 /*barriers*/;

// Ring depth of the persistent kernel: as many stages of `stage_bytes` as fit next to `fixed_bytes`, at most
// kPwMaxStages (the ring spans tile boundaries, so even a one- or two-chunk layer fills every stage).
inline int pw_stages(int stage_bytes, int fixed_bytes) {
  const int fit = (kPwMaxSmem - kPwSmemExtra - fixed_bytes) / stage_bytes;
  return fit < kPwMaxStages ? fit : kPwMaxStages;
}

// The plain persistent kernel keeps its two staging buffers next to a full ring at the widest tile.
constexpr int kPwStagingBytes = 2 * kCorrABytes;
static_assert(kPwMaxStages * (kCorrABytes + 2 * 128 * 128) + kPwStagingBytes + kPwSmemExtra <= kPwMaxSmem,
              "pw_tc_kernel<128, 0>: four ring stages and the staging buffers fit in shared memory");

// Output map of pw_tc_kernel's TMA stores: C = [M][N] at row pitch ldc, boxes of 64 rows x 16 columns.  16 divides every
// tile width, so a box never reaches into a neighbouring n-tile, and the N extent keeps the stores out of columns >= N of
// a wider buffer (the head's 320-column concat buffer).  TMA needs a 16-byte aligned base and pitch: returns 1 when
// either is not, and the kernel then stores from registers.
inline int make_tmap_out(CUtensorMap* m, float* C, int ldc, int M, int N) {
  if ((reinterpret_cast<uintptr_t>(C) & 15) || (ldc & 3)) return 1;
  return make_tmap_2d(m, C, (uint64_t)M, (uint64_t)N, (uint64_t)ldc, 64, 16);
}

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

// A GEMM with one K chunk (K <= 32) does little work per tile.  Such layers are cut into tiles of at most kPwNarrowNT
// columns and run on pw_tc_narrow_kernel, several CTAs per SM.  The A tile is then read once per n-tile, mostly from
// L2.  The tile width does not change any output element's sequence of mma3 products, so results are the same bit
// for bit.
constexpr int kPwNarrowNT = 32;
inline int pw_tile_n_one_chunk(int N) {
  const int Np = (N + 15) & ~15;
  const int tiles = (Np + kPwNarrowNT - 1) / kPwNarrowNT;
  const int need = (Np + tiles - 1) / tiles;
  return need <= 16 ? 16 : 32;
}

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
  if (e == cudaSuccess) e = cudaFuncSetAttribute(pw_tc_narrow_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPwMaxSmem);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(pw_tc_narrow_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPwMaxSmem);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return -1;
  }
  return 0;
}

// Persistent grid: one CTA per SM at most.
inline dim3 pw_grid(int tiles) { return dim3(tiles < num_sms() ? tiles : num_sms()); }

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
  const bool narrow = p.num_chunks == 1;
  const int NT = narrow ? pw_tile_n_one_chunk(N) : pw_tile_n(N);
  if (!NT) return -21;
  p.num_n_tiles = (((N + 15) & ~15) + NT - 1) / NT;
  p.num_tiles = ((M + 127) / 128) * p.num_n_tiles;
  p.last_ksteps = ((K - 32 * (p.num_chunks - 1)) + 7) / 8;
  p.relu = relu;
  p.dw_relu = p.dw_bias = p.box_bytes = p.tma_store = 0;
  p.stage_bytes = kCorrABytes + 2 * NT * 128;
  p.stages = narrow ? 1 : pw_stages(p.stage_bytes, kPwStagingBytes);
  CUtensorMap tmA, tmWh, tmWl;
  int r = make_tmap_2d(&tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, 128, 32);
  if (r) return r;
  r = make_tmap_2d(&tmWh, w_hi, (uint64_t)N, (uint64_t)K, (uint64_t)K, NT, 32);
  if (r) return r;
  r = make_tmap_2d(&tmWl, w_lo, (uint64_t)N, (uint64_t)K, (uint64_t)K, NT, 32);
  if (r) return r;
  cudaError_t e = cudaErrorInvalidValue;
  if (narrow) {
    const size_t smem_bytes = (size_t)p.stages * p.stage_bytes + kPwSmemExtra;
    if (NT == 16) e = launch_pdl(pw_tc_narrow_kernel<16>, dim3(p.num_tiles), dim3(kTcThreads), smem_bytes, s, tmA, tmWh, tmWl, p);
    else e = launch_pdl(pw_tc_narrow_kernel<32>, dim3(p.num_tiles), dim3(kTcThreads), smem_bytes, s, tmA, tmWh, tmWl, p);
    return e == cudaSuccess ? 0 : -23;
  }
  CUtensorMap tmC = tmA;
  r = make_tmap_out(&tmC, C, ldc, M, N);
  if (r < 0) return r;
  p.tma_store = r == 0;
  const size_t smem_bytes = (size_t)p.stages * p.stage_bytes + kPwStagingBytes + kPwSmemExtra;
  switch (NT) {
#define FEAR_PW_CASE(NT_)                                                                                               \
  case NT_:                                                                                                             \
    e = launch_pdl(pw_tc_kernel<NT_, 0>, pw_grid(p.num_tiles), dim3(kPwThreads), smem_bytes, s, tmA, tmWh, tmWl, tmA, tmA, \
                   tmC, p);                                                                                             \
    break;
    FEAR_PW_FOR_NT(FEAR_PW_CASE)
#undef FEAR_PW_CASE
  }
  return e == cudaSuccess ? 0 : -23;
}

// Depthwise-fused GEMM (option "fuse_dwpw", default on; tests/test_gpu_parity.py): 1x1 conv whose input is dw_k x dw_k depthwise(X)
// (+bias, ReLU), X = [B][map_w][map_w][K] channels-last, stride 1.  out = act(dw(X) * W^T + bias (+R)).
// Returns 1 when the shape is not covered (caller runs the two kernels separately): the shape is taken when two stages
// of [A tile | weights | box] (one for a one-chunk layer) fit in shared memory.  The kernel's ring of [weights | box]
// stages next to two A tiles then has at least as many stages, up to kPwMaxStages.
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
  p.num_tiles = (M / 128) * p.num_n_tiles;
  p.last_ksteps = ((K - 32 * (p.num_chunks - 1)) + 7) / 8;
  p.relu = relu;
  p.dw_relu = dw_relu;
  p.dw_bias = dw_b != nullptr;
  const int ih = 128 / map_w + dw_k - 1, iw = map_w + dw_k - 1;
  p.box_bytes = ih * iw * 128;
  p.stage_bytes = (2 * NT * 128 + p.box_bytes + dw_k * dw_k * 128 + 128 + 1023) & ~1023;
  if ((p.num_chunks < 2 ? 1 : 2) * (kCorrABytes + p.stage_bytes) + kPwSmemExtra > kPwMaxSmem) return 1;
  p.stages = pw_stages(p.stage_bytes, 2 * kCorrABytes);  // the two A tiles double as the epilogue's staging
  const size_t smem_bytes = (size_t)p.stages * p.stage_bytes + 2 * kCorrABytes + kPwSmemExtra;
  CUtensorMap tmX, tmWh, tmWl, tmDW, tmDB, tmC;
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
  // At NT <= 32 a tile is one staging slab, whose barriers and drain cost more next to the depthwise conv than the TMA
  // store saves (xif3_1 .. xif3_3, DESIGN.md 4.1): those tiles keep the stores from registers.
  tmC = tmX;
  r = NT > 32 ? make_tmap_out(&tmC, C, ldc, M, N) : 1;
  if (r < 0) return r;
  p.tma_store = r == 0;
  cudaError_t e = cudaErrorInvalidValue;
#define FEAR_PW_DW_LAUNCH(NT_, K_, MW_)                                                                              \
  e = launch_pdl(pw_tc_kernel<NT_, K_, MW_>, pw_grid(p.num_tiles), dim3(kPwThreads), smem_bytes, s, tmX, tmWh, tmWl, \
                 tmDW, tmDB, tmC, p)
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
