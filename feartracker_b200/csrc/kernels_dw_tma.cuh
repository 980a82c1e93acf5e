// TMA-fed depthwise convolution (channels-last fp32), sm_90a.
//
// The register-strip kernels in kernels_ffma.cuh fetch every input pixel straight from global memory; ncu shows
// them latency-bound on the 5x5 layers (2 TB/s of DRAM traffic, ~50 % L1 hit rate, 4x the algorithmic bytes
// through L2).  Here a persistent CTA streams (TH x TW pixels) x 32-channel tiles through a shared-memory ring:
//
//   producer      : (first warp of each group, one lane) one 4-D cp.async.bulk.tensor per tile -- box = [IH][IW][32 ch], IH = (TH-1)*S+K -- whose
//                   out-of-image halo is zero-filled by the TMA unit (= the conv's zero padding, no branches),
//                   plus the [K*K][32] weight slab and the 32 biases of that channel block, all on one mbarrier
//   consumer warps: two groups of four warps take alternate tiles; lane = (channel group of 4, tile position); each thread produces a TY x TX block of
//                   output pixels for its 4 channels from LDS.128 reads (a quarter warp reads 128 contiguous
//                   bytes: conflict free), FMA order (ky, kx ascending from the bias) identical to the other
//                   depthwise kernels so the results are bit-identical, then stores float4s (128 B / pixel).
//
// Every input byte is read from HBM/L2 once per tile (halo overlap only), every output byte written once.
#pragma once
#include "tc_common.cuh"

namespace fear {
namespace tc {

struct DwTmaParams {
  float* out;  // [B][Ho][Wo][C]
  int C4;      // C / 4
  int Ho, Wo;
  int tiles_x, tiles_y, cblocks;
  int num_tiles;
};

constexpr int kDwCB = 32;           // channels per tile
// GROUPS consumer groups per CTA; group g takes the tiles with (iteration % GROUPS) == g.  STAGES must be a
// multiple of GROUPS: every stage then belongs to ONE group, which waits on / refills it strictly in order.
// (With a shared ring a fast group could test full[s] while the previous use of that stage -- another group's
// tile -- is still outstanding, and an mbarrier parity wait cannot tell "two phases behind" from "done".)
// 8 warps = 2 per SM sub-partition, which leaves the full register budget to the 2x8-pixel thread blocks.

template <int K, int S, int TH, int TW>
struct DwTile {
  static constexpr int IH = (TH - 1) * S + K;
  static constexpr int IW = (TW - 1) * S + K;
  static constexpr int kInBytes = IH * IW * kDwCB * 4;
  static constexpr int kWBytes = K * K * kDwCB * 4;
  static constexpr int kBiasBytes = kDwCB * 4;
  static constexpr int kStageBytes = kInBytes + kWBytes + kBiasBytes;  // all multiples of 128
};

template <int K, int S, int TH, int TW, int STAGES>
constexpr int dw_tma_smem_bytes() {
  return STAGES * DwTile<K, S, TH, TW>::kStageBytes + 2 * STAGES * 8 + 128;
}

// GW = consumer warps working on one tile (per group); the default of 4 warps x (2 x 8)-pixel blocks has not been compared
// against other splits on the H100.
template <int K, int S, int TH, int TW, int TX, int TY, int STAGES, int GROUPS, bool RELU, bool BIAS, int GW = 4>
__global__ void __launch_bounds__(GROUPS * GW * 32, 1)
dw_tma_kernel(const __grid_constant__ CUtensorMap tmIn, const __grid_constant__ CUtensorMap tmW,
              const __grid_constant__ CUtensorMap tmBias, const DwTmaParams p) {
  using T = DwTile<K, S, TH, TW>;
  constexpr int P = K / 2;
  constexpr int IW = T::IW;
  constexpr int NIN = (TX - 1) * S + K;  // input columns feeding TX outputs
  constexpr int NR = (TY - 1) * S + K;   // input rows feeding TY outputs
  constexpr int PX = TW / TX, PY = TH / TY;
  constexpr int NPOS = PX * PY;
  static_assert(TW % TX == 0 && TH % TY == 0, "tile must be a multiple of the thread block");
  static_assert(STAGES % GROUPS == 0, "each stage must be owned by one consumer group");

  extern __shared__ uint8_t dw_smem_raw[];
  // (offset arithmetic on the __shared__ array itself keeps the address space visible to the compiler: LDS, not LD)
  uint8_t* smem = dw_smem_raw + ((128u - (smem_u32(dw_smem_raw) & 127u)) & 127u);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * T::kStageBytes);
  uint64_t* empty = full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], GW);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_trigger();  // (see tc_common.cuh) the next kernel may start its prologue on SMs we have left ...
  pdl_wait();     // ... and ours overlapped the previous kernel's tail; its results are visible from here on

  // One 4-D box (+ weight slab + biases) per tile, all completing on full[stage].
  auto issue_tile = [&](int tile, int stage) {
    const int cb = tile % p.cblocks;
    int rest = tile / p.cblocks;
    const int tx = rest % p.tiles_x;
    rest /= p.tiles_x;
    const int ty = rest % p.tiles_y;
    const int b = rest / p.tiles_y;
    uint8_t* st = smem + stage * T::kStageBytes;
    mbar_arrive_expect_tx(&full[stage], T::kInBytes + T::kWBytes + (BIAS ? T::kBiasBytes : 0));
    tma_load_4d(st, &tmIn, &full[stage], cb * kDwCB, tx * TW * S - P, ty * TH * S - P, b);
    tma_load_2d(st + T::kInBytes, &tmW, &full[stage], cb * kDwCB, 0);
    if (BIAS) tma_load_2d(st + T::kInBytes + T::kWBytes, &tmBias, &full[stage], cb * kDwCB, 0);
  };
  if (threadIdx.x == 0) {  // prologue: fill the ring
    for (int i = 0; i < STAGES; ++i) {
      const int tile = blockIdx.x + i * gridDim.x;
      if (tile < p.num_tiles) issue_tile(tile, i);
    }
  }

  // ---------------- consumers ----------------
  const int cg = lane & 7;  // channel group (float4) inside the 32-channel block
  const int group = warp / GW, gwarp = warp % GW;
  int it = 0;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++it) {
    if (it % GROUPS != group) continue;
    const int s = it % STAGES;
    const uint32_t ph = (uint32_t)(it / STAGES) & 1u;
    const int cb = tile % p.cblocks;
    int rest = tile / p.cblocks;
    const int tx = rest % p.tiles_x;
    rest /= p.tiles_x;
    const int ty = rest % p.tiles_y;
    const int b = rest / p.tiles_y;
    const int c4 = cb * (kDwCB / 4) + cg;
    mbar_wait(&full[s], ph);
    const F4* in4 = reinterpret_cast<const F4*>(smem + s * T::kStageBytes);
    const F4* w4 = reinterpret_cast<const F4*>(smem + s * T::kStageBytes + T::kInBytes);
    const F4* b4p = reinterpret_cast<const F4*>(smem + s * T::kStageBytes + T::kInBytes + T::kWBytes);

#pragma unroll 1
    for (int pos = gwarp * 4 + (lane >> 3); pos < NPOS; pos += GW * 4) {
      const int px = pos % PX, py = pos / PX;
      const int ox_l = px * TX, oy_l = py * TY;
      F4 acc[TY][TX];
      F4 bias4;
      if (BIAS) bias4 = b4p[cg];
      else bias4.lo = bias4.hi = 0ull;
#pragma unroll
      for (int y = 0; y < TY; ++y)
#pragma unroll
        for (int t = 0; t < TX; ++t) acc[y][t] = bias4;
      F4 wk[K][K];
      const F4* base = in4 + ((oy_l * S) * IW + ox_l * S) * (kDwCB / 4) + cg;
#pragma unroll
      for (int r = 0; r < NR; ++r) {
        F4 v[NIN];
#pragma unroll
        for (int i = 0; i < NIN; ++i) v[i] = base[(r * IW + i) * (kDwCB / 4)];
        if (r < K) {
#pragma unroll
          for (int kx = 0; kx < K; ++kx) wk[r < K ? r : 0][kx] = w4[(r * K + kx) * (kDwCB / 4) + cg];
        }
#pragma unroll
        for (int y = 0; y < TY; ++y) {
          const int ky = r - y * S;
          if (ky >= 0 && ky < K) {
#pragma unroll
            for (int kx = 0; kx < K; ++kx) {
              const F4 k = wk[(ky >= 0 && ky < K) ? ky : 0][kx];
#pragma unroll
              for (int t = 0; t < TX; ++t) ffma2(acc[y][t].lo, v[t * S + kx].lo, k.lo);
#pragma unroll
              for (int t = 0; t < TX; ++t) ffma2(acc[y][t].hi, v[t * S + kx].hi, k.hi);
            }
          }
        }
      }
      if (c4 < p.C4) {
        float4* o = reinterpret_cast<float4*>(p.out) +
                    (((long long)b * p.Ho + ty * TH + oy_l) * p.Wo + tx * TW + ox_l) * p.C4 + c4;
#pragma unroll
        for (int y = 0; y < TY; ++y)
#pragma unroll
          for (int t = 0; t < TX; ++t) {
            float4 r4 = f4_to_float4(acc[y][t]);
            if (RELU) {
              r4.x = fmaxf(r4.x, 0.f);
              r4.y = fmaxf(r4.y, 0.f);
              r4.z = fmaxf(r4.z, 0.f);
              r4.w = fmaxf(r4.w, 0.f);
            }
            o[((long long)y * p.Wo + t) * p.C4] = r4;
          }
      }
    }
    __syncwarp();
    if (lane == 0) {
      mbar_arrive(&empty[s]);
      if (gwarp == 0) {  // refill this stage with the tile STAGES iterations ahead once the whole group has left it
        const int next = tile + STAGES * gridDim.x;
        if (next < p.num_tiles) {
          mbar_wait(&empty[s], ph);
          issue_tile(next, s);
        }
      }
    }
    __syncwarp();
  }
}

// Host launcher.  Returns 0 on launch, 1 when the shape is not covered (caller falls back), < 0 on error.
template <int K, int S, int TH, int TW, int TX, int TY, int STAGES, int GROUPS, bool RELU, bool BIAS, int GW = 4>
inline int launch_dw_tma_t(cudaStream_t s, const float* in, const float* w, const float* bias, float* out, int B, int H,
                           int W, int C, int num_sms) {
  using T = DwTile<K, S, TH, TW>;
  const int Ho = H / S, Wo = W / S;
  if (Ho % TH || Wo % TW || C % 4) return 1;
  auto kern = dw_tma_kernel<K, S, TH, TW, TX, TY, STAGES, GROUPS, RELU, BIAS, GW>;
  constexpr int smem = dw_tma_smem_bytes<K, S, TH, TW, STAGES>();
  if (attr_needed(reinterpret_cast<const void*>(kern))) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return -30;
  }
  CUtensorMap tmIn, tmW, tmB;
  int r = make_tmap_nhwc(&tmIn, in, (uint64_t)B, (uint64_t)H, (uint64_t)W, (uint64_t)C, kDwCB, T::IW, T::IH);
  if (r) return r;
  r = make_tmap_2d_plain(&tmW, w, (uint64_t)K * K, (uint64_t)C, K * K, kDwCB);
  if (r) return r;
  if (BIAS) {
    r = make_tmap_2d_plain(&tmB, bias, 1, (uint64_t)C, 1, kDwCB);
    if (r) return r;
  } else {
    tmB = tmW;
  }
  DwTmaParams p;
  p.out = out;
  p.C4 = C / 4;
  p.Ho = Ho;
  p.Wo = Wo;
  p.tiles_x = Wo / TW;
  p.tiles_y = Ho / TH;
  p.cblocks = (C + kDwCB - 1) / kDwCB;
  p.num_tiles = B * p.tiles_x * p.tiles_y * p.cblocks;
  int grid = num_sms;
  if (grid > p.num_tiles) grid = p.num_tiles;
  if (launch_pdl(kern, dim3(grid), dim3(GROUPS * GW * 32), (size_t)smem, s, tmIn, tmW, tmB, p) != cudaSuccess) return -31;
  return 0;
}

}  // namespace tc
}  // namespace fear
