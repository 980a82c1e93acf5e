// sm_90a primitives used by the tensor-core kernels: mbarrier, TMA (cp.async.bulk.tensor),
// wgmma (mma_async kind tf32 / commit / wait), shared-memory matrix descriptors, tensor-map creation.
//
// All inline PTX here is architecture-specific to Hopper; the library is compiled for
// compute_90a only.  Nothing links against libcuda: cuTensorMapEncodeTiled is resolved at run
// time through cudaGetDriverEntryPoint so the .so still loads on a machine without a driver.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <mutex>
#include <set>
#include <string>
#include <unordered_map>

namespace fear {
namespace tc {

// ------------------------------------------------------------------------------------------
// Host: tensor maps
// ------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled& encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  return fn;
}

inline int resolve_driver() {
  if (encode_fn()) return 0;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
  if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) return -10;
  encode_fn() = (PFN_encodeTiled)p;
  return 0;
}

// ---- per-device library state -----------------------------------------------------------------
// cudaFuncSetAttribute and the "is this an sm_90 with a working driver entry point" answer are PER DEVICE, so they
// are keyed by the current device (every C entry point selects its handle's device before launching anything).
struct DeviceState {
  bool inited = false;    // fear_init() ran for this device
  bool tc_ready = false;  // tensor-core / TMA path usable
  int num_sms = 0;
  std::set<const void*> attrs;  // kernels whose opt-in shared-memory attribute has been set on this device
};
inline std::mutex& state_mutex() {
  static std::mutex m;
  return m;
}
inline DeviceState& dev_state() {
  static DeviceState st[64];
  int d = 0;
  cudaGetDevice(&d);
  return st[d & 63];
}
inline bool available() { return dev_state().tc_ready; }
inline int num_sms() { return dev_state().num_sms; }
// true exactly once per (device, kernel): the caller then sets the kernel's attributes.
inline bool attr_needed(const void* fn) {
  std::lock_guard<std::mutex> lock(state_mutex());
  return dev_state().attrs.insert(fn).second;
}

// ---- tensor maps (cached) ------------------------------------------------------------------------
// Encoding a CUtensorMap is a pure host-side function of (base, dims, strides, box, swizzle); the executor asks
// for the same few hundred maps every step (workspace pointers are stable), so they are memoised per host thread.
struct TmapKey {
  uint64_t v[16];
  bool operator==(const TmapKey& o) const { return memcmp(v, o.v, sizeof(v)) == 0; }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    uint64_t h = 1469598103934665603ull;
    for (uint64_t x : k.v) {
      h ^= x;
      h *= 1099511628211ull;
    }
    return (size_t)h;
  }
};
inline int encode_cached(CUtensorMap* m, CUtensorMapDataType dt, uint32_t rank, const void* base, const cuuint64_t* dims,
                         const cuuint64_t* strides, const cuuint32_t* box, CUtensorMapSwizzle sw,
                         CUtensorMapL2promotion promo) {
  if (resolve_driver()) return -10;
  static thread_local std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> cache;
  TmapKey k;
  memset(&k, 0, sizeof(k));
  k.v[0] = (uint64_t)(uintptr_t)base;
  k.v[1] = ((uint64_t)dt << 32) | ((uint64_t)rank << 16) | ((uint64_t)sw << 8) | (uint64_t)promo;
  for (uint32_t i = 0; i < rank; ++i) {
    k.v[2 + i] = dims[i];
    k.v[7 + i] = (i + 1 < rank) ? strides[i] : 0;
    k.v[12 + (i >> 1)] |= (uint64_t)box[i] << (32 * (i & 1));
  }
  auto it = cache.find(k);
  if (it != cache.end()) {
    *m = it->second;
    return 0;
  }
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = encode_fn()(m, dt, rank, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                           promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return -11;
  if (cache.size() > 8192) cache.clear();
  cache.emplace(k, *m);
  return 0;
}

// 2-D fp32 row-major tensor [rows][cols] with row pitch `pitch_floats`; box = [box_rows][box_cols];
// 128-byte swizzle when box_cols * 4 == 128, 64-byte swizzle for 64-byte rows, none otherwise.
inline int make_tmap_2d(CUtensorMap* m, const float* base, uint64_t rows, uint64_t cols, uint64_t pitch_floats,
                        uint32_t box_rows, uint32_t box_cols) {
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {pitch_floats * sizeof(float)};
  cuuint32_t box[2] = {box_cols, box_rows};
  CUtensorMapSwizzle sw = (box_cols * 4 == 128)  ? CU_TENSOR_MAP_SWIZZLE_128B
                          : (box_cols * 4 == 64) ? CU_TENSOR_MAP_SWIZZLE_64B
                                                 : CU_TENSOR_MAP_SWIZZLE_NONE;
  return encode_cached(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, base, dims, strides, box, sw,
                       CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

// 4-D fp32 channels-last activation tensor [B][H][W][C] (dims listed innermost first: C, W, H, B), no swizzle.
// The box may start at negative / end at out-of-range coordinates: TMA zero-fills those elements, which is
// exactly the zero padding of a "same" convolution (and it still counts the full box bytes on the mbarrier).
inline int make_tmap_nhwc(CUtensorMap* m, const float* base, uint64_t B, uint64_t H, uint64_t W, uint64_t C,
                          uint32_t box_c, uint32_t box_w, uint32_t box_h) {
  cuuint64_t dims[4] = {C, W, H, B};
  cuuint64_t strides[3] = {C * sizeof(float), W * C * sizeof(float), H * W * C * sizeof(float)};
  cuuint32_t box[4] = {box_c, box_w, box_h, 1};
  return encode_cached(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, base, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE,
                       CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}

// Generic unswizzled 3-D map (dims / box innermost first, strides in bytes for dims 1 and 2); out-of-range
// elements read as zero.  Used for the image patches of the fused stem kernel (fp32 planes or uint8 HWC rows).
inline int make_tmap_3d(CUtensorMap* m, CUtensorMapDataType dt, const void* base, uint64_t d0, uint64_t d1, uint64_t d2,
                        uint64_t stride1_bytes, uint64_t stride2_bytes, uint32_t b0, uint32_t b1, uint32_t b2) {
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {stride1_bytes, stride2_bytes};
  cuuint32_t box[3] = {b0, b1, b2};
  return encode_cached(m, dt, 3, base, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}

// Plain (unswizzled) 2-D map, used for the small per-layer weight / bias tables.
inline int make_tmap_2d_plain(CUtensorMap* m, const float* base, uint64_t rows, uint64_t cols, uint32_t box_rows,
                              uint32_t box_cols) {
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * sizeof(float)};
  cuuint32_t box[2] = {box_cols, box_rows};
  return encode_cached(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, base, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE,
                       CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}

// Launch `kern` with programmatic stream serialization (PDL) unless disabled or the stream is being captured
// into a CUDA graph (graphs keep the plain launch).
inline bool& pdl_enabled() {
  static bool on = true;  // fear_set_option("pdl", "0") restores plain stream-ordered launches
  return on;
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  const bool use = pdl_enabled() && cudaStreamIsCapturing(s, &cap) == cudaSuccess && cap == cudaStreamCaptureStatusNone;
  cfg.attrs = attr;
  cfg.numAttrs = use ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// ------------------------------------------------------------------------------------------
// Device helpers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (kernel error) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
#pragma unroll 1
  for (uint32_t spin = 0; spin < (1u << 26); ++spin)
    if (mbar_try_wait(bar, parity)) return;
  __trap();
}

// Same, for single-thread producer / issuer roles that may wait long: back off between polls so the spinning
// warp does not compete for issue slots with the warps that do the work on the same SM sub-partition.
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
#pragma unroll 1
  for (uint32_t spin = 0; spin < (1u << 24); ++spin) {
    __nanosleep(64);
    if (mbar_try_wait(bar, parity)) return;
  }
  __trap();
}

__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// TMA: 2-D tile global -> shared, completion on an mbarrier (complete_tx::bytes).
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// TMA: 3-D tile global -> shared.
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0, int32_t c1,
                                            int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// TMA: 4-D tile global -> shared (coordinates innermost first; out-of-range parts are zero-filled).
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0, int32_t c1,
                                            int32_t c2, int32_t c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3)
      : "memory");
}
// TMA: 4-D tile global -> L2 only (no shared-memory destination, no completion to wait for).
__device__ __forceinline__ void tma_prefetch_4d(const CUtensorMap* m, int32_t c0, int32_t c1, int32_t c2, int32_t c3) {
  asm volatile("cp.async.bulk.prefetch.tensor.4d.L2.global.tile [%0, {%1, %2, %3, %4}];" ::"l"(reinterpret_cast<uint64_t>(m)),
               "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
// TMA: 2-D tile shared -> global (bulk async group).
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// Two independent round-to-nearest fp32 FMAs on the halves of 64-bit register pairs (the kernels keep two channels
// per 64-bit shared-memory word); bit-identical to two fmaf() calls.
struct __align__(16) F4 {
  unsigned long long lo, hi;  // (x, y), (z, w)
};
__device__ __forceinline__ void ffma2(unsigned long long& acc, unsigned long long a, unsigned long long b) {
  const float x = fmaf(__uint_as_float((uint32_t)a), __uint_as_float((uint32_t)b), __uint_as_float((uint32_t)acc));
  const float y = fmaf(__uint_as_float((uint32_t)(a >> 32)), __uint_as_float((uint32_t)(b >> 32)), __uint_as_float((uint32_t)(acc >> 32)));
  acc = (unsigned long long)__float_as_uint(x) | ((unsigned long long)__float_as_uint(y) << 32);
}
__device__ __forceinline__ unsigned long long pack2(uint32_t lo, uint32_t hi) {
  return (unsigned long long)lo | ((unsigned long long)hi << 32);
}
__device__ __forceinline__ float4 f4_to_float4(const F4& v) {
  float4 r;
  r.x = __uint_as_float((unsigned)(v.lo & 0xffffffffull));
  r.y = __uint_as_float((unsigned)(v.lo >> 32));
  r.z = __uint_as_float((unsigned)(v.hi & 0xffffffffull));
  r.w = __uint_as_float((unsigned)(v.hi >> 32));
  return r;
}

// ---- programmatic dependent launch (PDL) ---------------------------------------------------
// A kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may start while its predecessor in
// the stream is still draining: its CTAs run their prologue (barrier init, descriptor prefetch)
// on SMs the predecessor has already left, then block in pdl_wait() until the predecessor has completed and its
// writes are visible.  pdl_trigger() lets the *next* kernel do the same with us.  Both are no-ops for a normal launch.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---- wgmma (warpgroup MMA, tf32) ----------------------------------------------------------
// D[64 x N] += A[64 x 8] * B[N x 8]^T with the A fragment in REGISTERS and B a shared-memory descriptor; fp32
// accumulators in registers (thread (warp w, lane 4g + t) of the warpgroup holds rows 16w + g and 16w + g + 8,
// columns 8i + 2t and 8i + 2t + 1 of every 8-column group i; A: a0 = (g, t), a1 = (g + 8, t), a2 = (g, t + 4),
// a3 = (g + 8, t + 4)).  Wider tiles are composed of N = 64 / 32 / 16 instructions on adjacent weight rows.
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

#define FEAR_WG_D8(d, o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
template <int N>
__device__ __forceinline__ void wgmma_tf32(float* d, const uint32_t (&a)[4], uint64_t bdesc);
template <>
__device__ __forceinline__ void wgmma_tf32<16>(float* d, const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1;\n\t}\n"
      : FEAR_WG_D8(d, 0)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc));
}
template <>
__device__ __forceinline__ void wgmma_tf32<32>(float* d, const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "{%16, %17, %18, %19}, %20, p, 1, 1;\n\t}\n"
      : FEAR_WG_D8(d, 0), FEAR_WG_D8(d, 8)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc));
}
template <>
__device__ __forceinline__ void wgmma_tf32<64>(float* d, const uint32_t (&a)[4], uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}\n"
      : FEAR_WG_D8(d, 0), FEAR_WG_D8(d, 8), FEAR_WG_D8(d, 16), FEAR_WG_D8(d, 24)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc));
}
#undef FEAR_WG_D8

// Shared-memory B operand, K-major, 128-byte swizzle (rows of 128 B, 8-row atoms of 1024 B, tile base 1024-B
// aligned): start address >> 4 in bits [0,14), LBO (unused for swizzled K-major) = 1 in [16,30), SBO = 1024 B >> 4
// in [32,46), layout SWIZZLE_128B = 1 in [62,64).  Advancing K by one MMA step (8 tf32 = 32 B) adds 32 B to the
// start address; advancing N by 16 rows adds 2048 B.
__device__ __forceinline__ uint64_t wg_desc_k_sw128(uint32_t smem_addr) {
  uint64_t d = (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// 3xTF32 product of one K step into a (main, correction) accumulator pair, NT columns wide:
//   main += a_hi * w_hi ;  corr += a_hi * w_lo ;  corr += a_lo * w_hi          (result = main + corr)
// bh / bl: shared-memory addresses of the K step inside the w_hi / w_lo tiles.  Every tensor-core kernel of the
// library accumulates through this function in K order, so fused and unfused forms of a layer agree bit for bit.
template <int NT>
__device__ __forceinline__ void mma3(float* main, float* corr, const uint32_t (&ah)[4], const uint32_t (&al)[4],
                                     uint32_t bh, uint32_t bl) {
  static_assert(NT % 16 == 0 && NT <= 128, "tile width");
  constexpr int n0 = NT >= 64 ? 64 : (NT >= 32 ? 32 : 16);
  wgmma_tf32<n0>(main, ah, wg_desc_k_sw128(bh));
  wgmma_tf32<n0>(corr, ah, wg_desc_k_sw128(bl));
  wgmma_tf32<n0>(corr, al, wg_desc_k_sw128(bh));
  if constexpr (NT > n0) mma3<NT - n0>(main + n0 / 2, corr + n0 / 2, ah, al, bh + n0 * 128, bl + n0 * 128);
}

// A fragments of one 32-channel chunk (4 K steps) for this thread's rows r0 and r0 + 8 of a [rows][32] fp32 tile in
// the SWIZZLE_128B layout (16-byte chunk index ^ (row % 8)), split into tf32 hi (13 low mantissa bits cleared) and
// lo = v - hi (exact in fp32; the tensor core drops lo's own low bits: |err| <= 2^-21 |v|).
__device__ __forceinline__ void load_a_frags(const uint8_t* tile, int r0, int t, uint32_t (&hi)[4][4], uint32_t (&lo)[4][4]) {
  const int g = r0 & 7;
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int row = r0 + (e & 1) * 8, ch = 2 * j + (e >> 1);
      const float v = *reinterpret_cast<const float*>(tile + row * 128 + ((ch ^ g) << 4) + t * 4);
      const uint32_t h = __float_as_uint(v) & 0xFFFFE000u;
      hi[j][e] = h;
      lo[j][e] = __float_as_uint(v - __uint_as_float(h));
    }
}

// Host mirror of cvt.rna.tf32.f32 (round to nearest, ties away from zero; finite inputs).
inline float host_rna_tf32(float v) {
  uint32_t u;
  memcpy(&u, &v, 4);
  u = (u + 0x1000u) & 0xFFFFE000u;
  float r;
  memcpy(&r, &u, 4);
  return r;
}

// fp32 -> (hi, lo) with hi = rna_tf32(v), lo = rna_tf32(v - hi): v ~= hi + lo to ~2^-22 relative.
__device__ __forceinline__ void split_tf32(float v, float& hi, float& lo) {
  uint32_t h, l;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(v));
  hi = __uint_as_float(h);
  const float r = v - hi;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(l) : "f"(r));
  lo = __uint_as_float(l);
}

// Truncation split: hi = v with the 13 low mantissa bits cleared, lo = v - hi (exact in fp32; the tensor core then drops lo's own low bits: |err| <= 2^-21 |v|).
__device__ __forceinline__ void split_tf32_trunc(float v, float& hi, float& lo) {
  hi = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
  lo = v - hi;
}

}  // namespace tc
}  // namespace fear
