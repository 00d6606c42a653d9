// tc_common.cuh -- shared pieces of the sm_90a tensor-core kernels: PTX wrappers (mbarrier, TMA, programmatic dependent launch),
// the K-major 128B / 64B-swizzle wgmma smem descriptors, fp16 / TF32 split helpers, and the host-side CUtensorMap cache.
#pragma once
#include <cuda.h>

#include <map>
#include <mutex>
#include <string.h>
#include <stdlib.h>
#include <utility>

#include "common.cuh"
#include "wgmma.cuh"

namespace cdx {
namespace tc {

// ------------------------------------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok;
}
// Not inlined: a trap instruction inside a kernel makes ptxas hold the whole kernel to its launch register count, which ignores
// the setmaxnreg budget of the consumer warpgroups (the 128-wide wgmma consumers then spill); behind a call it does not.
static __device__ __noinline__ void mbar_wait_timeout() { __trap(); }
// bounded wait: a protocol bug traps (error returned to the host) instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) mbar_wait_timeout();
  }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
               "l"(map), "r"(bar), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst),
               "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
// smem -> global tile store through the tensor map (bulk async group of the issuing thread); the smem tile is in the map's
// swizzled layout, rows / columns outside the tensor are clipped by the hardware
__device__ __forceinline__ void tma_store_2d(uint32_t src, const CUtensorMap* map, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(map), "r"(src), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(uint32_t src, const CUtensorMap* map, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(map), "r"(src), "r"(c0), "r"(c1),
               "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all bulk stores of this thread have completed: their writes are performed in global memory
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// all bulk stores of this thread have finished READING their shared-memory source (it may be overwritten)
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }   // all but the newest
// Programmatic dependent launch (launch attribute set by launch_ex below unless CDX_PDL=0; both instructions are no-ops without it):
// pdl_trigger() lets the next kernel of the stream start launching CTAs once every CTA of this grid has issued it, pdl_wait() blocks
// until the preceding grid has completed and flushed.  Rule in this code base: trigger at kernel entry, wait after the setup that
// touches no global memory and BEFORE the first global access of any thread (reads of a predecessor's output, and writes of buffers a
// predecessor may still read: the workspace arena is reused in stream order)
// A kernel launched this way overlaps its predecessor, so it must not read the predecessor's output through the non-coherent path
// (__ldg, or const __restrict__ pointers the compiler turns into LDG.CONSTANT): that path assumes the data is read-only for the whole
// lifetime of the kernel, and on sm_90 it returned stale values here.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// K-major, 128-byte-swizzled smem operand descriptor for wgmma (rows of 128 B, 8-row atoms of 1024 B; the tile base is
// 1024-byte aligned, so the base-offset field stays 0).  Advancing along K inside the 128-byte row = adding (bytes >> 4).
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);       // start address
  d |= (uint64_t)1 << 16;                        // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;              // stride byte offset: 8 rows * 128 B
  d |= (uint64_t)1 << 62;                        // SWIZZLE_128B
  return d;
}
// K-major, 64-byte-swizzled variant (rows of 64 B = 32 fp16, 8-row atoms of 512 B; the tile base is 1024-byte aligned).  Advancing
// one k16 step (32 B) along the row = adding 2 to the start-address field, as with make_desc.
__device__ __forceinline__ uint64_t make_desc_sw64(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);       // start address
  d |= (uint64_t)1 << 16;                        // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(512 >> 4) << 32;               // stride byte offset: 8 rows * 64 B
  d |= (uint64_t)2 << 62;                        // SWIZZLE_64B
  return d;
}

// exponent e such that amax * 2^e lies in [2^14, 2^15): |x * 2^e| < 2^15 for every |x| <= amax (0 for an all-zero tensor)
__device__ __forceinline__ int h16_exp_of(float amax) {
  const int be = (int)((__float_as_uint(amax) >> 23) & 0xffu);
  if (be == 0 || be == 0xff) return 0;
  // 2^2 <= amax < 2^15: no rescale.  The split is then exact to 2^-25 absolute (fp16 subnormal spacing of the lo term), i.e.
  // <= 2^-27 of the tensor's max -- below fp32's own rounding of the products -- and the split warps skip one multiply per element
  if (be - 127 >= 2 && be - 127 <= 14) return 0;
  return min(max(14 - (be - 127), -100), 100);
}
__device__ __forceinline__ float exp2i(int e) { return __uint_as_float((uint32_t)(min(max(e, -126), 127) + 127) << 23); }
__device__ __forceinline__ uint32_t rn_tf32(uint32_t bits) { return (bits + 0x1000u) & 0xFFFFE000u; }


// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

struct MapKey {
  const void* ptr;
  uint64_t dims[4], strides[3];
  uint32_t box[4], es[4];
  int rank;
  int esize;
  int swz;
  bool operator<(const MapKey& o) const { return memcmp(this, &o, sizeof(MapKey)) < 0; }
};

// fp32 (esize 4) or fp16 (esize 2), 128B swizzle (swz 128) or 64B swizzle (swz 64: boxes with a 64-byte inner extent -- with the
// 128B mode the hardware pads such a box to 128-byte rows in shared memory), zero OOB fill.  dims/box innermost first; strides in bytes for dims 1..rank-1.
// `estr` (optional): element traversal strides; with stride s along a dim, box[i] = n*s loads n elements.
inline const CUtensorMap& get_map(const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides, const uint32_t* box,
                                  const uint32_t* estr = nullptr, int esize = 4, int swz = 128) {
  // node-based map: returned references stay valid; on overflow the live generation is parked in `old` (and the generation
  // before it dropped), so a reference handed out earlier in the same call can never dangle
  static std::map<MapKey, CUtensorMap> cache, old;
  static std::mutex mtx;                       // engines on different devices may encode concurrently
  std::lock_guard<std::mutex> lock(mtx);
  MapKey k;
  memset(&k, 0, sizeof(k));
  k.ptr = ptr;
  k.rank = rank;
  k.esize = esize;
  k.swz = swz;
  for (int i = 0; i < rank; ++i) { k.dims[i] = dims[i]; k.box[i] = box[i]; k.es[i] = estr ? estr[i] : 1; }
  for (int i = 0; i < rank - 1; ++i) k.strides[i] = strides[i];
  auto it = cache.find(k);
  if (it != cache.end()) return it->second;
  if (cache.size() > 65536) {
    old.clear();
    old.swap(cache);
  }
  CUtensorMap m;
  cuuint64_t gd[4];
  cuuint64_t gs[3];
  cuuint32_t bx[4], es[4];
  for (int i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; es[i] = estr ? estr[i] : 1; }
  for (int i = 0; i < rank - 1; ++i) gs[i] = strides[i];
  EncodeTiledFn enc = get_encode();
  if (!enc) throw Error(CDX_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
  CUresult r = enc(&m, esize == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<void*>(ptr), gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swz == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char b[256];
    snprintf(b, sizeof(b), "cuTensorMapEncodeTiled failed (%d): rank %d dims %llu %llu %llu %llu box %u %u %u %u", (int)r, rank,
             (unsigned long long)gd[0], (unsigned long long)(rank > 1 ? gd[1] : 0), (unsigned long long)(rank > 2 ? gd[2] : 0),
             (unsigned long long)(rank > 3 ? gd[3] : 0), bx[0], rank > 1 ? bx[1] : 0, rank > 2 ? bx[2] : 0, rank > 3 ? bx[3] : 0);
    throw Error(CDX_E_CUDA, b);
  }
  return cache.emplace(k, m).first->second;
}

inline bool pdl_enabled() {
  static const bool on = getenv("CDX_PDL") == nullptr || atoi(getenv("CDX_PDL")) != 0;      // default on; CDX_PDL=0 disables
  return on;
}
// one launch path for the kernels that take part in programmatic dependent launch (and / or need a cluster dimension)
template <typename... KArgs, typename... Args>
inline void launch_ex(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, unsigned cluster_x, Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute attr[2];
  unsigned na = 0;
  if (cluster_x > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = cluster_x; attr[na].val.clusterDim.y = 1; attr[na].val.clusterDim.z = 1;
    ++na;
  }
  if (pdl_enabled()) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr; cfg.numAttrs = na;
  CDX_CUDA(cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...));
}

inline bool a16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
inline bool pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }


}  // namespace tc
}  // namespace cdx
