// engine.cu -- per-device context: workspace arena, error state.
#include <cstdarg>
#include <cstdio>

#include "common.cuh"

namespace cdx {

static thread_local std::string g_last_error;
void set_last_error(const std::string& m) { g_last_error = m; }
const std::string& last_error() { return g_last_error; }

// Stack allocator over one device slab.  Every top-level ABI call first replays its op sequence in `dry` mode
// (no launches, no memory touched) to learn the high-water mark, grows the slab if needed, then runs for real --
// so steady-state calls never touch cudaMalloc and the slab size is exact.
void* Arena::alloc(size_t bytes) {
  bytes = (bytes + 255) & ~(size_t)255;
  void* p = nullptr;
  if (dry) {
    p = reinterpret_cast<void*>((uintptr_t)0x1000 + off);   // never dereferenced
  } else {
    if (off + bytes > cap) throw Error(CDX_E_NOMEM, "arena: allocation beyond the dry-run high-water mark (engine bug)");
    p = base + off;
  }
  off += bytes;
  if (off > high) high = off;
  return p;
}

void Arena::begin_dry() { dry = true; off = 0; high = 0; }

void Arena::end_dry() {
  dry = false;
  off = 0;
  if (high > cap) {
    cudaDeviceSynchronize();   // earlier calls may still be using the old slab
    if (base) cudaFree(base);
    base = nullptr;
    cap = 0;
    const size_t want = high + (1u << 20);
    cudaError_t err = cudaMalloc(&base, want);
    if (err != cudaSuccess) throw Error(CDX_E_NOMEM, std::string("arena cudaMalloc(") + std::to_string(want) + ") failed: " + cudaGetErrorString(err));
    cap = want;
  }
}

ProfScope::ProfScope(Engine& eng, cudaStream_t st, int tag, double flops, double bytes, int launches) : e(eng), s(st) {
  if (!e.prof.on || e.dry()) return;
  ProfRec r;
  cudaEventCreate(&r.a);
  cudaEventCreate(&r.b);
  r.tag = tag; r.flops = flops; r.bytes = bytes; r.launches = launches;
  r.note[0] = 0;
  cudaEventRecord(r.a, s);
  idx = (int)e.prof.recs.size();
  e.prof.recs.push_back(r);
}
void ProfScope::note(const char* fmt, ...) {
  if (idx < 0) return;
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(e.prof.recs[idx].note, sizeof(e.prof.recs[idx].note), fmt, ap);
  va_end(ap);
}
ProfScope::~ProfScope() {
  if (idx >= 0) cudaEventRecord(e.prof.recs[idx].b, s);
}

// A pool is created by the first network call that needs it, in the middle of enqueueing that call.  cudaMemset runs on the legacy
// default stream, which a non-blocking stream does not wait for: the target U-Net of a two-engine lock-step loop runs on such a
// stream (PairStreams), and its kernels would accumulate into the pool while the memset clears it.  Wait for the zeroing once.
static void wait_pool_zeroed() {
  const cudaError_t err = cudaDeviceSynchronize();
  if (err != cudaSuccess) throw Error(CDX_E_CUDA, std::string("pool zeroing: ") + cudaGetErrorString(err));
}

float* Engine::amax_slot() {
  if (dry()) return reinterpret_cast<float*>((uintptr_t)0x100);   // never dereferenced
  if (!amax_pool) {
    if (cudaMalloc(&amax_pool, (size_t)amax_cap * sizeof(float)) != cudaSuccess) throw Error(CDX_E_NOMEM, "amax pool allocation failed");
    if (cudaMemset(amax_pool, 0, (size_t)amax_cap * sizeof(float)) != cudaSuccess) throw Error(CDX_E_CUDA, "amax pool memset failed");
    wait_pool_zeroed();
  }
  if (amax_used >= amax_cap) throw Error(CDX_E_NOMEM, "amax pool exhausted (engine bug: amax_reset not called per network call)");
  return amax_pool + amax_used++;
}
double* Engine::stat_alloc(size_t n) {
  n = (n + 31) & ~(size_t)31;
  if (dry()) { stat_dry += n; return reinterpret_cast<double*>((uintptr_t)0x1000); }   // never dereferenced
  if (!stat_pool) {
    if (cudaMalloc(&stat_pool, stat_cap * sizeof(double)) != cudaSuccess) throw Error(CDX_E_NOMEM, "statistics pool allocation failed");
    if (cudaMemset(stat_pool, 0, stat_cap * sizeof(double)) != cudaSuccess) throw Error(CDX_E_CUDA, "statistics pool memset failed");
    wait_pool_zeroed();
  }
  if (stat_used + n > stat_cap) throw Error(CDX_E_NOMEM, "statistics pool exhausted");
  double* p = stat_pool + stat_used;
  stat_used += n;
  return p;
}
// Both pools are fully zero when created; a call dirties [0, used), so zeroing [0, high-water) keeps everything beyond clean.
void Engine::pools_reset(cudaStream_t s) {
  if (dry()) return;
  if (amax_used > amax_high) amax_high = amax_used;
  if (stat_used > stat_high) stat_high = stat_used;
  if (amax_pool && amax_high) cudaMemsetAsync(amax_pool, 0, (size_t)amax_high * sizeof(float), s);
  if (stat_pool && stat_high) cudaMemsetAsync(stat_pool, 0, stat_high * sizeof(double), s);
  amax_high = 0; stat_high = 0;
  amax_used = 0; stat_used = 0;
}

void Arena::destroy() {
  if (base) cudaFree(base);
  base = nullptr;
  cap = off = high = 0;
}

}  // namespace cdx
