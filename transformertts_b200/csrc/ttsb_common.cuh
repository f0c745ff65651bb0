// Shared device helpers for the sm_90a kernels: mbarrier, TMA, wgmma shared-memory matrix descriptors and the
// shared-memory accumulator image of the GEMM epilogues (the wgmma instructions themselves are in wgmma_sm90.cuh).
// Everything is inline PTX; no CUTLASS dependency.  Compile with -gencode arch=compute_90a,code=sm_90a.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ttsb {

// ------------------------------------------------------------------------------------------------
// error plumbing (host)
// ------------------------------------------------------------------------------------------------
void set_last_error(const char* fmt, ...);
int check_cuda(cudaError_t e, const char* what);

#define TTSB_CUDA_OK(expr)                                  \
  do {                                                      \
    int _rc = ::ttsb::check_cuda((expr), #expr);            \
    if (_rc != 0) return _rc;                               \
  } while (0)

// ------------------------------------------------------------------------------------------------
// small device utilities
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ void split_bf16(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(v);
  lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}
__device__ __forceinline__ uint32_t pack_bf16(__nv_bfloat16 a, __nv_bfloat16 b) {
  return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}

// The clip of a packed ragged batch that holds item x: the largest c in [0, n) with tab[c] <= x, for a non-decreasing
// prefix table tab (device memory) with tab[0] <= x
__device__ __forceinline__ int find_clip(const int32_t* __restrict__ tab, int n, int x) {
  int lo = 0, hi = n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(tab + mid) <= x) lo = mid; else hi = mid;
  }
  return lo;
}

// Stateless dropout decision shared by forward and backward kernels: keep element `idx` of dropout site `site` when the
// 32-bit mix of (seed, site, idx) is >= thresh = p * 2^32 (keras Dropout semantics: kept values are scaled by 1/(1-p)).
// c_drop_salt (one copy per translation unit, zero unless a host sets it with ttsb_set_dropout_salt) is XORed into the seed:
// a training step captured as a CUDA graph has its `seed` arguments frozen at capture, so the per-step variation comes from
// this device-resident word, refreshed by memcpy nodes at the head of the graph.
static __constant__ uint32_t c_drop_salt = 0;
// One 32-bit hash serves TWO consecutive elements (16 bits each; the rate is resolved to 2^-16): the per-element cost of the
// mask is a large share of the per-element work of the attention-probability kernels of the training step.
// hash(pair) = mix((uint32)pair * C1 ^ hterm(seed, site, pair >> 32)).  Kernels that walk consecutive pairs hoist hterm and
// step the first term by C1 per pair (dropout_hterm / dropout_mix below) instead of redoing the 64-bit index arithmetic.
constexpr uint32_t DROPOUT_C1 = 0x9E3779B1u;
__device__ __forceinline__ uint32_t dropout_hterm(uint32_t seed, uint32_t site, uint32_t pair_hi) {
  seed ^= c_drop_salt;
  return pair_hi * 0x85EBCA77u ^ seed * 0xC2B2AE3Du ^ site * 0x27D4EB2Fu;
}
__device__ __forceinline__ uint32_t dropout_mix(uint32_t x) {
  x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15; x *= 0x846CA68Bu; x ^= x >> 16;
  return x;
}
__device__ __forceinline__ uint32_t dropout_hash(uint32_t seed, uint32_t site, uint64_t pair) {
  return dropout_mix((uint32_t)pair * DROPOUT_C1 ^ dropout_hterm(seed, site, (uint32_t)(pair >> 32)));
}
__device__ __forceinline__ bool dropout_keep(uint32_t seed, uint32_t site, uint64_t idx, uint32_t thresh) {
  const uint32_t h = dropout_hash(seed, site, idx >> 1);
  return ((idx & 1) ? (h >> 16) : (h & 0xffffu)) >= (thresh >> 16);
}
// decisions for elements idx_even and idx_even + 1 (idx_even must be even) from one hash
__device__ __forceinline__ void dropout_keep2(uint32_t seed, uint32_t site, uint64_t idx_even, uint32_t thresh, bool& k0, bool& k1) {
  const uint32_t h = dropout_hash(seed, site, idx_even >> 1);
  k0 = (h & 0xffffu) >= (thresh >> 16);
  k1 = (h >> 16) >= (thresh >> 16);
}
__host__ __device__ __forceinline__ uint32_t dropout_thresh(float p) { return p > 0.f ? (uint32_t)((double)p * 4294967296.0) : 0u; }

// Every translation unit that draws dropout decisions defines one of these (TTSB_DEFINE_SALT_SETTER(name)); host.cu calls
// them all from ttsb_set_dropout_salt.
#define TTSB_DEFINE_SALT_SETTER(name)                                                                           \
  namespace ttsb {                                                                                              \
  int name(const uint32_t* salt_dev, cudaStream_t stream) {                                                     \
    return check_cuda(cudaMemcpyToSymbolAsync(c_drop_salt, salt_dev, sizeof(uint32_t), 0, cudaMemcpyDeviceToDevice, stream), #name); \
  }                                                                                                             \
  }

// ------------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("{\n.reg .b64 st;\nmbarrier.arrive.shared::cta.b64 st, [%0];\n}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("{\n.reg .b64 st;\nmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n}" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n.reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Spin-wait with a hang guard: a broken pipeline traps after 2^28 polls instead of hanging the GPU box.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins == 0x10000000u) { asm volatile("trap;"); }
  }
}
// The same with a suspend-time hint: the hardware parks the warp until the phase completes (or the hint expires) instead of
// re-issuing the poll, which leaves the issue slots to the other warps of the scheduler.  Used by attn_probs_tc.cu, whose
// softmax warpgroups wait for K tiles while sharing schedulers with each other; the GEMM kernels keep the polling wait above
// for their pipeline barriers.
__device__ __forceinline__ void mbar_wait_parked(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  for (;;) {
    uint32_t ok;
    asm volatile(
        "{\n.reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n"
        "selp.u32 %0, 1, 0, p;\n}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(20000u)
        : "memory");
    if (ok) return;
    if (++spins == 0x4000000u) { asm volatile("trap;"); }
  }
}
// 16-byte store to shared memory through its 32-bit shared address: a store through a generic pointer derived from the
// dynamic-smem base compiles to a generic ST.E (address-space resolution in the LSU) instead of STS
__device__ __forceinline__ void st_shared_v4(void* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(smem_u32(p)), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

// ------------------------------------------------------------------------------------------------
// fences
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ------------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor, tile mode, mbarrier completion)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// shared -> global tile store (bulk async group); rows / columns outside the tensor are clipped by the TMA unit
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, const void* src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all committed bulk stores of this thread have finished READING shared memory (the buffers may be rewritten)
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// ... all but the most recent committed group have finished reading (double-buffered staging)
__device__ __forceinline__ void tma_store_wait_read_but_one() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
// ... have completed (global writes performed)
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ------------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptors (sm_90 format)
// ------------------------------------------------------------------------------------------------
// K-major operand tile stored as rows of 128 bytes (64 bf16) with the 128-byte swizzle TMA writes
// (CU_TENSOR_MAP_SWIZZLE_128B): 8-row groups are 1024 B apart (SBO), LBO is unused for swizzled K-major layouts (set to 1),
// layout type 1 (SWIZZLE_128B) in bits [62,64).  The tile base must be 1024-byte aligned; advancing K by 16 elements adds
// 32 bytes to the start address (+2 in descriptor units).
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);       // start address, bits [0,14)
  d |= (uint64_t)1 << 16;                        // leading byte offset (ignored), bits [16,30)
  d |= (uint64_t)(1024 >> 4) << 32;              // stride byte offset = 1024 B, bits [32,46)
  d |= (uint64_t)1 << 62;                        // SWIZZLE_128B
  return d;
}
// MN-major operand (the M or N index is contiguous: each 128-byte row holds 64 m/n for ONE k): the tile is stored as
// blocks of [64 k rows x 64 mn] (what a TMA box of 64 x 64 bf16 with the 128B swizzle writes); LBO = byte distance between
// consecutive 64-wide blocks along M/N, SBO = 1024 B between groups of 8 k rows.  Advancing K by 16 adds 2048 B.
__device__ __forceinline__ uint64_t make_smem_desc_mn_sw128(uint32_t saddr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)(lbo_bytes >> 4) << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// Register budget hand-over between warpgroups (the producer warpgroup of a warp-specialised kernel needs few registers,
// the wgmma warpgroups hold their accumulators in registers)
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// One lane of a fully converged warp.  The TMA issuing warps run their role code warp-uniformly and predicate only the
// issuing instructions on this, so every operand stays in uniform registers.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n.reg .pred p;\nelect.sync _|p, 0xffffffff;\nselp.u32 %0, 1, 0, p;\n}" : "=r"(pred));
  return pred != 0;
}

// ------------------------------------------------------------------------------------------------
// Accumulator image: the GEMM kernels park a finished 128 x N fp32 tile in shared memory as rows of ACC_PITCH(N) floats
// so that their epilogues run one thread per output row.  A pitch of N + 4 floats (N % 16 == 0) keeps the 16-byte row
// accesses of eight consecutive rows in distinct banks.
// ------------------------------------------------------------------------------------------------
__host__ __device__ constexpr int acc_pitch(int n) { return n + 4; }
// the wgmma accumulator fragment of one 64 x N warpgroup product (see wgmma_sm90.cuh) -> image rows [row0, row0 + 64)
template <int R>
__device__ __forceinline__ void acc_store_fragment(float* img, int pitch, int row0, int col0, const float (&d)[R]) {
  const int t = threadIdx.x & 127;
  const int r = row0 + 16 * (t >> 5) + ((t & 31) >> 2);
  const int c = col0 + 2 * (t & 3);
#pragma unroll
  for (int i = 0; i < R / 4; ++i) {
    *reinterpret_cast<float2*>(img + (size_t)r * pitch + c + 8 * i) = make_float2(d[4 * i], d[4 * i + 1]);
    *reinterpret_cast<float2*>(img + (size_t)(r + 8) * pitch + c + 8 * i) = make_float2(d[4 * i + 2], d[4 * i + 3]);
  }
}
// 16 consecutive floats of one image row (16-byte aligned)
__device__ __forceinline__ void acc_ld16(const float* p, uint32_t (&r)[16]) {
  const uint32_t s = smem_u32(p);
#pragma unroll
  for (int j = 0; j < 4; ++j)
    asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(r[4 * j]), "=r"(r[4 * j + 1]), "=r"(r[4 * j + 2]), "=r"(r[4 * j + 3])
                 : "r"(s + 16 * j) : "memory");
}
__device__ __forceinline__ void acc_st16(float* p, const uint32_t (&r)[16]) {
  const uint32_t s = smem_u32(p);
#pragma unroll
  for (int j = 0; j < 4; ++j)
    asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(s + 16 * j), "r"(r[4 * j]), "r"(r[4 * j + 1]), "r"(r[4 * j + 2]),
                 "r"(r[4 * j + 3]) : "memory");
}

// 32-byte global stores / loads as two 16-byte accesses (one full sector per lane)
__device__ __forceinline__ void st_global_v4(void* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.global.v4.b32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void st_global_v8(void* p, const uint32_t (&v)[8]) {
  st_global_v4(p, v[0], v[1], v[2], v[3]);
  st_global_v4(static_cast<uint8_t*>(p) + 16, v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ void st_global_v8f(float* p, const float* v) {
  asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]) : "memory");
  asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p + 4), "f"(v[4]), "f"(v[5]), "f"(v[6]), "f"(v[7]) : "memory");
}
__device__ __forceinline__ void ld_global_nc_v8f(const float* p, float* v) {
  asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v[0]), "=f"(v[1]), "=f"(v[2]), "=f"(v[3]) : "l"(p));
  asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v[4]), "=f"(v[5]), "=f"(v[6]), "=f"(v[7]) : "l"(p + 4));
}
__device__ __forceinline__ void ld_global_nc_v8(const void* p, uint32_t (&v)[8]) {
  const uint8_t* q = static_cast<const uint8_t*>(p);
  asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "l"(q));
  asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v[4]), "=r"(v[5]), "=r"(v[6]), "=r"(v[7]) : "l"(q + 16));
}

}  // namespace ttsb
