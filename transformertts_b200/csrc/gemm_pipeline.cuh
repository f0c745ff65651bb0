// The TMA -> wgmma pipeline shared by the tensor-core GEMM kernels (gemm_tc.cu: Dense / concat-projection / Conv1D,
// bgemm_tc.cu: the batched products and weight gradients of the training step).  A persistent CTA of 384 threads:
//   warp 8      TMA producer: fills a ring of k-block stages (128B-swizzled A [128 x 64] and B [block_n x 64] tiles);
//               control flow is warp-uniform and the elected lane issues (see elect_one)
//   warps 0-7   two wgmma warpgroups, rows [64*wg, +64) of the tile, fp32 accumulators in registers.  Once the ring is
//               drained they park the tile in it as an accumulator image and run the epilogue from there, one thread per
//               output row: warp (quarter = warp & 3, half = warp >> 2) owns rows [32*quarter, +32) and one half of the
//               tile's 16-column chunks, so two warps per SM sub-partition hide each other's latencies
//   warps 9-11  idle: the producer warpgroup hands its registers to the others with setmaxnreg
// The producer refills the ring only after the epilogue has released the previous tile's image (no double buffering).
// A kernel supplies the TMA loads of a stage, the wgmma products of a k block and its epilogue.  16-bit outputs leave
// through staging boxes in the ring (stage_out_offset, staged_slab_begin / _end) as TMA tile stores: a thread owns one
// output ROW, so direct stores are 32-byte pieces of 32 different rows per warp instruction (request-rate bound).
#pragma once
#include <cuda_bf16.h>

#include "ttsb_common.cuh"
#include "ttsb_host.h"
#include "wgmma_sm90.cuh"

namespace ttsb {

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;
constexpr int GEMM_MAX_BN = 256;
constexpr int GEMM_THREADS = 384;
constexpr int GEMM_EPI_WARPS = 8;                        // the consumer / epilogue warps
constexpr int GEMM_NCH = GEMM_MAX_BN / 64;               // wgmma n64 products per k step (the tile width rounded up to 64)
constexpr int A_TILE_BYTES = GEMM_BM * GEMM_BK * 2;      // 16 KiB
constexpr int B_TILE_BYTES = GEMM_MAX_BN * GEMM_BK * 2;  // 32 KiB
constexpr int MN_BOX_BYTES = 64 * 128;                   // one [64 k x 64 mn] TMA box of an MN-major operand
// accumulator image [128 rows][acc_pitch(max_bn) floats]: written once the ring is drained, so it overlays the ring
__host__ __device__ constexpr int img_bytes(int max_bn) { return GEMM_BM * acc_pitch(max_bn) * 4; }
// staged 16-bit stores: two boxes x four row quarters of [32 rows x 64 cols] (4 KiB, 128B swizzle), in the ring behind the image
__host__ __device__ constexpr int stage_out_offset(int max_bn) { return (img_bytes(max_bn) + 1023) / 1024 * 1024; }
constexpr int STAGE_OUT_BYTES = 2 * 4 * 4096;

__device__ __forceinline__ uint8_t* align_smem_1024(uint8_t* p) {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~(uintptr_t)1023);
}
// named barriers: 5 = the 256 consumer threads, 1 + quarter = the two warps of a row quarter
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 5, 256;" ::: "memory"); }
__device__ __forceinline__ void quarter_sync(int quarter) { asm volatile("bar.sync %0, 64;" ::"r"(1 + quarter) : "memory"); }

// Ring of kStages stages at the (1024-aligned) shared-memory base, followed by GEMM_RING_BAR_BYTES of barriers: full[s]
// completes when stage s has landed (one arrival + the TMA bytes), empty[s] when the 8 consumer warps are done reading it,
// img_free when the epilogue has released the previous tile's image.  Every thread constructs its own GemmRing: the producer
// and the consumers each advance their own copy of the position (img_phase / first are the producer's only).
constexpr int GEMM_RING_BAR_BYTES = 256;
template <int kStages, int kStageBytes>
struct GemmRing {
  static constexpr int kBytes = kStages * kStageBytes;
  static_assert((2 * kStages + 1) * 8 <= GEMM_RING_BAR_BYTES, "ring barriers");
  uint8_t* smem;
  uint64_t* full;
  int stage = 0;
  uint32_t phase = 0;
  uint32_t img_phase = 0;  // producer: parity of the next img_free completion
  bool first = true;       // producer: no image to wait for before the first tile

  __device__ explicit GemmRing(uint8_t* base) : smem(base), full(reinterpret_cast<uint64_t*>(base + kBytes)) {}
  __device__ uint64_t* empty() const { return full + kStages; }
  __device__ uint64_t* img_free() const { return full + 2 * kStages; }
  __device__ void init() const {  // one thread, before the fence / __syncthreads that publish the barriers
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full + s, 1);
      mbar_init(empty() + s, GEMM_EPI_WARPS);
    }
    mbar_init(img_free(), 1);
  }
  __device__ __forceinline__ void advance() {
    if (++stage == kStages) { stage = 0; phase ^= 1; }
  }

  // producer, start of a tile: the ring holds the previous tile's accumulator image until its epilogue is done
  __device__ __forceinline__ void wait_image_free() {
    if (!first) {
      mbar_wait(img_free(), img_phase);
      img_phase ^= 1;
    }
    first = false;
  }
  // producer: wait for the next slot to be empty, arm it for tx bytes and let the elected lane issue load(full barrier, slot)
  template <class Load>
  __device__ __forceinline__ void produce(bool leader, uint32_t tx, Load&& load) {
    mbar_wait(empty() + stage, phase ^ 1);
    uint8_t* st = smem + stage * kStageBytes;
    if (leader) {
      mbar_arrive_expect_tx(full + stage, tx);
      load(full + stage, st);
    }
    advance();
  }

  // consumers: the kbs k blocks of a tile.  issue(stage shared address, kb) issues the wgmma products of k block kb
  // (accumulate flag off for the first products of kb 0).  A stage is released once the products of the next k block are
  // in flight (their predecessors have finished reading it), the last one after the drain.
  template <int NCH, class Issue>
  __device__ __forceinline__ void mma_tile(int kbs, float (&acc)[NCH][32], Issue&& issue) {
    const bool lane0 = (threadIdx.x & 31) == 0;
    int prev_stage = -1;
    for (int kb = 0; kb < kbs; ++kb) {
      mbar_wait(full + stage, phase);
      wgmma_fence();
      issue(smem_u32(smem + stage * kStageBytes), kb);
      wgmma_commit();
      wgmma_wait<1>();
      if (prev_stage >= 0) {
        __syncwarp();
        if (lane0) mbar_arrive(empty() + prev_stage);
      }
      prev_stage = stage;
      advance();
    }
    wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < NCH; ++c) wgmma_fence_regs(acc[c]);
    if (prev_stage >= 0) {
      __syncwarp();
      if (lane0) mbar_arrive(empty() + prev_stage);
    }
  }

  // consumers, end of a tile: the staging boxes and the image lie in the ring, so the TMA stores must have read them (the
  // lane that issued them waits) and the generic-proxy writes are ordered before the producer's refill
  __device__ __forceinline__ void release_tile(bool store_issuer) const {
    if (store_issuer) tma_store_wait_read();
    fence_proxy_async_smem();
    consumer_sync();
    if (threadIdx.x == 0) mbar_arrive(img_free());
  }
  // consumers, end of the kernel: staged stores fully written out before exit
  __device__ __forceinline__ static void finish(bool store_issuer) {
    if (store_issuer) tma_store_wait_all();
  }
};

// consumers: both warpgroups are done reading the ring; park the tile in it (n64 blocks c < nmma; the rest was not computed)
template <int NCH>
__device__ __forceinline__ void park_tile(float* img, int pitch, int wg, int nmma, const float (&acc)[NCH][32]) {
  consumer_sync();
#pragma unroll
  for (int c = 0; c < NCH; ++c)
    if (c < nmma) acc_store_fragment(img, pitch, wg * 64, c * 64, acc[c]);
  consumer_sync();
}

// bf16 of 16 floats, packed pairwise with cvt.rn.bf16x2; pack_hi_lo adds lo = bf16(y - hi)
__device__ __forceinline__ void pack_hi(const float (&y)[16], uint32_t (&h)[8]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const __nv_bfloat162 hh = __floats2bfloat162_rn(y[2 * j], y[2 * j + 1]);
    h[j] = *reinterpret_cast<const uint32_t*>(&hh);
  }
}
__device__ __forceinline__ void pack_hi_lo(const float (&y)[16], uint32_t (&h)[8], uint32_t (&l)[8], bool want_lo) {
  pack_hi(y, h);
  if (want_lo) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float f0 = __uint_as_float(h[j] << 16), f1 = __uint_as_float(h[j] & 0xffff0000u);
      const __nv_bfloat162 ll = __floats2bfloat162_rn(y[2 * j] - f0, y[2 * j + 1] - f1);
      l[j] = *reinterpret_cast<const uint32_t*>(&ll);
    }
  }
}

// one 16-column chunk (32 bytes) into row lrow of a 128B-swizzled [32 x 64] 16-bit box: 16-byte pieces k0 and k0 + 1 of
// the 128-byte row, piece index ^= lrow & 7
__device__ __forceinline__ void st_box_chunk(uint8_t* box, int lrow, int k0, const uint32_t (&h)[8]) {
  const uint32_t o0 = lrow * 128 + ((k0 ^ (lrow & 7)) << 4), o1 = lrow * 128 + (((k0 + 1) ^ (lrow & 7)) << 4);
  st_shared_v4(box + o0, h[0], h[1], h[2], h[3]);
  st_shared_v4(box + o1, h[4], h[5], h[6], h[7]);
}

// A 64-column slab of a staged 16-bit epilogue, run by the two warps of a row quarter once they hold their image chunks.
// Each fills a [32 rows x 64 cols] 128B-swizzled box per plane (warp `half` writes chunks 2*half, 2*half + 1 with
// st_box_chunk) between staged_slab_begin and staged_slab_end; then the issuing lane hands the boxes to the TMA unit.
// Two planes use boxes A (hi) and B (lo) on every slab, so the previous slab's stores must have been read out; one plane
// alternates A and B, so only the store issued two slabs ago must have been.  Returns the hi box; the lo box is B.
__device__ __forceinline__ uint8_t* staged_slab_lo_box(uint8_t* stage_out, int quarter) { return stage_out + 4 * 4096 + quarter * 4096; }
__device__ __forceinline__ uint8_t* staged_slab_begin(uint8_t* stage_out, int quarter, bool issuer, bool two, uint32_t& slab_ctr) {
  uint8_t* box_a = stage_out + quarter * 4096;
  uint8_t* box_b = staged_slab_lo_box(stage_out, quarter);
  uint8_t* box_hi = two ? box_a : ((slab_ctr & 1u) ? box_b : box_a);
  ++slab_ctr;
  if (issuer) {
    if (two) tma_store_wait_read(); else tma_store_wait_read_but_one();
  }
  quarter_sync(quarter);
  return box_hi;
}
// the boxes are written: store(box_hi) issues the slab's TMA store(s) on the issuing lane, which then commits them
template <class Store>
__device__ __forceinline__ void staged_slab_end(int quarter, bool issuer, Store&& store) {
  fence_proxy_async_smem();
  quarter_sync(quarter);
  if (issuer) {
    store();
    tma_store_commit();
  }
}

// Launches a pipeline kernel persistently: min(work, SMs) CTAs, or with `pair` min(work, SMs / 2) clusters of two CTAs.
// The shared-memory limit is raised once per device and kernel.
template <auto kKernel, class... Args>
int launch_pipeline(int smem_bytes, int work, bool pair, cudaStream_t stream, const char* what, const Args&... args) {
  static PerDevice<bool> attr_set;
  if (!attr_set.get()) {
    TTSB_CUDA_OK(cudaFuncSetAttribute(kKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    attr_set.get() = true;
  }
  const int cta_per_item = pair ? 2 : 1, slots = num_sms() / cta_per_item;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(cta_per_item * (work < slots ? work : slots));
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = stream;
  cudaLaunchAttribute cluster{};
  cluster.id = cudaLaunchAttributeClusterDimension;
  cluster.val.clusterDim.x = 2;
  cluster.val.clusterDim.y = 1;
  cluster.val.clusterDim.z = 1;
  cfg.attrs = &cluster;
  cfg.numAttrs = pair ? 1 : 0;
  TTSB_CUDA_OK(cudaLaunchKernelEx(&cfg, kKernel, args...));
  count_launch();
  return check_cuda(cudaGetLastError(), what);
}

}  // namespace ttsb
