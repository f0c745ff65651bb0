// Host-side plumbing of libttsb.so: thread-local error text, launch counter, cuTensorMapEncodeTiled lookup.
#include <stdarg.h>
#include <stdio.h>

#include <atomic>

#include "../../include/ttsb.h"
#include "ttsb_host.h"

namespace ttsb {

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return 0;
  set_last_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
  return TTSB_ERR_CUDA;
}

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

int current_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return dev;
}

int num_sms() {
  static PerDevice<int> sms;
  int& n = sms.get();
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, current_device()) != cudaSuccess || n <= 0) n = 132;  // H100 SXM
  }
  return n;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

static int encode(CUtensorMap* out, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                  const cuuint32_t* box, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
  EncodeTiledFn fn = get_encode();
  if (!fn) {
    set_last_error("cuTensorMapEncodeTiled is not available from the driver");
    return TTSB_ERR_CUDA;
  }
  if (reinterpret_cast<uintptr_t>(base) & 15) {
    set_last_error("TMA base pointer %p is not 16-byte aligned", base);
    return TTSB_ERR_INVALID_ARGUMENT;
  }
  for (int i = 0; i + 1 < rank; ++i) {
    if (strides_bytes[i] & 15) {
      set_last_error("TMA stride %llu is not a multiple of 16 bytes", (unsigned long long)strides_bytes[i]);
      return TTSB_ERR_INVALID_ARGUMENT;
    }
  }
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes, box,
                  estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu,%llu box %u,%u)", (int)r, rank,
                   (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
    return TTSB_ERR_CUDA;
  }
  return 0;
}

int make_tmap_bf16_3d(CUtensorMap* out, const void* base, uint64_t dim0, uint64_t dim1, uint64_t dim2, uint64_t stride1,
                      uint64_t stride2, uint32_t box0, uint32_t box1) {
  const cuuint64_t dims[3] = {dim0, dim1, dim2};
  const cuuint64_t strides[2] = {stride1 * 2, stride2 * 2};
  const cuuint32_t box[3] = {box0, box1, 1};
  return encode(out, base, 3, dims, strides, box);
}

int make_tmap_bf16_3d_sw64(CUtensorMap* out, const void* base, uint64_t dim0, uint64_t dim1, uint64_t dim2, uint64_t stride1,
                           uint64_t stride2, uint32_t box0, uint32_t box1) {
  const cuuint64_t dims[3] = {dim0, dim1, dim2};
  const cuuint64_t strides[2] = {stride1 * 2, stride2 * 2};
  const cuuint32_t box[3] = {box0, box1, 1};
  return encode(out, base, 3, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_64B);
}

int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t dim0, uint64_t dim1, uint64_t stride1, uint32_t box0,
                      uint32_t box1) {
  const cuuint64_t dims[2] = {dim0, dim1};
  const cuuint64_t strides[1] = {stride1 * 2};
  const cuuint32_t box[2] = {box0, box1};
  return encode(out, base, 2, dims, strides, box);
}

}  // namespace ttsb

extern "C" const char* ttsb_last_error(void) { return ttsb::g_err; }
extern "C" int ttsb_abi_version(void) { return TTSB_ABI_VERSION; }
extern "C" int64_t ttsb_launch_count(void) { return ttsb::g_launches.load(); }
extern "C" void ttsb_reset_launch_count(void) { ttsb::g_launches.store(0); }
extern "C" void ttsb_add_launch_count(int64_t n) { ttsb::g_launches.fetch_add(n, std::memory_order_relaxed); }

extern "C" int ttsb_set_dropout_salt(const uint32_t* salt_dev, void* stream) {
  if (!salt_dev) { ttsb::set_last_error("ttsb_set_dropout_salt: salt_dev is NULL"); return TTSB_ERR_INVALID_ARGUMENT; }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int rc = ttsb::set_salt_gemm(salt_dev, s);
  if (!rc) rc = ttsb::set_salt_rowops(salt_dev, s);
  if (!rc) rc = ttsb::set_salt_train_ops(salt_dev, s);
  if (!rc) rc = ttsb::set_salt_bgemm(salt_dev, s);
  if (!rc) rc = ttsb::set_salt_attn_probs(salt_dev, s);
  return rc;
}
