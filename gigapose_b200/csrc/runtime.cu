// Host runtime shared by the C-ABI files (runtime.h): error state, the launch counter, the kernel launcher, TMA
// descriptor encoders and device opening.
#include "runtime.h"

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <mutex>
#include <string>

namespace {

thread_local std::string g_last_error;
std::atomic<uint64_t> g_launches{0};

// Raises the kernel's dynamic shared memory limit to `smem` on the current device, once per (kernel, device):
// cudaFuncSetAttribute applies to the current device's context only.
cudaError_t opt_in_smem(const void* kernel, size_t smem) {
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, size_t> opted;   // (kernel, device) -> bytes opted in to
  int dev = 0;
  if (cudaError_t e = cudaGetDevice(&dev)) return e;
  std::lock_guard<std::mutex> lock(mu);
  size_t& have = opted[{kernel, dev}];
  if (have >= smem) return cudaSuccess;
  if (cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) return e;
  have = smem;
  return cudaSuccess;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
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

}  // namespace

extern "C" {
const char* gp_last_error(void) { return g_last_error.c_str(); }
uint64_t gp_launch_count(void) { return g_launches.load(); }
}

namespace gp {

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return code;
}

// Off by default: the 1-CTA-per-SM kernels hold most of the shared memory until they exit, so a dependent grid cannot
// become resident early enough to hide much more than its own prologue (not measured on H100; scripts/pdl_ab.py does).
// GIGAPOSE_PDL=1 turns it on (read at every launch).
bool pdl_enabled() {
  const char* ev = getenv("GIGAPOSE_PDL");
  return ev ? (ev[0] != '0') : false;
}

cudaError_t launch_kernel(const void* kernel, dim3 grid, dim3 block, size_t smem, cudaStream_t stream, int cluster_x,
                          bool pdl, void** args) {
  cudaError_t e = smem > 48 * 1024 ? opt_in_smem(kernel, smem) : cudaSuccess;
  if (e == cudaSuccess) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    int na = 0;
    if (cluster_x > 1) {
      attr[na].id = cudaLaunchAttributeClusterDimension;
      attr[na].val.clusterDim.x = cluster_x; attr[na].val.clusterDim.y = 1; attr[na].val.clusterDim.z = 1;
      ++na;
    }
    if (pdl && pdl_enabled()) {
      attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      attr[na].val.programmaticStreamSerializationAllowed = 1;
      ++na;
    }
    cfg.attrs = attr; cfg.numAttrs = na;
    e = cudaLaunchKernelExC(&cfg, kernel, args);
  }
  if (e == cudaSuccess) g_launches.fetch_add(1, std::memory_order_relaxed);
  else cudaGetLastError();                       // returned to the caller; not left for an unrelated later check
  return e;
}

int make_map_ex(CUtensorMap* map, void* ptr, uint64_t rows, uint64_t cols, uint32_t box_cols, uint32_t box_rows,
                int swizzle_bytes) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return fail(GP_ERR_UNSUPPORTED, "cuTensorMapEncodeTiled not available from this driver");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * sizeof(uint16_t)};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  const CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(GP_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return GP_OK;
}

int make_map(CUtensorMap* map, void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  return make_map_ex(map, ptr, rows, cols, 32, box_rows, 64);
}

// the traversal box spans out * stride input elements along x and y
int make_map_nhwc(CUtensorMap* map, void* ptr, uint64_t C, uint64_t W, uint64_t H, uint64_t N, uint32_t out_w,
                  uint32_t out_h, uint32_t stride) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return fail(GP_ERR_UNSUPPORTED, "cuTensorMapEncodeTiled not available from this driver");
  cuuint64_t dims[4] = {C, W, H, N};
  cuuint64_t strides[3] = {C * sizeof(uint16_t), W * C * sizeof(uint16_t), H * W * C * sizeof(uint16_t)};
  cuuint32_t box[4] = {32, out_w * stride, out_h * stride, 1};
  cuuint32_t estr[4] = {1, stride, stride, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(GP_ERR_CUDA, "cuTensorMapEncodeTiled (NHWC) failed with CUresult %d", (int)r);
  return GP_OK;
}

int make_map_raw(CUtensorMap* map, void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                 const uint32_t* box, const uint32_t* elem_strides) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return fail(GP_ERR_UNSUPPORTED, "cuTensorMapEncodeTiled not available from this driver");
  cuuint64_t d[5], st[4];
  cuuint32_t b[5], es[5];
  for (int i = 0; i < rank; ++i) { d[i] = dims[i]; b[i] = box[i]; es[i] = elem_strides[i]; if (i + 1 < rank) st[i] = strides_bytes[i]; }
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, ptr, d, st, b, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(GP_ERR_CUDA, "cuTensorMapEncodeTiled (raw, rank %d) failed with CUresult %d", rank, (int)r);
  return GP_OK;
}

int open_device(int device, int* num_sms) {
  GP_CUDA(cudaSetDevice(device));
  int major = 0, minor = 0;
  GP_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
  GP_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device));
  if (major != 9 || minor != 0)
    return fail(GP_ERR_UNSUPPORTED, "device %d is sm_%d%d; this library contains sm_90a code only", device, major, minor);
  GP_CUDA(cudaDeviceGetAttribute(num_sms, cudaDevAttrMultiProcessorCount, device));
  return GP_OK;
}

}  // namespace gp
