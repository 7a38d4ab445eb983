// Host runtime shared by the C-ABI files: error reporting, the CUDA check, the kernel launcher (which counts every
// launch gp_launch_count() reports), TMA descriptor encoders, caller-memory carving, device opening and event timing.
// Not installed.
#pragma once
#include "../../include/gigapose_b200.h"

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <utility>

namespace gp {

// Stores the formatted message gp_last_error() returns (per host thread) and returns `code`.
int fail(int code, const char* fmt, ...);

#define GP_CUDA(expr)                                                                                     \
  do {                                                                                                    \
    cudaError_t _e = (expr);                                                                              \
    if (_e != cudaSuccess) return gp::fail(GP_ERR_CUDA, "%s failed: %s", #expr, cudaGetErrorString(_e)); \
  } while (0)

// Programmatic dependent launch for launch_ex(..., pdl = true): GIGAPOSE_PDL=1 turns it on (kernels launched this way
// call pdl_wait() before touching earlier kernels' data).
bool pdl_enabled();

// Enqueues one kernel; every kernel of the library is launched through here.  Opts the kernel in to `smem` bytes of
// dynamic shared memory on the current device the first time it asks for more than 48 KiB, adds an optional thread-block
// cluster and programmatic dependent launch, counts the launch when it was enqueued, and returns the launch's own error
// (which it does not leave behind for a later cudaGetLastError()).
cudaError_t launch_kernel(const void* kernel, dim3 grid, dim3 block, size_t smem, cudaStream_t stream, int cluster_x,
                          bool pdl, void** args);

template <typename... KArgs, typename... Args>
inline cudaError_t launch_ex(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, int cluster_x,
                             bool pdl, Args&&... args) {
  return [&](KArgs... a) {                     // the arguments converted to the kernel's parameter types
    void* ptrs[] = {&a..., nullptr};
    return launch_kernel(reinterpret_cast<const void*>(kernel), grid, block, smem, stream, cluster_x, pdl, ptrs);
  }(std::forward<Args>(args)...);
}

// bf16 TMA descriptors (cuTensorMapEncodeTiled); each returns GP_OK or a gp_last_error() code.
// [rows, cols] plane (cols contiguous) with explicit box and swizzle (64 or 128 = box_cols * 2 bytes)
int make_map_ex(CUtensorMap* map, void* ptr, uint64_t rows, uint64_t cols, uint32_t box_cols, uint32_t box_rows,
                int swizzle_bytes);
// [rows, cols] plane, box = 32 columns (SWIZZLE_64B) x box_rows
int make_map(CUtensorMap* map, void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows);
// NHWC plane [N, H, W, C] as a 4-D tensor {C, W, H, N}; box = 32 channels x out_w x out_h output positions taken with
// element stride `stride` along x and y.  Coordinates outside [0,W) x [0,H) -- a convolution's zero padding -- read 0.
int make_map_nhwc(CUtensorMap* map, void* ptr, uint64_t C, uint64_t W, uint64_t H, uint64_t N, uint32_t out_w,
                  uint32_t out_h, uint32_t stride);
// caller-chosen dimensions / byte strides (rank <= 5, SWIZZLE_64B): views whose rows overlap in memory
int make_map_raw(CUtensorMap* map, void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                 const uint32_t* box, const uint32_t* elem_strides);

// Caller memory (bank, workspace, weights) must start on, and is carved in, multiples of kAlign bytes.
constexpr size_t kAlign = 1024;
inline size_t align_up(size_t x) { return (x + kAlign - 1) / kAlign * kAlign; }

// bump allocator over caller memory; with base == nullptr it only measures
struct Carver {
  uint8_t* base;
  size_t off = 0;
  explicit Carver(void* b) : base(static_cast<uint8_t*>(b)) {}
  template <typename T>
  T* take(size_t count) {
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += align_up(count * sizeof(T));
    return p;
  }
};

// Makes `device` current and checks that it is sm_90 (the library holds sm_90a code only); *num_sms = its SM count.
int open_device(int device, int* num_sms);

// Average milliseconds of `iters` calls of run() (each returning GP_OK or an error code) on `stream`, between two CUDA
// events after one warm-up call; synchronises the stream.
template <typename Run>
int time_runs(cudaStream_t stream, int iters, float* avg_ms, Run&& run) {
  struct Events {
    cudaEvent_t start = nullptr, stop = nullptr;
    ~Events() {
      if (start) cudaEventDestroy(start);
      if (stop) cudaEventDestroy(stop);
    }
  } ev;
  GP_CUDA(cudaEventCreate(&ev.start));
  GP_CUDA(cudaEventCreate(&ev.stop));
  if (int e = run()) return e;                 // warm-up
  GP_CUDA(cudaEventRecord(ev.start, stream));
  for (int i = 0; i < iters; ++i)
    if (int e = run()) return e;
  GP_CUDA(cudaEventRecord(ev.stop, stream));
  GP_CUDA(cudaEventSynchronize(ev.stop));
  float ms = 0.f;
  GP_CUDA(cudaEventElapsedTime(&ms, ev.start, ev.stop));
  *avg_ms = ms / iters;
  return GP_OK;
}

}  // namespace gp
