// Host-side helpers shared by the C-ABI translation units: error reporting, TMA tensor-map encoding + cache.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ih {

// error plumbing (thread-local message returned by ih_last_error())
int set_error(int code, const char* fmt, ...);
#define IH_CHECK(cond, code, ...)                       \
  do {                                                  \
    if (!(cond)) return ::ih::set_error((code), __VA_ARGS__); \
  } while (0)
#define IH_CUDA(expr)                                                                       \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess) return ::ih::set_error(-100, "%s: %s", #expr, cudaGetErrorString(_e)); \
  } while (0)

enum { IH_ERR_ARG = -1, IH_ERR_SHAPE = -2, IH_ERR_ALIGN = -3, IH_ERR_TMAP = -4, IH_ERR_CUDA = -100 };

// Encode (or fetch from the process-wide cache) a tiled fp16 tensor map with a 128-byte (default) or 64-byte swizzle
// (box rows of 64 bytes: the GEMM epilogue's 32-column output slab).
// dims[0] is the contiguous dimension; strides_bytes[i] is the byte stride of dims[i+1].
// Returns 0 on success.
int get_tmap_f16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                 const uint32_t* box, int swizzle_bytes = 128);

int num_sms();

// launch counter (all kernels launched by this library since the last reset) -- bench.py's "gpu_launches"
void count_launch(int n = 1);

// Programmatic dependent launch (PDL): every kernel of this library executes griddepcontrol.wait before it touches
// global memory, so consecutive launches may overlap the next kernel's prologue (barrier init,
// descriptor prefetch, CTA scheduling) with the previous kernel's tail.  IH_PDL=0 in the environment disables it.
bool pdl_enabled();

// Every kernel of the library asks for the maximum shared-memory carve-out, so that consecutive kernels never force
// the SMs to re-partition L1/shared memory (a drain + reconfiguration between e.g. LayerNorm and a 193 KiB GEMM).
// Returns true the first time a kernel pointer is seen.
bool first_launch_of(const void* kern);
template <typename K>
inline void prefer_max_smem_carveout(K kern) {
  if (first_launch_of(reinterpret_cast<const void*>(kern)))
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                 Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  prefer_max_smem_carveout(kern);
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
  if (e == cudaSuccess) count_launch();
  return e;
}

}  // namespace ih
