// Small utility kernels.
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels/misc.cuh"

#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace bps {

namespace {

struct Blob {
  uint32_t w[256];  // 1 KiB carried in the kernel parameter space
};

// The payload travels as a by-value kernel argument: it is snapshotted at
// launch time, so the host may overwrite its copy immediately, no pinned
// buffer can be read late, and the update is ordered on the stream like any
// other kernel (used to feed optimizer hyper-parameters to captured graphs).
__global__ void write_blob_kernel(uint32_t* dst, Blob b, int nwords) {
  int i = threadIdx.x;
  if (i < nwords) dst[i] = b.w[i];
}

__global__ void l2_flush_kernel(uint4* buf, size_t n, uint32_t v) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) buf[i] = make_uint4(v, v, v, v);
}

}  // namespace

cudaError_t launch_write_blob(void* dst, const void* src, size_t nbytes, cudaStream_t stream) {
  if ((nbytes & 3) || (reinterpret_cast<uintptr_t>(dst) & 3)) return cudaErrorInvalidValue;
  const char* s = static_cast<const char*>(src);
  char* d = static_cast<char*>(dst);
  while (nbytes > 0) {
    size_t chunk = nbytes < sizeof(Blob) ? nbytes : sizeof(Blob);
    Blob b;
    memcpy(b.w, s, chunk);
    write_blob_kernel<<<1, 256, 0, stream>>>(reinterpret_cast<uint32_t*>(d), b, (int)(chunk / 4));
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    s += chunk;
    d += chunk;
    nbytes -= chunk;
  }
  return cudaSuccess;
}

namespace {
template <class T>
__global__ void scale_inplace_kernel(T* x, size_t n, float alpha) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    x[i] = (T)((float)x[i] * alpha);
}
}  // namespace

cudaError_t launch_scale_inplace(void* x, size_t n, int dtype, float alpha, cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  const int grid = (int)((n + 1023) / 1024 < 132 * 8 ? (n + 1023) / 1024 : 132 * 8);   // 8 CTAs per H100 SM
  if (dtype == 0) scale_inplace_kernel<float><<<grid, 256, 0, stream>>>((float*)x, n, alpha);
  else if (dtype == 1) scale_inplace_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>((__nv_bfloat16*)x, n, alpha);
  else if (dtype == 2) scale_inplace_kernel<__half><<<grid, 256, 0, stream>>>((__half*)x, n, alpha);
  else return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t launch_l2_flush(void* buf, size_t nbytes, uint32_t value, cudaStream_t stream) {
  l2_flush_kernel<<<132 * 4, 512, 0, stream>>>(static_cast<uint4*>(buf), nbytes / 16, value);
  return cudaGetLastError();
}

}  // namespace bps
