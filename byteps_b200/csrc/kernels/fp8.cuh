// FP8 casts of a row-major [M, K] bf16 / fp16 tensor (dtype: WIRE_BF16 / WIRE_F16) for the FP8 linear layers.
// M and K are multiples of 16; the input, the outputs and the bias gradient have 16-byte aligned bases.  Offsets are
// 64-bit.  Arithmetic is IEEE fp32 (the extension is not built with fast-math).
//
// A tensor's delayed-scaling state is one Fp8State in device memory, written only by these kernels:
//   s = fmax / max(max(hist), 1e-12f), fmax = 448 (E4M3) or 57344 (E5M2).
//
//   fp8_amax   read-only pass: a = max |x|.  Seeds the state: hist = {a, 0, ...}, count = 0, scale = fmax /
//              max(a, 1e-12f).  A non-finite a seeds hist = 0 and scale = NaN, so every cast before the first
//              finite one gives a NaN inverse scale.
//   fp8_cast   one pass: q = satfinite_rn(x * scale) in E4M3 or E5M2, written row-major [M, K] (FP8_ROWS),
//              transposed [K, M] (FP8_COLS) or both; the transpose goes through shared memory.  The same pass takes
//              a = max |x| (order-free) and, with dbias, the fp32 column sums of x written in the input dtype (fixed
//              order: per block, then runs of 16 blocks, then the runs, so results are bit-identical run to run).
//              Its last block writes *inv = 1 / scale (the inverse scale this call applied; NaN when a is not
//              finite) and, when a is finite, hist[count % 16] = a, ++count and the next scale from the history.
//              A non-finite a leaves the state as it was.
//              act applies an elementwise prologue to what is read, before everything above, its result rounded to
//              the input dtype first: FP8_ACT_GELU x -> gelu(x) (erf form), FP8_ACT_DGELU x -> the GELU gradient
//              dx * gelu'(z), z read from aux at the same offsets (aux: [M, K] in the input dtype, 16-byte aligned;
//              null for the other two).  FP8_ACT_GELU takes no dbias.  Both compute exactly what torch's gelu / gelu_backward kernels write, so a
//              fused cast equals the cast of the torch op's output bit for bit.
//   Both need fp8_workspace(...) floats of workspace and zeroed uint32 counters, not shared by two launches that can
//   be in flight at the same time.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace bps {

constexpr int kFp8History = 16;

struct Fp8State {
  float hist[kFp8History];
  float scale;
  uint32_t count;
};

enum Fp8Format : int { FP8_E4M3 = 0, FP8_E5M2 = 1 };
enum Fp8Layout : int { FP8_ROWS = 1, FP8_COLS = 2, FP8_BOTH = 3 };
enum Fp8Act : int { FP8_ACT_NONE = 0, FP8_ACT_GELU = 1, FP8_ACT_DGELU = 2 };

// (fp32 workspace floats, zeroed uint32 counters) of one fp8_cast (dbias or not, act) / fp8_amax launch
void fp8_cast_workspace(size_t M, int K, int dtype, int fmt, int layout, bool dbias, int act, size_t* floats,
                        int* counters);
void fp8_amax_workspace(size_t M, int K, int dtype, size_t* floats, int* counters);

cudaError_t launch_fp8_amax(const void* x, int dtype, size_t M, int K, int fmt, Fp8State* state, float* ws,
                            uint32_t* counters, cudaStream_t s);
cudaError_t launch_fp8_cast(const void* x, int dtype, size_t M, int K, int fmt, int layout, Fp8State* state,
                            void* out_rows, void* out_cols, float* inv, void* dbias, float* ws, uint32_t* counters,
                            cudaStream_t s, int act = FP8_ACT_NONE, const void* aux = nullptr);

}  // namespace bps
