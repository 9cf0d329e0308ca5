// sc16_harness.cu -- TEST INFRASTRUCTURE: the sc16 sample conversion of csrc/rx_common.cuh (RawSc16::cvt),
// unchanged, on every int16 value (tests/test_sc16.py), and a throughput comparison of the two exact int16 -> float forms
// it could use.  Built by gen2_uhf_rfid_reader_b200.build.build_harness with the library's nvcc flags.
//
// Every entry point takes device pointers, runs on the default stream and returns a cudaError_t.
#include <cuda_runtime.h>

#include "rx_common.cuh"

using namespace rfid_b200;

#define SH_API extern "C" __attribute__((visibility("default")))

namespace {

// word i (0 <= i < 65536) holds I = i - 32768 in the low half-word and Q = ~I in the high one, so both halves see every
// int16 value; out[s][i] = RawSc16::cvt(word, scales[s])
__global__ void cvt_kernel(const float* scales, int nscale, float2* out)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 65536) return;
  const uint32_t lo = (uint32_t)(i - 32768) & 0xFFFFu;
  const uint32_t w = lo | ((~lo & 0xFFFFu) << 16);
  for (int s = 0; s < nscale; s++) out[(size_t)s * 65536 + i] = RawSc16::cvt(w, scales[s]);
}

// the two exact forms of (float)i for an int16 i: I2F (RawSc16::cvt), and a full-rate integer add and float subtract --
// 0x4B400000 + i is the float 1.5 * 2^23 + i, whose ulp is 1, for |i| < 2^22
template <int V>
__device__ __forceinline__ float to_f32(int i)
{
  if (V == 0) return (float)i;
  return __fsub_rn(__int_as_float(0x4B400000 + i), 12582912.0f);
}

// throughput: every thread converts and scales both halves of `iters` pseudo-random words (an LCG, the same for both
// forms) and folds them into a sum that is stored, so nothing is optimised away
template <int V>
__global__ void rate_kernel(int iters, float scale, float* sink)
{
  uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
  float acc0 = 0.f, acc1 = 0.f;
#pragma unroll 8
  for (int k = 0; k < iters; k++) {
    w = w * 1664525u + 1013904223u;
    const int i = (int)(w << 16) >> 16, q = (int)w >> 16;
    acc0 = f_add(acc0, f_mul(to_f32<V>(i), scale));
    acc1 = f_add(acc1, f_mul(to_f32<V>(q), scale));
  }
  sink[blockIdx.x * blockDim.x + threadIdx.x] = f_add(acc0, acc1);
}

}  // namespace

SH_API int sc16_harness_convert(const float* d_scales, int nscale, float* d_out)
{
  cvt_kernel<<<65536 / 256, 256>>>(d_scales, nscale, reinterpret_cast<float2*>(d_out));
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  return (int)e;
}

// form 0 = (float)i, 1 = the integer add + float subtract; d_sink holds blocks * 256 floats.  *ms: the best of `reps` launches
SH_API int sc16_harness_rate(int form, int blocks, int iters, int reps, float* d_sink, float* ms)
{
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  float best = 1e30f;
  cudaError_t e = cudaSuccess;
  for (int r = 0; r < reps && e == cudaSuccess; r++) {
    cudaEventRecord(a);
    if (form == 0) rate_kernel<0><<<blocks, 256>>>(iters, 1.0f / 32767.0f, d_sink);
    else rate_kernel<1><<<blocks, 256>>>(iters, 1.0f / 32767.0f, d_sink);
    cudaEventRecord(b);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaEventSynchronize(b);
    float t = 0.f;
    if (e == cudaSuccess && r > 0 && cudaEventElapsedTime(&t, a, b) == cudaSuccess && t < best) best = t;   // r = 0 warms up
  }
  cudaEventDestroy(a);
  cudaEventDestroy(b);
  *ms = best;
  return (int)e;
}
