// Developer aid: cabsf_quick (+ its risky flag) against cabsf_ref on the GPU: random inputs over many magnitude
// ranges, the rounding-boundary neighbourhoods, zeros.  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -fmad=false
//   -o tools/micro/cabs_check tools/micro/cabs_check.cu ; run on the GPU box.  Prints mismatches (must be 0) and the risky rate.
#include <cstdio>
#include <cstdint>
#include "../../gen2_uhf_rfid_reader_b200/csrc/rx_common.cuh"
using namespace rfid_b200;

__device__ unsigned long long splitmix(unsigned long long& x)
{
  unsigned long long z = (x += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

__global__ void check(unsigned long long seed, int iters, int mode, unsigned long long* bad, unsigned long long* risky_n,
                      unsigned long long* unflagged_bad)
{
  unsigned long long st = seed + 0x1234567ull * (blockIdx.x * blockDim.x + threadIdx.x);
  unsigned long long nb = 0, nr = 0, nu = 0;
  for (int i = 0; i < iters; i++) {
    const unsigned long long r1 = splitmix(st), r2 = splitmix(st);
    float re, im;
    if (mode == 0) {            // magnitudes like the matched filter's output (|y| up to ~1e3), arbitrary mantissas
      re = __uint_as_float(((unsigned)r1 & 0x807FFFFFu) | ((100u + (unsigned)(r1 >> 40) % 40u) << 23));
      im = __uint_as_float(((unsigned)r2 & 0x807FFFFFu) | ((100u + (unsigned)(r2 >> 40) % 40u) << 23));
    } else if (mode == 1) {     // any finite float bit pattern (including subnormals, zeros)
      re = __uint_as_float((unsigned)r1);
      im = __uint_as_float((unsigned)r2);
      if (!isfinite(re)) re = 0.f;
      if (!isfinite(im)) im = 0.f;
    } else {                    // one component tiny or zero
      re = __uint_as_float(((unsigned)r1 & 0x807FFFFFu) | ((120u + (unsigned)(r1 >> 40) % 16u) << 23));
      im = (r2 & 1) ? 0.f : __uint_as_float(((unsigned)r2 & 0x807FFFFFu) | ((60u + (unsigned)(r2 >> 40) % 60u) << 23));
    }
    bool risky;
    const float q = cabsf_quick(re, im, risky);
    const float e = cabsf_ref(re, im);
    const float f = risky ? e : q;
    if (__float_as_uint(f) != __float_as_uint(e)) nb++;
    if (!risky && __float_as_uint(q) != __float_as_uint(e)) nu++;
    if (risky) nr++;
  }
  atomicAdd(bad, nb);
  atomicAdd(risky_n, nr);
  atomicAdd(unflagged_bad, nu);
}

int main()
{
  unsigned long long *d, h[3];
  cudaMalloc(&d, 24);
  for (int mode = 0; mode < 3; mode++) {
    cudaMemset(d, 0, 24);
    const int blocks = 148 * 8, threads = 256, iters = mode == 0 ? 16384 : 4096;
    check<<<blocks, threads>>>(42 + mode, iters, mode, d, d + 1, d + 2);
    cudaDeviceSynchronize();
    cudaMemcpy(h, d, 24, cudaMemcpyDeviceToHost);
    const double n = (double)blocks * threads * iters;
    printf("mode %d: %.3g samples, mismatches after fallback %llu, unflagged mismatches %llu, risky rate %.3g\n", mode, n, h[0],
           h[2], h[1] / n);
  }
  return 0;
}
