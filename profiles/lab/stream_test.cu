// stream_test.cu — what does the memory system give a kernel with K2's traffic mix (read ts i64 + val f64, write out f64,
// 24 B per element) when the access pattern is ideal (grid-stride, fully contiguous), and with per-warp private rows
// (warp w streams row w of [S x 1000] the way a warp-per-series kernel does)?
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#define CK(x) do { cudaError_t e__ = (x); if (e__ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e__)); exit(1);} } while (0)

__global__ void contiguous(const long long* __restrict__ ts, const double* __restrict__ val, double* __restrict__ out, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = val[i] * (double)(ts[i] & 3);
}
template <int U>
__global__ void per_warp_rows(const long long* __restrict__ ts, const double* __restrict__ val, double* __restrict__ out, unsigned S, int N) {
  const int lane = threadIdx.x & 31;
  const unsigned warps = gridDim.x * (blockDim.x >> 5);
  for (unsigned s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < S; s += warps) {
    const size_t base = (size_t)s * N;
    for (int j = 0; j < N; j += 32 * U) {
      long long t[U]; double v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) { const int i = j + 32 * u + lane; t[u] = i < N ? ts[base + i] : 0; v[u] = i < N ? val[base + i] : 0.0; }
#pragma unroll
      for (int u = 0; u < U; ++u) { const int i = j + 32 * u + lane; if (i < N) out[base + i] = v[u] * (double)(t[u] & 3); }
    }
  }
}
// the same with K2U's extras switched on one by one: X&1 second read of val 19 rows back, X&2 of the predecessor,
// X&4 one validity word per chunk, X&8 per-row dependent set-up loads (offsets -> first / last timestamp, last value)
template <int U, int X>
__global__ void rows_extras(const long long* __restrict__ ts, const double* __restrict__ val, double* __restrict__ out,
                            const unsigned long long* __restrict__ offsets, unsigned* __restrict__ vw, unsigned S, int N) {
  const int lane = threadIdx.x & 31;
  const unsigned warps = gridDim.x * (blockDim.x >> 5);
  for (unsigned s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < S; s += warps) {
    size_t base = (size_t)s * N;
    double bias = 0.0;
    if (X & 8) {
      base = offsets[s];
      const size_t end = offsets[s + 1];
      bias = (double)((ts[base] + ts[end - 1]) & 1) + val[end - 1];
    }
    for (int j = 0; j < N; j += 32 * U) {
      long long t[U]; double v[U], f[U], p[U];
#pragma unroll
      for (int u = 0; u < U; ++u) { const int i = j + 32 * u + lane; t[u] = i < N ? ts[base + i] : 0; v[u] = i < N ? val[base + i] : 0.0; }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int i = j + 32 * u + lane;
        f[u] = ((X & 1) && i >= 19 && i < N) ? val[base + i - 19] : 0.0;
        p[u] = ((X & 2) && i >= 1 && i < N) ? val[base + i - 1] : 0.0;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int i = j + 32 * u + lane;
        if (i < N) out[base + i] = (v[u] - f[u]) * (double)(t[u] & 3) + p[u] + bias;
        if ((X & 4) && lane == 0) vw[(size_t)s * 32 + ((j >> 5) + u)] = 0xffffffffu;
      }
    }
  }
}
// K2U's streaming loop with the neighbours taken out of the warp instead of out of the cache: M = 1 shuffles (the asked
// lane provides v or the chunk before), M = 2 a per-warp shared-memory ring of the values; validity words kept in a
// register and stored once per row; per-row dependent set-up loads as in rows_extras<.., 8>.
template <int U, int M>
__global__ void rows_neighbours(const long long* __restrict__ ts, const double* __restrict__ val, double* __restrict__ out,
                                const unsigned long long* __restrict__ offsets, unsigned* __restrict__ vw, unsigned S, int N) {
  __shared__ double ring[8][2 * U * 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned warps = gridDim.x * (blockDim.x >> 5);
  const int back = 19;
  const int src_f = (lane - back) & 31, src_p = (lane - 1) & 31;
  const bool same_f = lane + back < 32;
  for (unsigned s = blockIdx.x * (blockDim.x >> 5) + warp; s < S; s += warps) {
    const size_t base = offsets[s];
    const size_t end = offsets[s + 1];
    const double bias = (double)((ts[base] + ts[end - 1]) & 1) + val[end - 1];
    double carry = 0.0;
    unsigned acc = 0;
    int slot = 0;
    for (int j = 0; j < N; j += 32 * U) {
      long long t[U]; double v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) { const int i = j + 32 * u + lane; t[u] = i < N ? ts[base + i] : 0; v[u] = i < N ? val[base + i] : 0.0; }
      if (M == 2) {
#pragma unroll
        for (int u = 0; u < U; ++u) ring[warp][slot * U * 32 + 32 * u + lane] = v[u];
        __syncwarp();
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int i = j + 32 * u + lane;
        double f, p;
        if (M == 1) {
          const double before = u == 0 ? carry : v[u - 1];
          f = __shfl_sync(0xffffffffu, same_f ? v[u] : before, src_f);
          p = __shfl_sync(0xffffffffu, lane == 31 ? before : v[u], src_p);
        } else {
          const int pos = slot * U * 32 + 32 * u + lane;
          f = ring[warp][(pos - back) & (2 * U * 32 - 1)];
          p = ring[warp][(pos - 1) & (2 * U * 32 - 1)];
        }
        if (i < N) out[base + i] = (v[u] - f) * (double)(t[u] & 3) + p + bias;
        if (lane == (((j >> 5) + u) & 31)) acc = 0xffffffffu;
      }
      carry = v[U - 1];
      slot ^= 1;
      if (M == 2) __syncwarp();
    }
    vw[(size_t)s * 32 + lane] = acc;
  }
}
int main(int argc, char** argv) {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  const unsigned S = 1250000; const int N = 1000; const size_t n = (size_t)S * N;
  long long* ts; double *val, *out;
  CK(cudaMalloc(&ts, n * 8)); CK(cudaMalloc(&val, n * 8)); CK(cudaMalloc(&out, n * 8));
  CK(cudaMemset(ts, 1, n * 8)); CK(cudaMemset(val, 0, n * 8));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  auto timeit = [&](const char* tag, auto f) {
    for (int i = 0; i < 2; ++i) f();
    CK(cudaEventRecord(e0)); for (int i = 0; i < 5; ++i) f(); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); ms /= 5; CK(cudaGetLastError());
    printf("%-32s %.3f ms  %.2f TB/s\n", tag, ms, 24.0 * n / (ms * 1e-3) / 1e12);
  };
  timeit("contiguous SMx8x256", [&] { contiguous<<<sms * 8, 256>>>(ts, val, out, n); });
  timeit("contiguous SMx4x512", [&] { contiguous<<<sms * 4, 512>>>(ts, val, out, n); });
  unsigned long long* offsets; unsigned* vw;
  CK(cudaMalloc(&offsets, ((size_t)S + 1) * 8)); CK(cudaMalloc(&vw, (size_t)S * 32 * 4));
  {
    unsigned long long* h = (unsigned long long*)malloc(((size_t)S + 1) * 8);
    for (size_t i = 0; i <= S; ++i) h[i] = i * N;
    CK(cudaMemcpy(offsets, h, ((size_t)S + 1) * 8, cudaMemcpyHostToDevice)); free(h);
  }
  timeit("extras 0", [&] { rows_extras<4, 0><<<sms * 4, 256>>>(ts, val, out, offsets, vw, S, N); });
  timeit("extras 1 (first)", [&] { rows_extras<4, 1><<<sms * 4, 256>>>(ts, val, out, offsets, vw, S, N); });
  timeit("extras 3 (first+prev)", [&] { rows_extras<4, 3><<<sms * 4, 256>>>(ts, val, out, offsets, vw, S, N); });
  timeit("extras 4 (vw)", [&] { rows_extras<4, 4><<<sms * 4, 256>>>(ts, val, out, offsets, vw, S, N); });
  timeit("extras 8 (setup)", [&] { rows_extras<4, 8><<<sms * 4, 256>>>(ts, val, out, offsets, vw, S, N); });
  timeit("extras 7 (first+prev+vw)", [&] { rows_extras<4, 7><<<sms * 4, 256>>>(ts, val, out, offsets, vw, S, N); });
  timeit("extras 15 (all)", [&] { rows_extras<4, 15><<<sms * 4, 256>>>(ts, val, out, offsets, vw, S, N); });
  timeit("extras 15 (all) U=2 x6", [&] { rows_extras<2, 15><<<sms * 6, 256>>>(ts, val, out, offsets, vw, S, N); });
  timeit("neighbours shuffle U=4 x4", [&] { rows_neighbours<4, 1><<<sms * 4, 256>>>(ts, val, out, offsets, vw, S, N); });
  timeit("neighbours smem    U=4 x4", [&] { rows_neighbours<4, 2><<<sms * 4, 256>>>(ts, val, out, offsets, vw, S, N); });
  timeit("neighbours shuffle U=2 x6", [&] { rows_neighbours<2, 1><<<sms * 6, 256>>>(ts, val, out, offsets, vw, S, N); });
  timeit("neighbours smem    U=2 x6", [&] { rows_neighbours<2, 2><<<sms * 6, 256>>>(ts, val, out, offsets, vw, S, N); });
  for (int ctas : {4}) {
    char tag[64];
    snprintf(tag, 64, "rows U=1 %dx256", ctas); timeit(tag, [&] { per_warp_rows<1><<<sms * ctas, 256>>>(ts, val, out, S, N); });
    snprintf(tag, 64, "rows U=2 %dx256", ctas); timeit(tag, [&] { per_warp_rows<2><<<sms * ctas, 256>>>(ts, val, out, S, N); });
    snprintf(tag, 64, "rows U=4 %dx256", ctas); timeit(tag, [&] { per_warp_rows<4><<<sms * ctas, 256>>>(ts, val, out, S, N); });
    snprintf(tag, 64, "rows U=8 %dx256", ctas); timeit(tag, [&] { per_warp_rows<8><<<sms * ctas, 256>>>(ts, val, out, S, N); });
  }
  return 0;
}
