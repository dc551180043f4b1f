// Do two kernels in two streams overlap on this box?  (spin kernels, 1 CTA each)
#include <cuda_runtime.h>
#include <cstdio>
__global__ void spin(long long cycles, int* sink) {
  const long long t0 = clock64();
  while (clock64() - t0 < cycles) {}
  if (sink && threadIdx.x == 9999) *sink = 1;
}
int main() {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  cudaStream_t a, b;
  cudaStreamCreateWithFlags(&a, cudaStreamNonBlocking);
  cudaStreamCreateWithFlags(&b, cudaStreamNonBlocking);
  cudaEvent_t e0, e1, eb;
  cudaEventCreate(&e0); cudaEventCreate(&e1); cudaEventCreateWithFlags(&eb, cudaEventDisableTiming);
  const long long cyc = 2000000;  // ~1 ms
  for (int rep = 0; rep < 2; ++rep) {
    cudaDeviceSynchronize();
    cudaEventRecord(e0, a);
    spin<<<1, 32, 0, a>>>(cyc, nullptr);
    spin<<<1, 32, 0, b>>>(cyc, nullptr);
    cudaEventRecord(eb, b);
    cudaStreamWaitEvent(a, eb, 0);
    cudaEventRecord(e1, a);
    cudaDeviceSynchronize();
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    printf("two streams, 1 CTA each: %.3f ms (1 kernel ~ %.3f ms)\n", ms, cyc / 1.98e6);
  }
  // full-machine persistent kernel (3 CTAs per SM x 256 threads spinning) + small kernel on the other stream
  cudaDeviceSynchronize();
  cudaEventRecord(e0, a);
  spin<<<sms * 3, 256, 0, a>>>(cyc, nullptr);
  spin<<<sms, 128, 0, b>>>(cyc, nullptr);
  cudaEventRecord(eb, b);
  cudaStreamWaitEvent(a, eb, 0);
  cudaEventRecord(e1, a);
  cudaDeviceSynchronize();
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  printf("3 x SMs x 256 + SMs x 128 in two streams: %.3f ms\n", ms);
  const char* e = getenv("CUDA_DEVICE_MAX_CONNECTIONS");
  printf("CUDA_DEVICE_MAX_CONNECTIONS=%s CUDA_LAUNCH_BLOCKING=%s\n", e ? e : "(unset)", getenv("CUDA_LAUNCH_BLOCKING") ? getenv("CUDA_LAUNCH_BLOCKING") : "(unset)");
  return 0;
}
