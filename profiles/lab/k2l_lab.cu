// k2l_lab.cu — standalone timing / bit-compare harness for the dominant kernel (K2L, rate) and the series-offset stage.
// Not product code: it includes the product's kernel headers from the tree given with -I and launches them the way
// b2p_range.cu does, on the BASELINE config-2 chunk shape, so that kernel variants can be compared in one run
// without the Python stack.  Prints one line per run:
//   tag S ms_k0 ms_k2l ms_step checksum_out checksum_valid handed_off
// Two binaries built from two source trees agree bit for bit iff their checksums agree.
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "b2p_kernel_lean.cuh"
#ifdef LAB_K2U
#include "k2u_experiment.cuh"
#endif

using namespace b2p;

#define CK(x)                                                                          \
  do {                                                                                 \
    cudaError_t e__ = (x);                                                             \
    if (e__ != cudaSuccess) {                                                          \
      fprintf(stderr, "%s: %s (%s:%d)\n", #x, cudaGetErrorString(e__), __FILE__, __LINE__); \
      exit(1);                                                                         \
    }                                                                                  \
  } while (0)

__global__ void checksum_kernel(const unsigned long long* p, size_t n, unsigned long long* acc) {
  unsigned long long h = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    h += p[i] * (2ull * i + 1ull) + (p[i] >> 29);
  for (int o = 16; o > 0; o >>= 1) h += __shfl_down_sync(0xffffffffu, h, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(acc, h);
}
__global__ void checksum32_kernel(const uint32_t* p, size_t n, unsigned long long* acc) {
  unsigned long long h = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    h += (unsigned long long)p[i] * (2ull * i + 1ull);
  for (int o = 16; o > 0; o >>= 1) h += __shfl_down_sync(0xffffffffu, h, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(acc, h);
}

#ifndef LAB_FN
#define LAB_FN 0
#endif
#ifndef LAB_FLAGS
#define LAB_FLAGS false
#endif

int main(int argc, char** argv) {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  const char* tag = argc > 1 ? argv[1] : "lab";
  const uint32_t S = argc > 2 ? (uint32_t)atoll(argv[2]) : 1250000u;
  const int iters = argc > 3 ? atoi(argv[3]) : 10;
  const int resets = argc > 4 ? atoi(argv[4]) : 0;
  const uint32_t jitter = argc > 5 ? (uint32_t)atoi(argv[5]) : 1000u;
  const uint32_t N = 1000;
  const int64_t T0 = 1700000000000ll, scrape = 15000, range = 300000;
  const size_t n_rows = (size_t)S * N;
  const int64_t T = N;
  const uint32_t Tw = (uint32_t)((T + 31) / 32);
  int64_t* ts; double* val; uint32_t* sid; uint64_t* offsets; double* out; uint32_t* valid; Status* status;
  uint32_t *w_list, *slow_list; unsigned long long* d_sum;
  CK(cudaMalloc(&ts, n_rows * 8)); CK(cudaMalloc(&val, n_rows * 8)); CK(cudaMalloc(&sid, n_rows * 4));
  CK(cudaMalloc(&offsets, ((size_t)S + 1) * 8)); CK(cudaMalloc(&out, (size_t)S * T * 8));
  CK(cudaMalloc(&valid, (size_t)S * Tw * 4)); CK(cudaMalloc(&status, sizeof(Status)));
  CK(cudaMalloc(&w_list, (size_t)S * 4)); CK(cudaMalloc(&slow_list, (size_t)S * 4)); CK(cudaMalloc(&d_sum, 16));
  CK(cudaMemset(status, 0, sizeof(Status)));
  CK(cudaMemset(out, 0xff, (size_t)S * T * 8));
  CK(cudaMemset(valid, 0xff, (size_t)S * Tw * 4));
  cudaStream_t st;
  CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  synth_fill_kernel<<<sms * 32, 256, 0, st>>>(0, S, N, T0, scrape, jitter, resets, 0x5EEDull, ts, val, sid);
  CK(cudaGetLastError());

  RangeArgs a{};
  a.start = T0; a.end = T0 + (N - 1) * scrape; a.interval = scrape; a.range = range; a.offset = 0;
  a.p0 = 0; a.p1 = 0; a.filter_nan = 1; a.T = T; a.Tw = Tw; a.tb = a.start - a.range;
  a.rel_max = (uint32_t)(a.range + (T - 1) * a.interval + 1);
  const double rs = (double)range / 1000.0;
  a.rcp_rs = 1.0 / rs; a.range_secs = rs; a.rcp_interval = 1.0 / (double)a.interval;
  a.start_mod = (uint32_t)(a.start % a.interval);
  a.ts = ts; a.val = val; a.offsets = offsets; a.n_rows = n_rows; a.n_series = S; a.out = out; a.valid = valid;
  a.status = status; a.slow_list = slow_list; a.w_list = w_list; a.use_w_list = 0;
#ifndef LAB_REF
  a.b_list = nullptr;
#endif

#ifndef LAB_UNI
#define LAB_UNI false
#endif
  auto kern = range_lean_kernel<LAB_FN, LAB_FLAGS, false, LAB_UNI>;
  if (LAB_UNI) CK(cudaMemset(&status->uniform, 1, 4));
#ifdef LAB_REF
  constexpr int kLeanWarps = kWarpsPerCta;
  constexpr size_t smem = (size_t)kWarpsPerCta * kLeanRing * 16 + kRcpTable * 8 + (size_t)kWarpsPerCta * 2 * 64 * 16 +
                          (size_t)kWarpsPerCta * (kLeanRing / 32) * 4;
#else
  constexpr size_t smem = lean_smem_bytes(LAB_UNI);
#endif
  CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int nb = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, kLeanWarps * 32, smem));
  cudaFuncAttributes fa;
  CK(cudaFuncGetAttributes(&fa, kern));
  const unsigned need = (S + kLeanWarps - 1) / kLeanWarps;
  if (getenv("LAB_K2L_CTAS_PER_SM")) nb = atoi(getenv("LAB_K2L_CTAS_PER_SM"));
  const unsigned cap = (unsigned)sms * (unsigned)(nb > 0 ? nb : 1);
  const unsigned grid = need < cap ? need : cap;

  auto run_k0 = [&]() {
    uint64_t blocks = (n_rows / 16 + 255) / 256;
    if (blocks > (uint64_t)sms * 16) blocks = (uint64_t)sms * 16;
    series_offsets_kernel<<<(unsigned)blocks, 256, 0, st>>>(sid, n_rows, S, 0u, offsets, status);
  };
#ifdef LAB_K2U
  auto ukern = range_uniform_kernel<LAB_FN>;
  int unb = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&unb, ukern, kUniWarps * 32, 0));
  CK(cudaFuncGetAttributes(&fa, ukern));
  nb = unb;
  CK(cudaMemset(&status->uniform, 1, 4));
  const unsigned uneed = (S + kUniWarps - 1) / kUniWarps;
  const unsigned ucap = (unsigned)sms * (unsigned)(getenv("LAB_K2U_CTAS_PER_SM") ? atoi(getenv("LAB_K2U_CTAS_PER_SM")) : unb);
  const unsigned ugrid = uneed < ucap ? uneed : ucap;
  auto run_k2l = [&]() {
    cudaMemsetAsync(&status->w_count, 0, 4, st);
    ukern<<<ugrid, kUniWarps * 32, 0, st>>>(a);
  };
#else
  auto run_k2l = [&]() {
    cudaMemsetAsync(&status->w_count, 0, 4, st);
    kern<<<grid, kLeanWarps * 32, smem, st>>>(a);
  };
#endif
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  auto timeit = [&](auto f) {
    for (int i = 0; i < 3; ++i) f();
    CK(cudaStreamSynchronize(st));
    CK(cudaEventRecord(e0, st));
    for (int i = 0; i < iters; ++i) f();
    CK(cudaEventRecord(e1, st));
    CK(cudaStreamSynchronize(st));
    CK(cudaGetLastError());
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    return ms / iters;
  };
  const float ms_k0 = timeit(run_k0);
  const float ms_k2l = timeit(run_k2l);
#if 0  /* K0 split experiment (search + validate kernels), dropped: see DESIGN.md */
  // K0 split: lower_bound search on the main stream, full-column validation on a side stream next to K2L
  cudaStream_t side;
  CK(cudaStreamCreateWithFlags(&side, cudaStreamNonBlocking));
  cudaEvent_t ev_in, ev_done;
  CK(cudaEventCreateWithFlags(&ev_in, cudaEventDisableTiming));
  CK(cudaEventCreateWithFlags(&ev_done, cudaEventDisableTiming));
  auto run_search = [&]() {
    series_offsets_search_kernel<<<(S + 1 + 255) / 256, 256, 0, st>>>(sid, n_rows, S, 0u, offsets);
  };
  const int val_ctas = getenv("LAB_VAL_CTAS") ? atoi(getenv("LAB_VAL_CTAS")) : sms;
  const int val_thr = getenv("LAB_VAL_THREADS") ? atoi(getenv("LAB_VAL_THREADS")) : 128;
  auto run_validate = [&](cudaStream_t s_) { series_validate_kernel<<<val_ctas, val_thr, 0, s_>>>(sid, n_rows, S, 0u, status); };
  // kernels whose shared-memory carve-out preferences differ cannot share an SM: ask for the same (maximum) carve-out
  CK(cudaFuncSetAttribute(series_validate_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  CK(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  const float ms_search = timeit(run_search);
  const float ms_val = timeit([&]() { run_validate(st); });
  CK(cudaMemsetAsync(offsets, 0, ((size_t)S + 1) * 8, st));
  const float ms_step = timeit([&]() {
    cudaEventRecord(ev_in, st);
    cudaStreamWaitEvent(side, ev_in, 0);
#if LAB_OVERLAP == 1
    run_validate(side);
    cudaEventRecord(ev_done, side);
    run_search();
    run_k2l();
#else
    run_search();
    run_k2l();
    run_validate(side);
    cudaEventRecord(ev_done, side);
#endif
    cudaStreamWaitEvent(st, ev_done, 0);
  });
  printf("   search=%.3f ms validate(alone)=%.3f ms\n", ms_search, ms_val);
  {  // one more overlapped step with events around each kernel: who runs when?
    cudaEvent_t t0, tv0, tv1, tk0, tk1, tend;
    for (cudaEvent_t* e : {&t0, &tv0, &tv1, &tk0, &tk1, &tend}) CK(cudaEventCreate(e));
    CK(cudaStreamSynchronize(st));
    CK(cudaEventRecord(t0, st));
    cudaStreamWaitEvent(side, t0, 0);
    CK(cudaEventRecord(tv0, side));
    run_validate(side);
    CK(cudaEventRecord(tv1, side));
    run_search();
    CK(cudaEventRecord(tk0, st));
    run_k2l();
    CK(cudaEventRecord(tk1, st));
    cudaStreamWaitEvent(st, tv1, 0);
    CK(cudaEventRecord(tend, st));
    CK(cudaStreamSynchronize(st));
    CK(cudaStreamSynchronize(side));
    float v0, v1, k0_, k1_, te_;
    cudaEventElapsedTime(&v0, t0, tv0); cudaEventElapsedTime(&v1, t0, tv1);
    cudaEventElapsedTime(&k0_, t0, tk0); cudaEventElapsedTime(&k1_, t0, tk1); cudaEventElapsedTime(&te_, t0, tend);
    printf("   timeline (ms from step start): validate [%.3f, %.3f]  k2l [%.3f, %.3f]  end %.3f\n", v0, v1, k0_, k1_, te_);
  }
#else
  const float ms_step = timeit([&]() { run_k0(); run_k2l(); });
#endif
  Status hs;
  CK(cudaMemcpy(&hs, status, sizeof hs, cudaMemcpyDeviceToHost));
  unsigned long long sums[2] = {0, 0};
  CK(cudaMemset(d_sum, 0, 16));
  checksum_kernel<<<sms * 8, 256, 0, st>>>(reinterpret_cast<const unsigned long long*>(out), (size_t)S * T, d_sum);
  checksum32_kernel<<<sms * 8, 256, 0, st>>>(valid, (size_t)S * Tw, d_sum + 1);
  CK(cudaStreamSynchronize(st));
  CK(cudaMemcpy(sums, d_sum, 16, cudaMemcpyDeviceToHost));
  unsigned long long off_sum = 0;
  CK(cudaMemset(d_sum, 0, 16));
  checksum_kernel<<<sms * 8, 256, 0, st>>>(reinterpret_cast<const unsigned long long*>(offsets), (size_t)S + 1, d_sum);
  CK(cudaStreamSynchronize(st));
  CK(cudaMemcpy(&off_sum, d_sum, 8, cudaMemcpyDeviceToHost));
  printf("   offsets=%016llx\n", off_sum);
  const double gs = (double)n_rows / (ms_step * 1e-3) / 1e9;
  printf("%-28s S=%u regs=%d ctas/sm=%d k0=%.3f k2l=%.3f step=%.3f ms  %.1f Gsamples/s  read_frac=%.3f  out=%016llx valid=%016llx handed=%u k0err=%u\n",
         tag, S, fa.numRegs, nb, ms_k0, ms_k2l, ms_step, gs, 20.0 * n_rows / (ms_step * 1e-3) / 1e9 / 3350.0, sums[0], sums[1],
         hs.w_count, hs.k0_errors);
  return 0;
}
