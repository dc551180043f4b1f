// b2p_context.cu — C ABI of libb200promql.so (see include/b200promql.h): the context (create / destroy, streams,
// counters, errors) and the NCCL communicator of the multi-GPU all-reduce.  The operators live in the other b2p_*.cu
// files; b2p_runtime.cuh is what they share.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>

#include "b2p_runtime.cuh"

using namespace b2p;

namespace {
thread_local std::string g_err;
}  // namespace

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

Nccl g_nccl;

// error of a non-zero Status::k0_errors word
int k0_fail(uint32_t k0) {
  if (k0 & kBinRowError) return fail(B2P_E_INVALID, "binary operator: a pair's row index is out of range");
  if (k0 & kSetKeyError) return fail(B2P_E_INVALID, "set operator: a row's key is >= n_keys");
  if (k0 & kScalarKeyError) return fail(B2P_E_INVALID, "scalar(): a row's series key is >= n_rows");
  if (k0 & kScalarOverlapError)
    return fail(B2P_E_INVALID, "scalar(): two rows of one series have a cell at the same step");
  if (k0 & kStepRangeError)
    return fail(B2P_E_INVALID, "step function: an eval timestamp's year is outside [-262143, 262143]");
  if (k0 & 1u) return fail(B2P_E_UNSORTED, "series-id column is not non-decreasing");
  return fail(B2P_E_UNSORTED, "series id >= n_series");
}

extern "C" {

const char* b2p_last_error(void) { return g_err.c_str(); }
const char* b2p_version(void) { return "b200promql 0.1 (sm_90a)"; }

int64_t b2p_num_steps(int64_t start, int64_t end, int64_t interval) {
  if (interval <= 0 || end < start) return 0;
  return (end - start) / interval + 1;
}

b2p_ctx* b2p_create(int device) {
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    fail(B2P_E_CUDA, "no CUDA device: %s — libb200promql has no CPU fallback", cudaGetErrorString(e));
    cudaGetLastError();
    return nullptr;
  }
  if (device < 0 || device >= ndev) {
    fail(B2P_E_INVALID, "device %d out of range (have %d)", device, ndev);
    return nullptr;
  }
  b2p_ctx* c = new (std::nothrow) b2p_ctx();
  if (!c) {
    fail(B2P_E_NOMEM, "out of host memory");
    return nullptr;
  }
  c->device = device;
  DeviceGuard g(device);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) c->num_sms = prop.multiProcessorCount;
  bool ok = cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking) == cudaSuccess;
  c->stream = c->own_stream;
  ok = ok && cudaMalloc(&c->d_ring, kStatusSlots * sizeof(Status)) == cudaSuccess;
  ok = ok && cudaMallocHost(&c->h_ring, kStatusSlots * sizeof(Status)) == cudaSuccess;
  ok = ok && cudaMalloc(&c->d_k0, sizeof(Status)) == cudaSuccess;
  ok = ok && cudaMallocHost(&c->h_k0, sizeof(Status)) == cudaSuccess;
  for (int i = 0; ok && i < 5; ++i)
    for (int j = 0; j < 2; ++j) ok = ok && cudaEventCreate(&c->ev[i][j]) == cudaSuccess;
  if (!ok) {
    fail(B2P_E_CUDA, "context creation failed: %s", cudaGetErrorString(cudaGetLastError()));
    b2p_destroy(c);
    return nullptr;
  }
  cudaMemset(c->d_ring, 0, kStatusSlots * sizeof(Status));
  cudaMemset(c->d_k0, 0, sizeof(Status));
  if (upload_rcp_table() != B2P_OK) {
    b2p_destroy(c);
    return nullptr;
  }
  if (const char* e = getenv("B2P_ENABLE_THREAD_TIER")) c->thread_tier = (e[0] == '1');
  if (const char* e = getenv("B2P_DISABLE_LEAN_TIER")) c->lean_tier = !(e[0] == '1');
  if (const char* e = getenv("B2P_LEAN_ADAPTIVE")) c->lean_adaptive = !(e[0] == '0');
  if (const char* e = getenv("B2P_LEAN_FORCE_FLAGS")) c->lean_force_flags = (e[0] == '1');
  if (const char* e = getenv("B2P_HOST_TS_SCAN")) c->host_ts_scan = (e[0] != '0');
  if (const char* e = getenv("B2P_UNIFORM")) c->uniform_mode = (e[0] == '0') ? 0 : (e[0] == '1' ? 1 : -1);
  if (const char* e = getenv("B2P_COMM_RESERVE_SMS")) c->comm_reserve_sms = atoi(e);
  if (const char* e = getenv("B2P_COMM_HEADSTART_US")) c->comm_headstart_cycles = (long long)(atof(e) * 1980.0);
  if (const char* e = getenv("B2P_ARENA_ROWS")) c->arena_rows_wanted = (size_t)strtoull(e, nullptr, 10);
  if (const char* e = getenv("B2P_TOPK_EXCHANGE_BYTES")) c->topk_exchange_cap = (size_t)strtoull(e, nullptr, 10);
  return c;
}

void b2p_destroy(b2p_ctx* c) {
  if (!c) return;
  DeviceGuard g(c->device);
  if (c->own_stream) cudaStreamSynchronize(c->own_stream);
  if (c->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(c->comm);
  if (c->s_comm) cudaStreamDestroy(c->s_comm);
  if (c->ev_comm_in) cudaEventDestroy(c->ev_comm_in);
  if (c->ev_comm_done) cudaEventDestroy(c->ev_comm_done);
  if (c->ev_comm_go) cudaEventDestroy(c->ev_comm_go);
  for (int i = 0; i < 5; ++i)
    for (int j = 0; j < 2; ++j)
      if (c->ev[i][j]) cudaEventDestroy(c->ev[i][j]);
  for (int i = 0; i < 2; ++i) {
    if (c->ev_h2d[i]) cudaEventDestroy(c->ev_h2d[i]);
    if (c->ev_comp[i]) cudaEventDestroy(c->ev_comp[i]);
    if (c->ev_d2h[i]) cudaEventDestroy(c->ev_d2h[i]);
  }
  if (c->s_h2d) cudaStreamDestroy(c->s_h2d);
  if (c->s_d2h) cudaStreamDestroy(c->s_d2h);
  if (c->d_ring) cudaFree(c->d_ring);
  if (c->h_ring) cudaFreeHost(c->h_ring);
  if (c->d_k0) cudaFree(c->d_k0);
  if (c->h_k0) cudaFreeHost(c->h_k0);
  if (c->own_stream) cudaStreamDestroy(c->own_stream);
  delete c;  // frees the device scratch (DevBuf members) on the context's device
}

int b2p_set_stream(b2p_ctx* c, void* cuda_stream) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  c->stream = reinterpret_cast<cudaStream_t>(cuda_stream);  // NULL == the legacy default stream
  return B2P_OK;
}

int b2p_use_own_stream(b2p_ctx* c) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  c->stream = c->own_stream;
  return B2P_OK;
}

int64_t b2p_last_slow_series(b2p_ctx* c) { return c ? c->last_slow : -1; }
int64_t b2p_last_h2d_bytes(b2p_ctx* c) { return c ? c->last_h2d_bytes : -1; }
int64_t b2p_last_exchange_bytes(b2p_ctx* c) { return c ? c->last_exchange_bytes : -1; }
int64_t b2p_last_group_keys_bytes(b2p_ctx* c) { return c ? c->last_group_keys_bytes : -1; }
int64_t b2p_last_warp_tier_series(b2p_ctx* c) { return c ? c->last_w : -1; }
int64_t b2p_launch_count(b2p_ctx* c) { return c ? c->launches : -1; }

double b2p_last_kernel_ms(b2p_ctx* c, int stage) {
  if (!c || stage < 0 || stage >= 5 || !c->ev_used[stage]) return -1.0;
  DeviceGuard g(c->device);
  float ms = -1.f;
  if (cudaEventElapsedTime(&ms, c->ev[stage][0], c->ev[stage][1]) != cudaSuccess) {
    cudaGetLastError();
    return -1.0;
  }
  return (double)ms;
}

/* ---- multi-GPU: the NCCL communicator and the exchanges of the sharded operators ----------------- */

int b2p_comm_unique_id(void* out_id, size_t bytes) {
  if (!out_id || bytes < sizeof(Nccl::unique_id)) return fail(B2P_E_INVALID, "need a %zu-byte buffer", sizeof(Nccl::unique_id));
  if (!g_nccl.load()) return fail(B2P_E_CUDA, "libnccl.so.2 not found (%s)", dlerror() ? dlerror() : "dlopen");
  Nccl::unique_id id;
  NCCL_TRY(g_nccl.GetUniqueId(&id));
  memcpy(out_id, &id, sizeof id);
  return B2P_OK;
}

int b2p_comm_init(b2p_ctx* c, const void* id_bytes, size_t bytes, int n_ranks, int rank) {
  if (!c || !id_bytes || bytes < sizeof(Nccl::unique_id) || n_ranks < 1 || rank < 0 || rank >= n_ranks)
    return fail(B2P_E_INVALID, "bad communicator arguments");
  if (c->comm) return fail(B2P_E_INVALID, "context already has a communicator");
  if (!g_nccl.load()) return fail(B2P_E_CUDA, "libnccl.so.2 not found (%s)", dlerror() ? dlerror() : "dlopen");
  DeviceGuard g(c->device);
  Nccl::unique_id id;
  memcpy(&id, id_bytes, sizeof id);
  // the tile all-reduces run next to the persistent range kernel: keep their footprint to a few SMs (an explicit
  // NCCL_MAX_CTAS / NCCL_MAX_NCHANNELS of the caller wins)
  setenv("NCCL_MAX_CTAS", "16", 0);
  setenv("NCCL_MAX_NCHANNELS", "16", 0);
  NCCL_TRY(g_nccl.CommInitRank(&c->comm, n_ranks, id, rank));
  c->comm_ranks = n_ranks;
  c->comm_rank = rank;
  int lo = 0, hi = 0;
  CU(cudaDeviceGetStreamPriorityRange(&lo, &hi));  // hi = numerically lowest = highest priority
  CU(cudaStreamCreateWithPriority(&c->s_comm, cudaStreamNonBlocking, hi));
  CU(cudaEventCreateWithFlags(&c->ev_comm_in, cudaEventDisableTiming));
  CU(cudaEventCreateWithFlags(&c->ev_comm_done, cudaEventDisableTiming));
  CU(cudaEventCreateWithFlags(&c->ev_comm_go, cudaEventDisableTiming));
  return B2P_OK;
}

int32_t b2p_comm_ranks(b2p_ctx* c, int32_t* rank) {
  if (rank) *rank = c ? c->comm_rank : 0;
  return c && c->comm ? c->comm_ranks : 0;
}

int b2p_comm_destroy(b2p_ctx* c) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (!c->comm) return B2P_OK;
  DeviceGuard g(c->device);
  cudaStreamSynchronize(c->stream);
  if (c->s_comm) cudaStreamSynchronize(c->s_comm);
  NCCL_TRY(g_nccl.CommDestroy(c->comm));
  c->comm = nullptr;
  c->comm_ranks = 1;
  c->comm_rank = 0;
  return B2P_OK;
}

}  // extern "C"

int allreduce_with_counts(b2p_ctx* c, void* val, int type, int op, uint32_t* cnt, uint64_t n, cudaStream_t s) {
  return nccl_group([&] {
    NCCL_TRY(g_nccl.AllReduce(val, val, n, type, op, c->comm, s));
    NCCL_TRY(g_nccl.AllReduce(cnt, cnt, n, Nccl::kUint32, Nccl::kSum, c->comm, s));
    return B2P_OK;
  });
}

int gather_blocks(b2p_ctx* c, void* buf, const uint64_t* sizes, size_t entry_bytes, int type) {
  if (!c->comm) return B2P_OK;
  return nccl_group([&] {
    char* at = static_cast<char*>(buf);
    for (int r = 0; r < c->comm_ranks; ++r) {
      const size_t bytes = sizes[r] * entry_bytes;
      if (bytes) NCCL_TRY(g_nccl.Broadcast(at, at, bytes / Nccl::bytes(type), type, r, c->comm, c->stream));
      at += bytes;
    }
    return B2P_OK;
  });
}
