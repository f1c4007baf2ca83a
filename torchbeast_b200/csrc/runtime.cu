// Library runtime: error plumbing, launch counter, optional per-op event profiler, misc C ABI.
#include <stdarg.h>
#include <string.h>

#include <atomic>
#include <mutex>
#include <vector>

#include "common.cuh"

namespace tb {

static thread_local char g_err[512] = "";
static std::atomic<unsigned long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return 2;
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return 0;
}

// ---- profiler ---------------------------------------------------------------------------
struct ProfRecord { const char* name; cudaEvent_t a, b; };
static std::mutex g_prof_mu;
static std::vector<ProfRecord> g_prof;
static std::atomic<int> g_prof_on{0};

ProfScope::ProfScope(const char* name, cudaStream_t st) : slot(-1), stream(st) {
  if (!g_prof_on.load(std::memory_order_relaxed)) return;
  ProfRecord r;
  r.name = name;
  if (cudaEventCreate(&r.a) != cudaSuccess || cudaEventCreate(&r.b) != cudaSuccess) return;
  cudaEventRecord(r.a, st);
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof.push_back(r);
  slot = int(g_prof.size()) - 1;
}

ProfScope::~ProfScope() {
  if (slot < 0) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (slot < int(g_prof.size())) cudaEventRecord(g_prof[slot].b, stream);
}

}  // namespace tb

using namespace tb;

extern "C" {

int tb_abi_version(void) { return TB_ABI_VERSION; }
const char* tb_last_error(void) { return g_err; }
size_t tb_workspace_bytes(void) { return kWorkspaceBytes; }
uint64_t tb_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int tb_device_info(int* sm, int* major, int* minor) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  cudaDeviceProp prop;
  if (e == cudaSuccess) e = cudaGetDeviceProperties(&prop, dev);
  if (e != cudaSuccess) { set_error("tb_device_info: %s", cudaGetErrorString(e)); return 2; }
  if (sm) *sm = prop.multiProcessorCount;
  if (major) *major = prop.major;
  if (minor) *minor = prop.minor;
  return 0;
}

int tb_profile_enable(int on) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (on) {
    for (auto& r : g_prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    g_prof.clear();
  }
  g_prof_on.store(on ? 1 : 0);
  return 0;
}

int tb_profile_collect(char* names_host, size_t names_cap, float* ms_host, int max_records) {
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { set_error("tb_profile_collect: %s", cudaGetErrorString(e)); return -1; }
  std::lock_guard<std::mutex> lk(g_prof_mu);
  int n = 0;
  size_t off = 0;
  for (auto& r : g_prof) {
    if (n >= max_records) break;
    float ms = 0.0f;
    if (cudaEventElapsedTime(&ms, r.a, r.b) != cudaSuccess) { cudaGetLastError(); continue; }
    const size_t len = strlen(r.name);
    if (off + len + 2 > names_cap) break;
    memcpy(names_host + off, r.name, len);
    names_host[off + len] = '\n';
    off += len + 1;
    ms_host[n++] = ms;
  }
  if (names_cap) names_host[off < names_cap ? off : names_cap - 1] = '\0';
  return n;
}

// The layout of tb_hparams as compiled, for a binding's check of its packing (host only).
int tb_hparams_layout(int64_t* out) {
  TB_REQUIRE(out, "tb_hparams_layout: null pointer");
  const int64_t layout[] = {
      int64_t(sizeof(tb_hparams)),
      int64_t(offsetof(tb_hparams, discounting)), int64_t(offsetof(tb_hparams, baseline_cost)),
      int64_t(offsetof(tb_hparams, entropy_cost)), int64_t(offsetof(tb_hparams, clip_rho)),
      int64_t(offsetof(tb_hparams, clip_pg_rho)), int64_t(offsetof(tb_hparams, clip_rewards)),
      int64_t(offsetof(tb_hparams, max_norm)), int64_t(offsetof(tb_hparams, alpha)), int64_t(offsetof(tb_hparams, eps)),
      int64_t(offsetof(tb_hparams, momentum)), int64_t(offsetof(tb_hparams, weight_decay)),
      int64_t(offsetof(tb_hparams, beta1)), int64_t(offsetof(tb_hparams, beta2))};
  memcpy(out, layout, sizeof(layout));
  return 0;
}

// Host side of the learner-queue ingest (SURVEY 8(f) N1): one actor hands its [T1, ...] rollout over by writing it into
// batch column b of a pinned [T1, B, ...] slot - what actorpool.cc:493-506 + the BatchingQueue's torch::cat (actorpool.cc:
// 49-55) do with per-rollout tensors and a concatenation.  Plain memcpy per (leaf, time step): leaf l of the slot starts
// at slot_base + leaf_offset[l], a row (one time step of one column) is row_bytes[l] bytes, the source is the actor's
// contiguous [T1, row] array.  No CUDA calls: runs on the calling host thread (ctypes releases the GIL for its duration,
// which is the point - 48 Python actor threads otherwise serialise on it).
int tb_host_write_rollout_column(uint8_t* slot_base, const int64_t* leaf_offset, const int64_t* row_bytes, int num_leaves,
                                 int64_t T1, int64_t B, int64_t b, const uint8_t* const* src) {
  TB_REQUIRE(slot_base && leaf_offset && row_bytes && src, "tb_host_write_rollout_column: null pointer");
  TB_REQUIRE(num_leaves >= 1 && T1 >= 1 && B >= 1 && b >= 0 && b < B, "tb_host_write_rollout_column: bad sizes");
  for (int l = 0; l < num_leaves; ++l) {
    const int64_t rb = row_bytes[l];
    if (!src[l] || rb <= 0) continue;
    uint8_t* dst = slot_base + leaf_offset[l] + b * rb;
    const uint8_t* s = src[l];
    for (int64_t t = 0; t < T1; ++t) memcpy(dst + t * B * rb, s + t * rb, size_t(rb));
  }
  return 0;
}

}  // extern "C"
