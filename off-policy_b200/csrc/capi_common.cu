// Error reporting, launch accounting and device queries shared by every entry point.
#include <limits.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <unordered_map>

#include "mx_internal.h"

static thread_local char g_err[512] = "";
long long g_mx_launches = 0;
#if !MX_EMU
int g_mx_pdl = -1;    // programmatic dependent launch: -1 (default) = for latency-bound learner steps only (rows <= g_mx_pdl_rows; set per step by the
                      // learner), 1 = every launch, 0 = never (the dependents' prologues take SM resources from kernels that are
                      // throughput-bound, so PDL is meant for the small steps; the row threshold is not yet measured on the H100)
int g_mx_pdl_rows = 12288;
int g_mx_pdl_auto = 0;      // the learner's per-step decision in automatic mode
int g_mx_pdl_skip_next = 0;
#endif

// runtime options shared by the product and the emulated build (mx_set_option)
int g_mx_p2p_timeout_ms = 10000;      // how long a rank waits for a peer's gradient before it sets the sticky abort word (tests shorten it)
int g_mx_p2p_ll = 1;          // data-parallel exchange inside k_optim_fused: 1 = flag-in-data lines (no fence / counter / flag hop), 0 = slots + per-rank flags
int g_mx_mixer_split = 1;      // 1: split mixer (hypernet-forward / core / hypernet-backward kernels) whenever the forked branch is
                               //    in use; 2: always; 0: always the single fused k_mixer
int g_mx_overlap = 1;          // state-only kernels (weight-image prep, mixer hypernets) on a forked branch beside the agent-net
                               // kernels: 1 = when the step is latency-bound (rows <= g_mx_overlap_rows), 2 = always, 0 = never
int g_mx_mid_fused = 1;        // 1: k_qhead + k_mix_core + k_qhead_bwd as ONE kernel (k_mid) when the split mixer is in use and no debug
                               //    outputs are requested; 0: three launches
int g_mx_overlap_rows = 1 << 20; // forked branch up to this many rows, serial beyond (not yet measured on the H100)
int mx_set_option_common(const char* name, int value) {
  if (!strcmp(name, "mixer_split")) { g_mx_mixer_split = value; return 0; }
  if (!strcmp(name, "overlap")) { g_mx_overlap = value; return 0; }
  if (!strcmp(name, "overlap_rows")) { g_mx_overlap_rows = value; return 0; }
  if (!strcmp(name, "mid_fused")) { g_mx_mid_fused = value; return 0; }
  if (!strcmp(name, "optim_fused")) { g_mx_optim_fused = value; return 0; }
  if (!strcmp(name, "p2p_ll")) { g_mx_p2p_ll = value; return 0; }
  if (!strcmp(name, "p2p_timeout_ms")) { g_mx_p2p_timeout_ms = value; return 0; }
#if !MX_EMU
  if (!strcmp(name, "smem_carveout")) { g_mx_smem_carveout = value; return 0; }
#else
  if (!strcmp(name, "smem_carveout")) return 0;
#endif
  if (!strcmp(name, "gather_tma")) { g_mx_gather_tma = value; return 0; }      // 1: episode gather on the TMA unit (default), 0: vectorised loads
  return -1;
}

void mx_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" const char* mx_last_error(void) { return g_err; }
extern "C" int mx_abi_version(void) { return MX_ABI_VERSION; }

// ---- host fences: "has the stream consumed this pinned staging buffer yet?" -------------------------------------------------------------
// The drop-in buffers reuse a few pinned host blocks (insert staging, sampled-index ring); a block may be rewritten only after the copy
// that read it has completed.  A pool of timing-less CUDA events behind three tiny calls: a torch.cuda.Event().record() costs the
// host ~8 us per call (it resolves the current stream object first), these ~1 us.
// A released fence goes to a free list and is handed out again, so a process may create and drop buffers without running out.
#define MX_MAX_FENCES 256
#if !MX_EMU
static cudaEvent_t g_fence[MX_MAX_FENCES];
static unsigned char g_fence_set[MX_MAX_FENCES];
#endif
static int g_fence_n = 0;
static unsigned char g_fence_live[MX_MAX_FENCES];
static int g_fence_free[MX_MAX_FENCES];
static int g_fence_nfree = 0;
static bool fence_ok(int id) { return id >= 0 && id < g_fence_n && g_fence_live[id]; }
extern "C" int mx_host_fence_alloc(void) {
  if (g_fence_nfree > 0) {
    const int id = g_fence_free[--g_fence_nfree];
    g_fence_live[id] = 1;
    return id;
  }
  if (g_fence_n >= MX_MAX_FENCES) { mx_set_error("mx_host_fence_alloc: out of fences (%d held)", MX_MAX_FENCES); return -1; }
#if !MX_EMU
  if (cudaEventCreateWithFlags(&g_fence[g_fence_n], cudaEventDisableTiming) != cudaSuccess) { mx_set_error("mx_host_fence_alloc: cudaEventCreate failed"); return -1; }
  g_fence_set[g_fence_n] = 0;
#endif
  g_fence_live[g_fence_n] = 1;
  return g_fence_n++;
}
extern "C" int mx_host_fence_release(int id) {
  if (!fence_ok(id)) { mx_set_error("mx_host_fence_release: bad fence"); return 1; }
#if !MX_EMU
  if (g_fence_set[id]) cudaEventSynchronize(g_fence[id]);      // the copy it guards has finished before the id is handed out again
  g_fence_set[id] = 0;
#endif
  g_fence_live[id] = 0;
  g_fence_free[g_fence_nfree++] = id;
  return 0;
}
extern "C" int mx_host_fence_record(int id, void* stream) {
  if (!fence_ok(id)) { mx_set_error("mx_host_fence_record: bad fence"); return 1; }
#if !MX_EMU
  if (cudaEventRecord(g_fence[id], (cudaStream_t)stream) != cudaSuccess) { mx_set_error("mx_host_fence_record: cudaEventRecord failed"); return 1; }
  g_fence_set[id] = 1;
#else
  (void)stream;
#endif
  return 0;
}
extern "C" int mx_host_fence_wait(int id) {       // returns once everything enqueued before the last record of this fence has completed
  if (!fence_ok(id)) { mx_set_error("mx_host_fence_wait: bad fence"); return 1; }
#if !MX_EMU
  if (g_fence_set[id]) {
    const cudaError_t e = cudaEventSynchronize(g_fence[id]);      // also the first place an asynchronous fault of earlier work surfaces
    if (e != cudaSuccess) { mx_set_error("mx_host_fence_wait: cudaEventSynchronize failed: %s", cudaGetErrorString(e)); return 1; }
  }
#endif
  return 0;
}
extern "C" int64_t mx_sizeof(const char* n) {
  if (!n) return -1;
#define MX_SZ(T) if (!strcmp(n, #T)) return (int64_t)sizeof(T)
  MX_SZ(mx_batch); MX_SZ(mx_replay_cfg); MX_SZ(mx_replay_layout); MX_SZ(mx_qmix_cfg); MX_SZ(mx_maddpg_cfg); MX_SZ(mx_param_entry);
  MX_SZ(mx_policy_step_args); MX_SZ(mx_episodes); MX_SZ(mx_trng_draw);
#undef MX_SZ
  return -1;
}
extern "C" int mx_is_cuda_build(void) { return MX_EMU ? 0 : 1; }
extern "C" int64_t mx_launch_count(void) { return g_mx_launches; }

int g_mx_prof_on = 0;
#include <string>
#include <vector>
#if MX_EMU
// CPU-emulated unit-test build: the same marks, stamped with the host clock (kernels run synchronously there)
#include <chrono>
static std::vector<std::pair<std::string, double>> g_marks;
static double g_prof_start;
static double emu_now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
void mx_prof_mark(const char* name, cudaStream_t) { g_marks.emplace_back(name, emu_now_ms()); }
extern "C" int mx_profile_begin(void*) {
  g_marks.clear();
  g_prof_start = emu_now_ms();
  g_mx_prof_on = 1;
  return 0;
}
extern "C" int mx_profile_end(void*, char* names_buf, int32_t buf_len, float* ms, int32_t max_n) {
  g_mx_prof_on = 0;
  std::string names;
  double prev = g_prof_start;
  int n = 0;
  for (auto& m : g_marks) {
    if (n < max_n) {
      ms[n] = (float)(m.second - prev);
      if (n) names += ";";
      names += m.first;
      ++n;
    }
    prev = m.second;
  }
  if (names_buf && buf_len > 0) snprintf(names_buf, buf_len, "%s", names.c_str());
  g_marks.clear();
  return n;
}
#else
static std::vector<std::pair<std::string, cudaEvent_t>> g_marks;
static cudaEvent_t g_prof_start;
void mx_prof_mark(const char* name, cudaStream_t s) {
  cudaEvent_t e;
  cudaEventCreate(&e);
  cudaEventRecord(e, s);
  g_marks.emplace_back(name, e);
}
extern "C" int mx_profile_begin(void* stream) {
  for (auto& m : g_marks) cudaEventDestroy(m.second);
  g_marks.clear();
  cudaEventCreate(&g_prof_start);
  cudaEventRecord(g_prof_start, (cudaStream_t)stream);
  g_mx_prof_on = 1;
  return 0;
}
extern "C" int mx_profile_end(void* stream, char* names_buf, int32_t buf_len, float* ms, int32_t max_n) {
  g_mx_prof_on = 0;
  cudaStreamSynchronize((cudaStream_t)stream);
  std::string names;
  cudaEvent_t prev = g_prof_start;
  int n = 0;
  for (auto& m : g_marks) {
    if (n < max_n) {
      float t = 0.f;
      cudaEventElapsedTime(&t, prev, m.second);
      ms[n] = t;
      if (n) names += ";";
      names += m.first;
      ++n;
    }
    prev = m.second;
  }
  if (names_buf && buf_len > 0) snprintf(names_buf, buf_len, "%s", names.c_str());
  for (auto& m : g_marks) cudaEventDestroy(m.second);
  g_marks.clear();
  cudaEventDestroy(g_prof_start);
  return n;
}
#endif

#if !MX_EMU
int g_mx_smem_carveout = 100;

// What each kernel launched so far has been configured for: its dynamic shared-memory limit and the carveout option it was given.
struct MxKernelConfig {
  size_t smem = 0;
  int carveout = INT_MIN;
};
static std::unordered_map<const void*, MxKernelConfig> g_kernel_config;

int mx_launch_config(const char* name, const void* kern, size_t smem, MxLaunchKind kind, cudaLaunchConfig_t* cfg) {
  if (kind == MX_PLAIN && smem == 0) return 0;
  MxKernelConfig& k = g_kernel_config[kern];
  if (smem > k.smem) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
      cudaGetLastError();
      mx_set_error("%s: %zu bytes of shared memory are more than the kernel can be configured for", name, smem);
      return MX_ERR_SMEM;
    }
    k.smem = smem;
  }
  if (kind == MX_STEP) {
    if (k.carveout != g_mx_smem_carveout) {
      cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, g_mx_smem_carveout < 0 ? -1 : g_mx_smem_carveout);
      k.carveout = g_mx_smem_carveout;
    }
    if ((g_mx_pdl > 0 || (g_mx_pdl < 0 && g_mx_pdl_auto)) && !g_mx_pdl_skip_next) {
      cfg->attrs[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
      cfg->attrs[0].val.programmaticStreamSerializationAllowed = 1;
      cfg->numAttrs = 1;
    }
    g_mx_pdl_skip_next = 0;
  }
  return 0;
}
int mx_launch_done(const char* name, cudaStream_t s) {
  ++g_mx_launches;
  MX_MARK(name, s);
  return mx_check_launch(name);
}
int mx_num_sms() {
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 148;
  }
  return sms;
}
int mx_check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    mx_set_error("CUDA error after %s: %s", what, cudaGetErrorString(e));
    return 2;
  }
  return 0;
}
#endif
