// Library-wide entry points: version, error text, device info, scheduler-slot binding.
#include <stdarg.h>
#include <string.h>

#include <atomic>

#include "tc_common.cuh"

namespace edet {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// Library options (edet_set_option): one table, looked up by name.
struct Option {
  const char* name;
  int lo, hi;                  // accepted range (further restricted by `allowed` below)
  std::atomic<int> value;
};
static Option g_options[] = {
    {"dw_impl", 0, 2, {0}},          // 0 auto (tiled kernel where eligible), 1 register kernel only
    {"stem_impl", 0, 1, {0}},        // 0 tensor-core stem, 1 CUDA-core stem
    {"sepconv_impl", 0, 2, {0}},     // 0 TMA-staged input (1 buffer, 4 CTAs/SM), 1 loads from global, 2 TMA, 2 buffers, 3 CTAs/SM
    {"pw_teams", 0, 3, {0}},         // 0 auto, 2 / 3 consumer warpgroups in pointwise_tc
    {"pw_smem_kb", 0, 227, {0}},     // 0 auto, else shared-memory budget of a pointwise_tc CTA
    {"persist_slack", 0, 132, {0}},  // CTAs a persistent kernel leaves out of its grid
    {"max_ctas", 0, 4096, {0}},      // 0 no cap, else the grid of a persistent kernel (at most its work)
    {"pw_share_w", 0, 1, {0}},       // 0 auto, 1 = pointwise_tc streams W per 64-row tile
};
static Option* find_option(const char* name) {
  for (Option& o : g_options)
    if (strcmp(name, o.name) == 0) return &o;
  return nullptr;
}
static int option_value(int idx) { return g_options[idx].value.load(std::memory_order_relaxed); }
int option_dw_impl() { return option_value(0); }
int option_stem_impl() { return option_value(1); }
int option_sepconv_impl() { return option_value(2); }
int option_pw_teams() { return option_value(3); }
int option_pw_smem_kb() { return option_value(4); }
int option_persist_slack() { return option_value(5); }
int option_max_ctas() { return option_value(6); }
int option_pw_share_w() { return option_value(7); }

int current_device() {
  int dev = -1;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) {
    set_error("cudaGetDevice failed or device ordinal %d >= %d", dev, kMaxDevices);
    return -1;
  }
  return dev;
}

int device_sm_count() {
  static std::atomic<int> cached[kMaxDevices];
  const int dev = current_device();
  if (dev < 0) return 0;
  int v = cached[dev].load(std::memory_order_relaxed);
  if (v == 0) {
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) {
      set_error("cudaDeviceGetAttribute(MultiProcessorCount) failed");
      return 0;
    }
    cached[dev].store(v, std::memory_order_relaxed);
  }
  return v;
}

int persistent_grid(int total_work, int ctas_per_sm) {
  const int sms = device_sm_count();
  if (!sms) return 0;
  int grid = ctas_per_sm * sms - option_persist_slack();
  const int cap = option_max_ctas();
  if (cap && grid > cap) grid = cap;
  if (grid > total_work) grid = total_work;
  return grid < 1 ? 1 : grid;
}

namespace pwtc {
// zero-initialised in every context that loads the module; each slot resets itself
__device__ unsigned g_tile_sched[2 * kSchedSlots];

// The calling thread's binding (edet_sched_bind): the next slot to hand out and how many are
// left; and the slot of its most recent slot-using launch (edet_last_sched_slot).
static thread_local unsigned* t_bound_next = nullptr;
static thread_local int t_bound_left = 0;
static thread_local unsigned* t_last_slot = nullptr;

int next_sched_slot(unsigned** slot) {
  if (t_bound_next != nullptr) {
    if (t_bound_left == 0) {
      set_error("scheduler slots: every slot bound by edet_sched_bind is in use; nothing launched");
      return EDET_ERR_INVALID;
    }
    *slot = t_last_slot = t_bound_next;
    t_bound_next += 2;
    --t_bound_left;
    return EDET_OK;
  }
  static std::atomic<unsigned*> base[kMaxDevices];
  static std::atomic<unsigned> next[kMaxDevices];
  const int dev = current_device();
  if (dev < 0) return EDET_ERR_CUDA;
  unsigned* b = base[dev].load(std::memory_order_acquire);
  if (b == nullptr) {
    void* addr = nullptr;
    if (cudaGetSymbolAddress(&addr, g_tile_sched) != cudaSuccess || addr == nullptr) {
      set_error("cudaGetSymbolAddress(g_tile_sched) failed");
      return EDET_ERR_CUDA;
    }
    b = static_cast<unsigned*>(addr);
    base[dev].store(b, std::memory_order_release);
  }
  const unsigned i = next[dev].fetch_add(1u, std::memory_order_relaxed) % kSchedSlots;
  *slot = t_last_slot = b + 2 * i;
  return EDET_OK;
}
}  // namespace pwtc
}  // namespace edet

extern "C" int edet_version(void) { return 200; }
extern "C" int edet_set_option(const char* name, int value) {
  using namespace edet;
  EDET_CHECK_ARG(name != nullptr, "set_option: null name");
  Option* o = find_option(name);
  if (o == nullptr) {
    set_error("set_option: unknown option '%s'", name);
    return EDET_ERR_INVALID;
  }
  EDET_CHECK_ARG(value >= o->lo && value <= o->hi, "set_option: %s must be in %d..%d (got %d)", name,
                 o->lo, o->hi, value);
  EDET_CHECK_ARG(strcmp(name, "pw_teams") != 0 || value != 1, "set_option: pw_teams must be 0, 2 or 3");
  EDET_CHECK_ARG(strcmp(name, "pw_smem_kb") != 0 || value == 0 || value >= 64,
                 "set_option: pw_smem_kb must be 0 or 64..227");
  o->value.store(value, std::memory_order_relaxed);
  return EDET_OK;
}
extern "C" int edet_get_option(const char* name, int* value) {
  using namespace edet;
  EDET_CHECK_ARG(name != nullptr && value != nullptr, "get_option: null pointer");
  Option* o = find_option(name);
  if (o == nullptr) {
    set_error("get_option: unknown option '%s'", name);
    return EDET_ERR_INVALID;
  }
  *value = o->value.load(std::memory_order_relaxed);
  return EDET_OK;
}
extern "C" const char* edet_last_error(void) { return edet::g_err; }
extern "C" int edet_sched_bind(void* slots, int count) {
  using namespace edet;
  EDET_CHECK_ARG(slots == nullptr || count > 0, "sched_bind: count must be > 0 (got %d)", count);
  EDET_CHECK_ARG(reinterpret_cast<uintptr_t>(slots) % 8 == 0, "sched_bind: slots must be 8-byte aligned");
  pwtc::t_bound_next = static_cast<unsigned*>(slots);
  pwtc::t_bound_left = slots ? count : 0;
  return EDET_OK;
}
extern "C" int edet_last_sched_slot(void** slot) {
  using namespace edet;
  EDET_CHECK_ARG(slot != nullptr, "last_sched_slot: null pointer");
  *slot = pwtc::t_last_slot;
  return EDET_OK;
}
extern "C" int edet_device_info(int* sm_count, int* cc) {
  int dev = 0, sms = 0, major = 0, minor = 0;
  EDET_CHECK_CUDA(cudaGetDevice(&dev));
  EDET_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  EDET_CHECK_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  EDET_CHECK_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  if (sm_count) *sm_count = sms;
  if (cc) *cc = major * 10 + minor;
  return EDET_OK;
}
