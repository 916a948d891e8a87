// C ABI glue: error strings, launch counter, tap-GEMM dispatch.
#include "tapgemm.cuh"
#include <atomic>
#include <cstdarg>
#include <memory>
#include <vector>

namespace b200vc {

static thread_local char g_err[1024] = "";
static std::atomic<long long> g_launches{0};

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

}  // namespace b200vc

// A recorded launch sequence: what a per-shape "model handle" is below Python (include/b200vc.h, b200vc_plan_*).
struct b200vc_plan {
  std::vector<std::function<int(void*)>> steps;
};

namespace b200vc {
static thread_local b200vc_plan* g_recording = nullptr;
bool plan_recording() { return g_recording != nullptr; }
void plan_push(std::function<int(void*)> step) { g_recording->steps.push_back(std::move(step)); }
}  // namespace b200vc

using namespace b200vc;

extern "C" {

const char* b200vc_version(void) { return "b200vc 0.1 (sm_90a)"; }
const char* b200vc_last_error(void) { return g_err; }
int64_t b200vc_launch_count(void) { return (int64_t)g_launches.load(); }
void b200vc_count_launches(int64_t n) { g_launches.fetch_add((long long)n, std::memory_order_relaxed); }
int64_t b200vc_sizeof_tapgemm_params(void) { return (int64_t)sizeof(b200vc_tapgemm_params); }

int b200vc_plan_begin(b200vc_plan** out) {
  B200VC_REQUIRE(out != nullptr, "plan_begin: null handle pointer");
  B200VC_REQUIRE(g_recording == nullptr, "plan_begin: this thread is already recording a plan");
  *out = new b200vc_plan();
  g_recording = *out;
  return kOk;
}

int b200vc_plan_end(void) {
  B200VC_REQUIRE(g_recording != nullptr, "plan_end: no plan is being recorded on this thread");
  g_recording = nullptr;
  return kOk;
}

int b200vc_plan_size(const b200vc_plan* plan) { return plan ? (int)plan->steps.size() : -1; }

int b200vc_plan_run(const b200vc_plan* plan, void* stream) {
  B200VC_REQUIRE(plan != nullptr, "plan_run: null plan");
  B200VC_REQUIRE(g_recording == nullptr, "plan_run: called while recording");
  for (const auto& st : plan->steps) {
    const int rc = st(stream);
    if (rc) return rc;
  }
  return kOk;
}

int b200vc_plan_destroy(b200vc_plan* plan) {
  if (g_recording == plan) g_recording = nullptr;
  delete plan;
  return kOk;
}

int b200vc_tapgemm(const b200vc_tapgemm_params* p, int backend, void* stream) {
  B200VC_REQUIRE(p != nullptr, "tapgemm: null descriptor");
  if (plan_recording()) {       // the descriptor is copied: the caller's struct need not outlive the call
    auto copy = std::make_shared<b200vc_tapgemm_params>(*p);
    plan_push([copy, backend](void* s) -> int { return b200vc_tapgemm(copy.get(), backend, s); });
    return kOk;
  }
  B200VC_REQUIRE(p->A && p->Wt && p->out, "tapgemm: null operand pointer");
  B200VC_REQUIRE(p->ntaps >= 1 && p->ntaps <= B200VC_MAX_TAPS, "tapgemm: ntaps %d out of range", p->ntaps);
  B200VC_REQUIRE(p->BW >= 1 && p->BH >= 1 && p->BW * p->BH == TG_TILE_M, "tapgemm: BW*BH must be 128 (got %d x %d)", p->BW, p->BH);
  B200VC_REQUIRE(p->N >= 1 && p->Kc >= 1, "tapgemm: bad N/Kc %d/%d", p->N, p->Kc);
  B200VC_REQUIRE(p->OW >= 1 && p->OH >= 1 && p->OB >= 1, "tapgemm: empty output space");
  B200VC_REQUIRE(p->a_stride[0] == 1, "tapgemm: A must be channels-last (a_stride[0]==1)");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (backend == B200VC_BACKEND_TC_TF32)          // auto: weight-stationary kernel where it applies, else persistent
    return tapgemm_ws_applicable(*p) ? tapgemm_ws_launch(*p, s) : tapgemm_tc2_launch(*p, s);
  if (backend == B200VC_BACKEND_TC_TF32_PERSISTENT) return tapgemm_tc2_launch(*p, s);
  if (backend == B200VC_BACKEND_TC_TF32_TILE) return tapgemm_tc_launch(*p, s);
  if (backend == B200VC_BACKEND_TC_TF32_WS) return tapgemm_ws_launch(*p, s);
  if (backend == B200VC_BACKEND_SIMT_FP32) return tapgemm_simt_launch(*p, s);
  set_last_error("tapgemm: unknown backend %d", backend);
  return kErrInvalidArg;
}

int b200vc_tapgemm_set_rows256(int on) {
  tapgemm_tc2_set_rows256(on);
  return kOk;
}

int b200vc_tapgemm_tc_supported(const b200vc_tapgemm_params* p) {
  return (p && tapgemm_tc_supported(*p)) ? 1 : 0;
}

int b200vc_tapgemm_ws_applicable(const b200vc_tapgemm_params* p) {
  return (p && tapgemm_ws_applicable(*p)) ? 1 : 0;
}

}  // extern "C"
