// Error text, ABI version and the launch counter shared by every entry point.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>

#include "common.cuh"

namespace d3b {

static thread_local char g_error[512] = "";
static std::atomic<unsigned long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
}

static std::atomic<int> g_pdl{1};
bool pdl_enabled() { return g_pdl.load(std::memory_order_relaxed) != 0; }

// default schedule of the 3x3 stride-1 dense layers; the environment variable D3B_BEV_VARIANT overrides it at load
constexpr int kDefaultBevVariant = 2;      // automatic (pixel-stationary): see d3b_set_bev_variant
static int initial_bev_variant() {
  const char* e = std::getenv("D3B_BEV_VARIANT");
  if (e != nullptr && e[0] >= '0' && e[0] <= '2' && e[1] == 0) return e[0] - '0';
  return kDefaultBevVariant;
}
static std::atomic<int> g_bev_variant{initial_bev_variant()};
int bev_variant() { return g_bev_variant.load(std::memory_order_relaxed); }

void count_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

}  // namespace d3b

extern "C" const char* d3b_last_error(void) { return d3b::g_error; }
extern "C" int d3b_abi_version(void) { return 2; }
extern "C" void d3b_set_pdl(int on) { d3b::g_pdl.store(on ? 1 : 0, std::memory_order_relaxed); }
extern "C" void d3b_set_bev_variant(int v) { d3b::g_bev_variant.store(v >= 0 && v <= 2 ? v : 2, std::memory_order_relaxed); }
extern "C" int d3b_get_bev_variant(void) { return d3b::bev_variant(); }
extern "C" unsigned long long d3b_launch_count(void) {
  return d3b::g_launches.load(std::memory_order_relaxed);
}
