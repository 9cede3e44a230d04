// Error plumbing + version entry points of the C-ABI (include/b200rl.h).
#include "common.cuh"
#include <cstring>
#include <vector>

namespace b200rl {
static thread_local char g_err[512] = {0};
char* err_buf() { return g_err; }
int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

static long long g_launches = 0;
void note_launches(int n) { g_launches += n; }
long long launches() { return g_launches; }

// ------------------------------------------------------------------ profiling
struct ProfRec { const char* name; double flops, bytes; cudaEvent_t a, b; };
static bool g_prof_on = false;
static std::vector<ProfRec> g_recs;
static std::vector<cudaEvent_t> g_pool;
static size_t g_pool_next = 0;
static cudaEvent_t prof_event() {
    if (g_pool_next == g_pool.size()) {
        cudaEvent_t e;
        cudaEventCreate(&e);
        g_pool.push_back(e);
    }
    return g_pool[g_pool_next++];
}
bool prof_enabled() { return g_prof_on; }
void prof_begin(cudaStream_t s, const char* name, double flops, double bytes) {
    ProfRec r{name, flops, bytes, prof_event(), prof_event()};
    cudaEventRecord(r.a, s);
    g_recs.push_back(r);
}
void prof_end(cudaStream_t s) { cudaEventRecord(g_recs.back().b, s); }
}  // namespace b200rl

extern "C" long long b200rl_launch_count(void) { return b200rl::launches(); }
extern "C" void b200rl_profile_enable(int on) { b200rl::g_prof_on = on != 0; }
extern "C" void b200rl_profile_reset(void) { b200rl::g_recs.clear(); b200rl::g_pool_next = 0; }
// Synchronises the device, aggregates per kernel name and writes a JSON array into buf.
extern "C" int b200rl_profile_summary(char* buf, size_t cap) {
    using namespace b200rl;
    if (!buf || cap < 4) return fail(B200RL_ERR_INVALID_ARGUMENT, "profile_summary: buffer too small");
    cudaDeviceSynchronize();
    struct Agg { const char* name; int n; double ms, flops, bytes; };
    std::vector<Agg> aggs;
    for (auto& r : g_recs) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, r.a, r.b) != cudaSuccess) { cudaGetLastError(); continue; }
        Agg* a = nullptr;
        for (auto& x : aggs) if (strcmp(x.name, r.name) == 0) { a = &x; break; }
        if (!a) { aggs.push_back(Agg{r.name, 0, 0, 0, 0}); a = &aggs.back(); }
        a->n += 1; a->ms += ms; a->flops += r.flops; a->bytes += r.bytes;
    }
    size_t o = 0;
    o += snprintf(buf + o, cap - o, "[");
    for (size_t i = 0; i < aggs.size() && o + 256 < cap; ++i)
        o += snprintf(buf + o, cap - o, "%s{\"name\":\"%s\",\"launches\":%d,\"ms\":%.6f,\"flops\":%.6e,\"bytes\":%.6e}",
                      i ? "," : "", aggs[i].name, aggs[i].n, aggs[i].ms, aggs[i].flops, aggs[i].bytes);
    snprintf(buf + o, cap - o, "]");
    return B200RL_OK;
}

extern "C" int b200rl_version(void) { return 100; }  // 0.1.0
extern "C" const char* b200rl_last_error(void) { return b200rl::err_buf(); }
extern "C" int b200rl_compiled_arch(void) {
    return B200RL_ARCH;
}
