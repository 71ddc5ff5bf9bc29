// Library-level plumbing of the ts_b200 C ABI: version, thread-local error text, launch counter.
#include <atomic>
#include <cstdarg>
#include <cstdio>

#include "common.cuh"

namespace tsb {
namespace {
thread_local char g_err[512] = "";
std::atomic<int64_t> g_launches{0};
}  // namespace

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int device_ordinal() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) dev = 0;
    return dev;
}
int num_sms() {      // of the CURRENT device (the one the caller's stream and tensors live on)
    static int sms[kMaxDevices] = {};
    const int dev = device_ordinal();
    if (sms[dev] == 0) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;  // H100 SXM
        sms[dev] = n;
    }
    return sms[dev];
}
}  // namespace tsb

extern "C" int ts_version(void) { return TS_B200_ABI_VERSION; }
extern "C" const char* ts_last_error(void) { return tsb::g_err; }
extern "C" int64_t ts_launch_count(void) { return tsb::g_launches.load(std::memory_order_relaxed); }
extern "C" void ts_reset_launch_count(void) { tsb::g_launches.store(0, std::memory_order_relaxed); }

// ---- host side: the reference's minibatch order, bit for bit ------------------------------------------
// Batch.split draws ONE np.random.permutation(len) per pass from numpy's GLOBAL legacy RandomState
// (batch.py:1209).  That draw defines the minibatch composition, so it stays on the host and on numpy's
// algorithm -- MT19937, masked rejection sampling (random_interval) and the backward Fisher-Yates loop of
// RandomState.shuffle -- but as a tight int32 loop writing straight into the pinned upload buffer instead of
// numpy's generic-itemsize memcpy swaps + astype + copy.  The caller passes numpy's state in and writes the
// advanced state back (np.random.get_state / set_state), so every other consumer of the global stream sees
// exactly what it would have seen after np.random.permutation(n).
namespace {
constexpr int kMtN = 624, kMtM = 397;
inline void mt19937_gen(uint32_t* key) {
    constexpr uint32_t A = 0x9908b0dfu, UP = 0x80000000u, LO = 0x7fffffffu;
    int i = 0;
    uint32_t y;
    for (; i < kMtN - kMtM; ++i) {
        y = (key[i] & UP) | (key[i + 1] & LO);
        key[i] = key[i + kMtM] ^ (y >> 1) ^ ((0u - (y & 1u)) & A);
    }
    for (; i < kMtN - 1; ++i) {
        y = (key[i] & UP) | (key[i + 1] & LO);
        key[i] = key[i + (kMtM - kMtN)] ^ (y >> 1) ^ ((0u - (y & 1u)) & A);
    }
    y = (key[kMtN - 1] & UP) | (key[0] & LO);
    key[kMtN - 1] = key[kMtM - 1] ^ (y >> 1) ^ ((0u - (y & 1u)) & A);
}
}  // namespace

extern "C" int ts_host_mt19937_permutation(uint32_t* key, int32_t* pos, int64_t n, int32_t* out) {
    TS_REQUIRE(key && pos && out && n >= 0 && n <= 0x7fffffffLL && *pos >= 0 && *pos <= kMtN,
               "ts_host_mt19937_permutation: bad arguments");
    int p = *pos;
    for (int64_t i = 0; i < n; ++i) out[i] = (int32_t)i;
    // one iteration per DRAW: a rejected draw (v > i) swaps out[i] with itself and does not advance -- no
    // data-dependent branch (random_interval's do/while mispredicts ~30 % of the time)
    int64_t i = n - 1;
    while (i >= 1) {
        if (p == kMtN) { mt19937_gen(key); p = 0; }
        const int avail = kMtN - p;
        int d = 0;
        for (; d < avail && i >= 1; ++d) {
            uint32_t y = key[p + d];
            y ^= (y >> 11); y ^= (y << 7) & 0x9d2c5680u; y ^= (y << 15) & 0xefc60000u; y ^= (y >> 18);
            const uint32_t ui = (uint32_t)i;
            const uint32_t v = y & (0xffffffffu >> __builtin_clz(ui));
            const bool ok = v <= ui;
            const uint32_t vv = ok ? v : ui;
            const int32_t t = out[vv]; out[vv] = out[i]; out[i] = t;
            i -= (int64_t)ok;
        }
        p += d;
    }
    *pos = p;
    return 0;
}
