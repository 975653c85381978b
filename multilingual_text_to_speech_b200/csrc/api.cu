// Library-wide state of libb200tts (include/b200tts.h): last error, launch counter, kernel timers, the device check, the precision,
// scratch and tensor-core switches, and the dropout-mask / uniform fills.  Every other entry point lives beside the kernels it runs.
#include <stdarg.h>
#include <atomic>
#include <mutex>
#include <vector>
#include <string>
#include "common.cuh"

namespace b200tts {

static thread_local char g_error[1024] = "";
static std::atomic<unsigned long long> g_launches{0};

void set_last_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
}

int check_cuda(cudaError_t e, const char* what, const char* file, int line) {
    if (e == cudaSuccess) {
        if (what[0] == 'c' && strncmp(what, "cudaGetLastError", 16) == 0) g_launches.fetch_add(1, std::memory_order_relaxed);
        return B200TTS_OK;
    }
    set_last_error("CUDA error %s (%s) at %s:%d in %s", cudaGetErrorName(e), cudaGetErrorString(e), file, line, what);
    return B200TTS_ERR_CUDA;
}

// ---- named kernel timers -------------------------------------------------------------------------
namespace {
struct KSpan { const char* name; cudaEvent_t e0, e1; bool closed; };
std::atomic<int> g_ktime_on{0};
std::mutex g_ktime_mu;
std::vector<KSpan> g_spans;
std::vector<cudaEvent_t> g_event_pool;
cudaEvent_t take_event() {
    if (!g_event_pool.empty()) { cudaEvent_t e = g_event_pool.back(); g_event_pool.pop_back(); return e; }
    cudaEvent_t e = nullptr;
    cudaEventCreate(&e);
    return e;
}
}  // namespace
void ktimer_start(const char* name, cudaStream_t st) {
    if (!g_ktime_on.load(std::memory_order_relaxed)) return;
    std::lock_guard<std::mutex> lk(g_ktime_mu);
    KSpan s{name, take_event(), take_event(), false};
    cudaEventRecord(s.e0, st);
    g_spans.push_back(s);
}
void ktimer_stop(const char* name, cudaStream_t st) {
    if (!g_ktime_on.load(std::memory_order_relaxed)) return;
    std::lock_guard<std::mutex> lk(g_ktime_mu);
    for (size_t i = g_spans.size(); i-- > 0;)
        if (!g_spans[i].closed && g_spans[i].name == name) { cudaEventRecord(g_spans[i].e1, st); g_spans[i].closed = true; return; }
}

int require_device() {
    static int cached = 0;   // 0 unknown, 1 ok, -1 bad
    if (cached == 1) return B200TTS_OK;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    cudaDeviceProp prop;
    if (e == cudaSuccess) e = cudaGetDeviceProperties(&prop, dev);
    if (e != cudaSuccess) {
        set_last_error("no usable CUDA device (%s); b200tts has no CPU fallback", cudaGetErrorString(e));
        cudaGetLastError();
        return B200TTS_ERR_CUDA;
    }
    if (prop.major != 9 || prop.minor != 0) {
        set_last_error("device %s is sm_%d%d; b200tts is built for sm_90a only", prop.name, prop.major, prop.minor);
        return B200TTS_ERR_UNSUPPORTED;
    }
    cached = 1;
    return B200TTS_OK;
}

namespace {
// counter-based generator: splitmix64 finaliser over (seed, stream, index/4); 16 bits per decision
__host__ __device__ __forceinline__ unsigned long long mix64(unsigned long long z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
// the key of stream (seed, stream_id), and the 64-bit draw of group g of it (4 keep decisions or one uniform)
__host__ __device__ __forceinline__ unsigned long long stream_key(unsigned long long seed, unsigned long long stream_id) {
    return mix64(seed ^ 0xD6E8FEB86659FD93ull) ^ (stream_id * 0xA24BAED4963EE407ull);
}
__device__ __forceinline__ unsigned long long stream_draw(unsigned long long key, unsigned long long g) {
    return mix64(key + g * 0x9E3779B97F4A7C15ull);
}
__global__ void fill_keep_mask_kernel(uint8_t* __restrict__ mask, size_t n, unsigned threshold, unsigned long long key,
                                      const unsigned long long* __restrict__ epoch) {
    if (epoch) key ^= mix64(*epoch * 0xC2B2AE3D27D4EB4Full + 0x165667B19E3779F9ull);
    // group g of 4 decisions comes from one 64-bit draw (16 bits each); a thread iteration produces 4 groups = one 16-byte store.
    // (same stream of decisions as a one-group-per-thread kernel: decision i depends on (key, i / 4, i % 4) only)
    const size_t groups = (n + 3) / 4, quads = (groups + 3) / 4;
    const bool aligned = (reinterpret_cast<uintptr_t>(mask) & 15) == 0;
    for (size_t q = blockIdx.x * (size_t)blockDim.x + threadIdx.x; q < quads; q += (size_t)gridDim.x * blockDim.x) {
        uint32_t w[4];
#pragma unroll
        for (int gg = 0; gg < 4; ++gg) {
            const unsigned long long r = stream_draw(key, q * 4 + gg);
            uint32_t v = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) v |= ((((unsigned)(r >> (16 * j)) & 0xFFFFu) >= threshold) ? 1u : 0u) << (8 * j);
            w[gg] = v;
        }
        const size_t i0 = q * 16;
        if (aligned && i0 + 16 <= n) {
            *reinterpret_cast<uint4*>(mask + i0) = make_uint4(w[0], w[1], w[2], w[3]);
        } else {
            for (int e = 0; e < 16; ++e)
                if (i0 + e < n) mask[i0 + e] = (uint8_t)((w[e >> 2] >> (8 * (e & 3))) & 0xFFu);
        }
    }
}
// element (i, r, p) of [steps, rows, width]: decision d = (step0[r] + i) * width + p of row r's stream, i.e. 16-bit field d % 4 of
// draw d / 4, as fill_keep_mask_kernel makes it
__global__ void fill_keep_mask_rows_kernel(uint8_t* __restrict__ mask, int steps, int rows, int width, unsigned threshold,
                                           const unsigned long long* __restrict__ seeds, const long long* __restrict__ step0,
                                           unsigned long long stream_id) {
    const long long n = (long long)steps * rows * width;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        const int p = (int)(idx % width);
        const long long ir = idx / width;
        const int r = (int)(ir % rows);
        const long long i = ir / rows;
        const unsigned long long d = (unsigned long long)(step0[r] + i) * width + p;
        const unsigned long long v = stream_draw(stream_key(seeds[r], stream_id), d >> 2);
        mask[idx] = (((unsigned)(v >> (16 * (d & 3))) & 0xFFFFu) >= threshold) ? 1 : 0;
    }
}

// element (r, i, u) of [rows, nsteps, width]: the top 24 bits of draw (t0[r] + i) * width + u of row r's stream, times 2^-24
__global__ void fill_uniform_rows_kernel(float* __restrict__ out, int rows, int nsteps, int width, const unsigned long long* __restrict__ seeds,
                                         const long long* __restrict__ t0, unsigned long long stream_id) {
    const long long n = (long long)rows * nsteps * width;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < n; idx += (long long)gridDim.x * blockDim.x) {
        const long long per_row = (long long)nsteps * width;
        const int r = (int)(idx / per_row);
        const unsigned long long d = (unsigned long long)(t0[r] * width + idx % per_row);
        out[idx] = (float)(stream_draw(stream_key(seeds[r], stream_id), d) >> 40) * 0x1p-24f;
    }
}
}  // namespace

}  // namespace b200tts
using namespace b200tts;

extern "C" {

const char* b200tts_last_error(void) { return g_error; }
int b200tts_version(void) { return 100; }
unsigned long long b200tts_launch_count(void) { return g_launches.load(); }
int b200tts_set_precision(int mode) {
    if (mode != B200TTS_PRECISION_FP32 && mode != B200TTS_PRECISION_BF16) { set_last_error("set_precision: unknown mode %d", mode); return B200TTS_ERR_INVALID; }
    set_precision_mode(mode);
    return B200TTS_OK;
}
int b200tts_get_precision(void) { return precision_mode(); }
int b200tts_kernel_timing(int enable) {
    std::lock_guard<std::mutex> lk(g_ktime_mu);
    for (auto& s : g_spans) { g_event_pool.push_back(s.e0); g_event_pool.push_back(s.e1); }
    g_spans.clear();
    g_ktime_on.store(enable ? 1 : 0);
    return B200TTS_OK;
}
int b200tts_kernel_timing_read(int index, char* name, int name_capacity, float* total_ms, int* count) {
    // distinct names in first-seen order; the caller synchronises the device first (elapsed times of unfinished spans fail)
    std::lock_guard<std::mutex> lk(g_ktime_mu);
    std::vector<const char*> names;
    for (auto& s : g_spans) {
        bool seen = false;
        for (auto n : names) seen = seen || strcmp(n, s.name) == 0;
        if (!seen) names.push_back(s.name);
    }
    if (index < 0 || index >= (int)names.size()) return 1;      // end of list
    float tot = 0.f; int cnt = 0;
    for (auto& s : g_spans)
        if (s.closed && strcmp(s.name, names[index]) == 0) {
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, s.e0, s.e1) != cudaSuccess) { cudaGetLastError(); set_last_error("kernel_timing_read: span of %s not finished (synchronize first)", s.name); return B200TTS_ERR_CUDA; }
            tot += ms; ++cnt;
        }
    if (name && name_capacity > 0) { strncpy(name, names[index], name_capacity - 1); name[name_capacity - 1] = 0; }
    if (total_ms) *total_ms = tot;
    if (count) *count = cnt;
    return B200TTS_OK;
}
int b200tts_set_scratch(void* ptr, size_t bytes) {
    if (ptr && (reinterpret_cast<uintptr_t>(ptr) & 1023)) { set_last_error("set_scratch: pointer must be 1024-byte aligned"); return B200TTS_ERR_INVALID; }
    set_tc_scratch(ptr, ptr ? bytes : 0);
    return B200TTS_OK;
}
int b200tts_set_tensor_core_gemm(int enabled) { set_tc_enabled(enabled ? 1 : 0); return B200TTS_OK; }

static const unsigned long long* g_mask_epoch = nullptr;
int b200tts_set_mask_epoch(const uint64_t* device_epoch) {
    g_mask_epoch = reinterpret_cast<const unsigned long long*>(device_epoch);
    return B200TTS_OK;
}
int b200tts_fill_keep_mask(uint8_t* mask, size_t n, float drop_rate, uint64_t seed, uint64_t stream_id, void* stream) {
    B200_TRY(require_device());
    B200_REQUIRE(mask || n == 0, "fill_keep_mask: null mask");
    B200_REQUIRE(drop_rate >= 0.f && drop_rate < 1.f, "fill_keep_mask: rate must be in [0,1)");
    if (n == 0) return B200TTS_OK;
    const unsigned threshold = (unsigned)(drop_rate * 65536.0f + 0.5f);
    const unsigned long long key = stream_key(seed, stream_id);
    size_t quads = (n + 15) / 16;
    int blocks = (int)((quads + 255) / 256 > NUM_SMS * 16 ? NUM_SMS * 16 : (quads + 255) / 256);
    if (blocks < 1) blocks = 1;
    fill_keep_mask_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(mask, n, threshold, key, g_mask_epoch);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_fill_keep_mask_rows(uint8_t* mask, int steps, int rows, int width, float drop_rate, const uint64_t* seeds, const int64_t* step0,
                                uint64_t stream_id, void* stream) {
    B200_REQUIRE(steps >= 0 && rows >= 1 && width >= 1, "fill_keep_mask_rows: %d steps, %d rows, width %d", steps, rows, width);
    B200_REQUIRE((mask || steps == 0) && seeds && step0, "fill_keep_mask_rows: null mask, seeds or step0");
    B200_REQUIRE(drop_rate >= 0.f && drop_rate < 1.f, "fill_keep_mask_rows: rate must be in [0,1)");
    B200_TRY(require_device());
    if (steps == 0) return B200TTS_OK;
    const unsigned threshold = (unsigned)(drop_rate * 65536.0f + 0.5f);
    fill_keep_mask_rows_kernel<<<grid_for((size_t)steps * rows * width), 256, 0, (cudaStream_t)stream>>>(
        mask, steps, rows, width, threshold, reinterpret_cast<const unsigned long long*>(seeds), reinterpret_cast<const long long*>(step0),
        stream_id);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_fill_uniform_rows(float* out, int rows, int nsteps, int width, const uint64_t* seeds, const int64_t* t0, uint64_t stream_id,
                              void* stream) {
    B200_REQUIRE(rows >= 1 && nsteps >= 0 && width >= 1, "fill_uniform_rows: %d rows, %d steps, width %d", rows, nsteps, width);
    B200_REQUIRE((out || nsteps == 0) && seeds && t0, "fill_uniform_rows: null output, seeds or t0");
    B200_TRY(require_device());
    if (nsteps == 0) return B200TTS_OK;
    fill_uniform_rows_kernel<<<grid_for((size_t)rows * nsteps * width), 256, 0, (cudaStream_t)stream>>>(
        out, rows, nsteps, width, reinterpret_cast<const unsigned long long*>(seeds), reinterpret_cast<const long long*>(t0), stream_id);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // extern "C"
