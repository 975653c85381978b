// extern "C" surface of libb200tts (see include/b200tts.h) + error / launch bookkeeping.
#include <stdarg.h>
#include <atomic>
#include <mutex>
#include <vector>
#include <string>
#include "decoder_internal.cuh"

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

static int require_device() {
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

int decoder_forward_impl(const b200tts_decoder_shape& s, const b200tts_decoder_params& w, const b200tts_decoder_inputs& in,
                         const b200tts_decoder_outputs& out, float* ws, size_t ws_bytes, cudaStream_t st,
                         const b200tts_decoder_state* state = nullptr, int first = 1);
int decoder_backward_impl(const b200tts_decoder_shape& s, const b200tts_decoder_params& w, const b200tts_decoder_inputs& in,
                          const b200tts_decoder_outputs& fwd_out, const b200tts_decoder_output_grads& dout, const float* fws,
                          float* bws, size_t bws_bytes, const b200tts_decoder_params& dw, float* d_memory, cudaStream_t st);
size_t decoder_bwd_workspace_floats(const b200tts_decoder_shape& s);
size_t attention_step_backward_workspace_elems(int B, int M, int A, int C, int K);
int attention_step_backward_impl(int B, int L, int M, int A, int C, int K, const float* q, const float* memory, const float* memT,
                                 const int* lengths, const float* Wloc, const float* Wc, const float* bias, const float* v,
                                 const float* cum_prev, const float* weights, const float* d_ctx, const float* d_weights, float* d_cum,
                                 float* d_q, float* d_memT, float* d_Wloc, float* d_Wc, float* d_v, float* ws, cudaStream_t st);
int attention_step_impl(int B, int L, int M, int D, int A, int C, int K, const float* query, const float* memory,
                        const float* memT, const int* lengths, const float* Wq, const float* Wloc, const float* Wc,
                        const float* bias, const float* v, float* cum, float* ctx, float* weights, float* workspace,
                        cudaStream_t st);
int forward_attention_step_impl(int B, int L, int M, int D, int A, const float* query, const float* memory, const float* memT,
                                const int* lengths, const float* Wq, const float* bias, const float* v, float* alpha, float* ctx,
                                float* weights, float* workspace, cudaStream_t st);
size_t forward_attention_step_backward_workspace_elems(int B, int M, int A);
int forward_attention_step_backward_impl(int B, int L, int M, int A, const float* q, const float* memory, const float* memT,
                                         const int* lengths, const float* bias, const float* v, const float* alpha_prev,
                                         const float* weights, const float* d_ctx, const float* d_weights, float* d_alpha, float* d_q,
                                         float* d_memT, float* d_v, float* ws, cudaStream_t st);


size_t convblock_saved_floats(const b200tts_convblock_shape& s);
size_t convblock_workspace_floats(const b200tts_convblock_shape& s);
int convblock_forward_impl(const b200tts_convblock_shape& s, const float* x, const float* weight, const float* gamma,
                           const float* beta, int affine_gstride, float* running_mean, float* running_var, const uint8_t* keep,
                           float* out, float* saved, float* ws, cudaStream_t st, const int32_t* lengths = nullptr);
int convblock_backward_impl(const b200tts_convblock_shape& s, const float* x, const float* weight, const float* gamma,
                            const float* beta, int affine_gstride, const uint8_t* keep, const float* saved, const float* dout,
                            float* dx, float* dweight, float* dgamma, float* dbeta, float* ws, cudaStream_t st);
size_t generator_workspace_floats(int G, int bn);
int generator_forward_impl(int G, int gd, int bn, long long R, const float* e, const float* Wb, const float* bb, const float* Wk,
                           const float* bk, float* eb, float* out, cudaStream_t st);
int generator_backward_impl(int G, int gd, int bn, long long R, const float* e, const float* Wb, const float* Wk, const float* eb,
                            const float* dout, float* de, float* dWb, float* dbb, float* dWk, float* dbk, float* ws, cudaStream_t st);
int embedding_forward_impl(float* out, int ldo, const float* table, const int* ids, long long ntok, int E, cudaStream_t st);
int embedding_backward_impl(float* dtable, int V, const float* dout, int ldo, const int* ids, long long ntok, int E, int padding_idx,
                            cudaStream_t st);
size_t bilstm_saved_floats(const b200tts_bilstm_shape& s);
size_t bilstm_workspace_floats(const b200tts_bilstm_shape& s);
int bilstm_forward_impl(const b200tts_bilstm_shape& s, const b200tts_bilstm_params& w, const float* x, const int* lengths, float* out,
                        float* saved, float* ws, cudaStream_t st);
int bilstm_backward_impl(const b200tts_bilstm_shape& s, const b200tts_bilstm_params& w, const int* lengths, const float* saved,
                         const float* dout, float* dx, const b200tts_bilstm_params& dw, float* ws, cudaStream_t st);

namespace {
// counter-based generator: splitmix64 finaliser over (seed, stream, index/4); 16 bits per decision
__host__ __device__ __forceinline__ unsigned long long mix64(unsigned long long z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
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
            const unsigned long long r = mix64(key + (q * 4 + gg) * 0x9E3779B97F4A7C15ull);
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
}  // namespace

}  // namespace b200tts

namespace b200tts {
size_t loss_workspace_floats();
int loss_forward_impl(const b200tts_loss_shape& s, const float* pre, const float* pre_t, const float* post, const float* post_t,
                      const float* stop, const float* stop_t, const float* align, const int* text_len, const int* target_len, float* losses,
                      float* ws, cudaStream_t st);
int loss_backward_impl(const b200tts_loss_shape& s, const float* pre, const float* pre_t, const float* post, const float* post_t,
                       const float* stop, const float* stop_t, const int* text_len, const int* target_len, const float* grad_losses,
                       float* d_pre, float* d_post, float* d_stop, float* d_align, cudaStream_t st);
size_t decoder_bwd_profile_offset(const b200tts_decoder_shape& s, int which);
void decoder_bwd_view_offsets(const b200tts_decoder_shape& s, size_t* out);
void set_tc_scratch(void* ptr, size_t bytes);
size_t adam_clip_scratch_floats();
int adam_clip_step_impl(float* p, float* g, float* m, float* v, size_t n, float lr, float beta1, float beta2, float eps, float weight_decay,
                        float max_norm, int step, float* scratch, cudaStream_t st);
void set_tc_enabled(int on);
int tc_enabled();
}
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
// Every query below answers for the step shape (T -> ceil(T / R) steps) that the forward and backward calls run on.
size_t b200tts_debug_persist_bwd_profile_offset(const b200tts_decoder_shape* shape, int which) {
    if (!shape || validate_decoder_shape(*shape) != B200TTS_OK) return 0;
    return decoder_bwd_profile_offset(step_shape(*shape), which);
}
size_t b200tts_debug_persist_profile_offset(const b200tts_decoder_shape* shape) {
    if (!shape || validate_decoder_shape(*shape) != B200TTS_OK) return 0;
    const b200tts_decoder_shape s = step_shape(*shape);
    return decoder_layout(s).persist * sizeof(float) + persist_layout(s).barrier + 256;
}
int b200tts_debug_decoder_views(const b200tts_decoder_shape* shape, size_t* out, int n) {
    if (!shape || !out || validate_decoder_shape(*shape) != B200TTS_OK) return 0;
    const b200tts_decoder_shape s = step_shape(*shape);
    const DecoderLayout l = decoder_layout(s);
    const PersistLayout pl = persist_layout(s);
    const TcPersistGeom g = tc_persist_geom(s);
    const size_t pbase = l.persist * sizeof(float);
    size_t v[26];
    const size_t fwd[11] = {l.ai, l.ca, l.hg, l.cg, l.ga, l.gg, l.q, l.cum, l.memT, l.fs, l.p1};
    for (int k = 0; k < 11; ++k) v[k] = fwd[k] * sizeof(float);
    v[11] = pbase + pl.aib;
    v[12] = pbase + pl.hgb;
    decoder_bwd_view_offsets(s, v + 13);
    v[24] = (size_t)g.Kp_att;
    v[25] = (size_t)g.Kp_gen;
    const int m = n < 26 ? n : 26;
    for (int k = 0; k < m; ++k) out[k] = v[k];
    return m;
}

int b200tts_gemm_f32(int transA, int transB, int M, int N, int K, float alpha, const float* A, int lda, const float* B,
                     int ldb, float beta, float* C, int ldc, const float* bias, int batch, long long strideA,
                     long long strideB, long long strideC, int splitk, float* workspace, void* stream) {
    B200_TRY(require_device());
    GemmDesc d;
    d.A = A; d.B = B; d.C = C; d.bias = bias; d.M = M; d.N = N; d.K = K; d.lda = lda; d.ldb = ldb; d.ldc = ldc;
    d.transA = transA; d.transB = transB; d.alpha = alpha; d.beta = beta; d.batch = batch < 1 ? 1 : batch;
    d.strideA = strideA; d.strideB = strideB; d.strideC = strideC; d.splitk = splitk < 1 ? 1 : splitk; d.partial = workspace;
    return gemm_run(d, (cudaStream_t)stream);
}

size_t b200tts_decoder_workspace_bytes(const b200tts_decoder_shape* shape) {
    if (!shape || validate_decoder_shape(*shape) != B200TTS_OK) return 0;
    return decoder_layout(step_shape(*shape)).total * sizeof(float);
}

int b200tts_decoder_path(const b200tts_decoder_shape* shape) {
    if (!shape || validate_decoder_shape(*shape) != B200TTS_OK) return 0;
    const PersistPlan p = persist_plan(step_shape(*shape));
    return (p.fwd ? 1 | 2 : 0) | (p.gen_bwd ? 4 | 8 : 0) | (p.att_bwd ? 16 | 32 : 0);
}

size_t b200tts_decoder_bwd_workspace_bytes(const b200tts_decoder_shape* shape) {
    if (!shape || validate_decoder_shape(*shape) != B200TTS_OK) return 0;
    return decoder_bwd_workspace_floats(step_shape(*shape)) * sizeof(float);
}

int b200tts_decoder_forward(const b200tts_decoder_shape* shape, const b200tts_decoder_params* params,
                            const b200tts_decoder_inputs* in, const b200tts_decoder_outputs* out, void* workspace,
                            size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && params && in && out, "decoder_forward: null argument");
    B200_TRY(require_device());
    return decoder_forward_impl(*shape, *params, *in, *out, (float*)workspace, workspace_bytes, (cudaStream_t)stream);
}

int b200tts_decoder_forward_chunk(const b200tts_decoder_shape* shape, const b200tts_decoder_params* params,
                                  const b200tts_decoder_inputs* in, const b200tts_decoder_outputs* out, b200tts_decoder_state* state,
                                  int first, void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && params && in && out && state, "decoder_forward_chunk: null argument");
    B200_REQUIRE(state->att_h && state->att_c && state->gen_h && state->gen_c && state->context && state->cum_weights && state->frame,
                 "decoder_forward_chunk: every state buffer is required");
    B200_REQUIRE(shape->R < 0 || shape->T % frames_per_step(*shape) == 0,
                 "decoder_forward_chunk: a chunk holds whole decoder steps (T=%d is not a multiple of R=%d)", shape->T, shape->R);
    B200_TRY(require_device());
    return decoder_forward_impl(*shape, *params, *in, *out, (float*)workspace, workspace_bytes, (cudaStream_t)stream, state, first);
}

int b200tts_decoder_backward(const b200tts_decoder_shape* shape, const b200tts_decoder_params* params,
                             const b200tts_decoder_inputs* in, const b200tts_decoder_outputs* fwd_out,
                             const b200tts_decoder_output_grads* dout, const void* fwd_workspace, void* bwd_workspace,
                             size_t bwd_workspace_bytes, const b200tts_decoder_params* d_params, float* d_memory,
                             void* stream) {
    B200_REQUIRE(shape && params && in && fwd_out && dout && fwd_workspace && bwd_workspace && d_params,
                 "decoder_backward: null argument");
    B200_TRY(require_device());
    return decoder_backward_impl(*shape, *params, *in, *fwd_out, *dout, (const float*)fwd_workspace, (float*)bwd_workspace,
                                 bwd_workspace_bytes, *d_params, d_memory, (cudaStream_t)stream);
}

size_t b200tts_attention_step_workspace_elems(int B, int L, int A) { return (size_t)B * A + (size_t)B * L; }

int b200tts_attention_step(int B, int L, int M, int D, int A, int C, int K, const float* query, const float* memory,
                           const float* memory_transform, const int32_t* text_lengths, const float* w_query,
                           const float* w_location, const float* w_loc_features, const float* bias, const float* w_energy,
                           float* cum_weights, float* context, float* weights, float* workspace, void* stream) {
    B200_TRY(require_device());
    B200_REQUIRE(query && memory && memory_transform && text_lengths && cum_weights && context && weights && workspace,
                 "attention_step: null argument");
    return attention_step_impl(B, L, M, D, A, C, K, query, memory, memory_transform, text_lengths, w_query, w_location,
                               w_loc_features, bias, w_energy, cum_weights, context, weights, workspace, (cudaStream_t)stream);
}

size_t b200tts_attention_step_backward_workspace_elems(int B, int M, int A, int C, int K) {
    return attention_step_backward_workspace_elems(B, M, A, C, K);
}
int b200tts_attention_step_backward(int B, int L, int M, int A, int C, int K, const float* q, const float* memory,
                                    const float* memory_transform, const int32_t* text_lengths, const float* w_location,
                                    const float* w_loc_features, const float* bias, const float* w_energy, const float* cum_prev,
                                    const float* weights, const float* d_context, const float* d_weights, float* d_cum, float* d_q,
                                    float* d_memory_transform, float* d_w_location, float* d_w_loc_features, float* d_w_energy,
                                    float* workspace, void* stream) {
    B200_TRY(require_device());
    B200_REQUIRE(q && memory && memory_transform && text_lengths && w_location && w_loc_features && bias && w_energy && cum_prev && weights &&
                 d_context && d_cum && d_q && d_memory_transform && d_w_location && d_w_loc_features && d_w_energy && workspace,
                 "attention_step_backward: null argument");
    return attention_step_backward_impl(B, L, M, A, C, K, q, memory, memory_transform, text_lengths, w_location, w_loc_features, bias,
                                        w_energy, cum_prev, weights, d_context, d_weights, d_cum, d_q, d_memory_transform, d_w_location,
                                        d_w_loc_features, d_w_energy, workspace, (cudaStream_t)stream);
}

size_t b200tts_forward_attention_step_workspace_elems(int B, int L, int A) { return (size_t)B * A + (size_t)B * L; }

int b200tts_forward_attention_step(int B, int L, int M, int D, int A, const float* query, const float* memory,
                                   const float* memory_transform, const int32_t* text_lengths, const float* w_query,
                                   const float* bias, const float* w_energy, float* alpha, float* context, float* weights,
                                   float* workspace, void* stream) {
    B200_TRY(require_device());
    B200_REQUIRE(query && memory && memory_transform && text_lengths && w_query && bias && w_energy && alpha && context && weights &&
                 workspace, "forward_attention_step: null argument");
    return forward_attention_step_impl(B, L, M, D, A, query, memory, memory_transform, text_lengths, w_query, bias, w_energy, alpha,
                                       context, weights, workspace, (cudaStream_t)stream);
}

size_t b200tts_forward_attention_step_backward_workspace_elems(int B, int M, int A) {
    return forward_attention_step_backward_workspace_elems(B, M, A);
}
int b200tts_forward_attention_step_backward(int B, int L, int M, int A, const float* q, const float* memory, const float* memory_transform,
                                            const int32_t* text_lengths, const float* bias, const float* w_energy, const float* alpha_prev,
                                            const float* weights, const float* d_context, const float* d_weights, float* d_alpha,
                                            float* d_q, float* d_memory_transform, float* d_w_energy, float* workspace, void* stream) {
    B200_TRY(require_device());
    B200_REQUIRE(q && memory && memory_transform && text_lengths && bias && w_energy && alpha_prev && weights && d_context && d_alpha &&
                 d_q && d_memory_transform && d_w_energy && workspace, "forward_attention_step_backward: null argument");
    return forward_attention_step_backward_impl(B, L, M, A, q, memory, memory_transform, text_lengths, bias, w_energy, alpha_prev,
                                                weights, d_context, d_weights, d_alpha, d_q, d_memory_transform, d_w_energy, workspace,
                                                (cudaStream_t)stream);
}

size_t b200tts_convblock_saved_bytes(const b200tts_convblock_shape* s) { return s ? convblock_saved_floats(*s) * sizeof(float) : 0; }
size_t b200tts_convblock_workspace_bytes(const b200tts_convblock_shape* s) { return s ? convblock_workspace_floats(*s) * sizeof(float) : 0; }

int b200tts_convblock_forward(const b200tts_convblock_shape* shape, const float* x, const float* weight, const float* gamma,
                              const float* beta, int affine_gstride, float* running_mean, float* running_var, const uint8_t* keep,
                              float* out, void* saved, void* workspace, void* stream) {
    B200_REQUIRE(shape && x && out && saved && workspace, "convblock_forward: null argument");
    B200_REQUIRE((weight || shape->stage == 2) && ((gamma && beta) || shape->stage == 1), "convblock_forward: null parameter");
    B200_TRY(require_device());
    return convblock_forward_impl(*shape, x, weight, gamma, beta, affine_gstride, running_mean, running_var, keep, out, (float*)saved,
                                  (float*)workspace, (cudaStream_t)stream);
}

int b200tts_convblock_forward_masked(const b200tts_convblock_shape* shape, const int32_t* lengths, const float* x, const float* weight,
                                     const float* gamma, const float* beta, int affine_gstride, float* running_mean, float* running_var,
                                     const uint8_t* keep, float* out, void* saved, void* workspace, void* stream) {
    B200_REQUIRE(shape && lengths && x && out && saved && workspace, "convblock_forward_masked: null argument");
    B200_REQUIRE(shape->stage == 0 && !shape->training, "convblock_forward_masked: eval mode and the whole block (stage 0) only");
    B200_REQUIRE(weight && gamma && beta, "convblock_forward_masked: null parameter");
    B200_TRY(require_device());
    return convblock_forward_impl(*shape, x, weight, gamma, beta, affine_gstride, running_mean, running_var, keep, out, (float*)saved,
                                  (float*)workspace, (cudaStream_t)stream, lengths);
}

int b200tts_convblock_backward(const b200tts_convblock_shape* shape, const float* x, const float* weight, const float* gamma,
                               const float* beta, int affine_gstride, const uint8_t* keep, const void* saved, const float* dout,
                               float* dx, float* dweight, float* dgamma, float* dbeta, void* workspace, void* stream) {
    B200_REQUIRE(shape && x && saved && dout && workspace, "convblock_backward: null argument");
    B200_REQUIRE((weight || shape->stage == 2) && ((gamma && beta) || shape->stage == 1), "convblock_backward: null parameter");
    B200_REQUIRE(dx || !shape->highway, "convblock_backward: highway blocks need dx");
    B200_TRY(require_device());
    return convblock_backward_impl(*shape, x, weight, gamma, beta, affine_gstride, keep, (const float*)saved, dout, dx, dweight, dgamma,
                                   dbeta, (float*)workspace, (cudaStream_t)stream);
}

int b200tts_lstm_cell_forward(int B, int D, int cell_kind, int training, float rate_h, float rate_c, float* gates, const float* h_prev,
                              const float* c_prev, const uint8_t* mask_h, const uint8_t* mask_c, float* h_out, float* c_out, void* stream) {
    B200_REQUIRE(B > 0 && D > 0 && gates && h_prev && c_prev && h_out && c_out, "lstm_cell_forward: bad argument");
    B200_REQUIRE(cell_kind == B200TTS_CELL_DROPOUT || cell_kind == B200TTS_CELL_ZONEOUT, "lstm_cell_forward: bad cell kind %d", cell_kind);
    B200_REQUIRE(rate_h >= 0.f && rate_h < 1.f && rate_c >= 0.f && rate_c < 1.f, "lstm_cell_forward: rates must be in [0, 1)");
    B200_TRY(require_device());
    CellFwdArgs a{};
    a.xproj = gates; a.gates = gates; a.part = nullptr; a.nsplit = 0; a.part_stride = 0;
    a.c_prev = c_prev; a.h_prev = h_prev; a.ld_hprev = D; a.c_out = c_out; a.h_out = h_out; a.ld_hout = D;
    a.mask_h = mask_h; a.mask_c = mask_c; a.kind = cell_kind; a.training = training; a.rate_h = rate_h; a.rate_c = rate_c;
    a.B = B; a.D = D;
    return launch_cell_fwd(a, (cudaStream_t)stream);
}
int b200tts_lstm_cell_backward(int B, int D, int cell_kind, int training, float rate_h, float rate_c, const float* gates, const float* c_prev,
                               const uint8_t* mask_h, const uint8_t* mask_c, const float* d_h, float* d_c, float* d_h_prev, float* d_gates,
                               void* stream) {
    B200_REQUIRE(B > 0 && D > 0 && gates && c_prev && d_h && d_c && d_h_prev && d_gates, "lstm_cell_backward: bad argument");
    B200_TRY(require_device());
    B200_CUDA(cudaMemsetAsync(d_h_prev, 0, (size_t)B * D * sizeof(float), (cudaStream_t)stream));
    CellBwdArgs a{};
    a.gates = gates; a.c_prev = c_prev; a.dh_static = d_h; a.ld_dhs = D; a.part = nullptr; a.nsplit = 0;
    a.dc_state = d_c; a.dhz_state = d_h_prev;       // in: zero recurrent term; out: the direct (zoneout) gradient of h_prev
    a.mask_h = mask_h; a.mask_c = mask_c; a.kind = cell_kind; a.training = training; a.rate_h = rate_h; a.rate_c = rate_c;
    a.dgates = d_gates; a.B = B; a.D = D; a.last = 0;
    return launch_cell_bwd(a, (cudaStream_t)stream);
}

size_t b200tts_generator_workspace_bytes(int G, int bn) { return generator_workspace_floats(G, bn) * sizeof(float); }

int b200tts_generator_forward(int G, int gd, int bn, long long R, const float* e, const float* Wb, const float* bb, const float* Wk,
                              const float* bk, float* eb, float* out, void* stream) {
    B200_REQUIRE(e && Wb && bb && Wk && bk && eb && out, "generator_forward: null argument");
    B200_TRY(require_device());
    return generator_forward_impl(G, gd, bn, R, e, Wb, bb, Wk, bk, eb, out, (cudaStream_t)stream);
}

int b200tts_generator_backward(int G, int gd, int bn, long long R, const float* e, const float* Wb, const float* Wk, const float* eb,
                               const float* dout, float* de, float* dWb, float* dbb, float* dWk, float* dbk, void* workspace,
                               void* stream) {
    B200_REQUIRE(e && Wb && Wk && eb && dout && de && dWb && dbb && dWk && dbk && workspace, "generator_backward: null argument");
    B200_TRY(require_device());
    return generator_backward_impl(G, gd, bn, R, e, Wb, Wk, eb, dout, de, dWb, dbb, dWk, dbk, (float*)workspace, (cudaStream_t)stream);
}

int b200tts_embedding_forward(float* out, int ldo, const float* table, const int32_t* ids, long long ntok, int E, void* stream) {
    B200_REQUIRE(out && table && ids && ntok >= 0 && E > 0 && ldo >= E, "embedding_forward: bad argument");
    B200_TRY(require_device());
    return embedding_forward_impl(out, ldo, table, ids, ntok, E, (cudaStream_t)stream);
}

int b200tts_embedding_backward(float* dtable, int V, const float* dout, int ldo, const int32_t* ids, long long ntok, int E,
                               int padding_idx, void* stream) {
    B200_REQUIRE(dtable && dout && ids && V > 0 && E > 0 && ldo >= E, "embedding_backward: bad argument");
    B200_TRY(require_device());
    return embedding_backward_impl(dtable, V, dout, ldo, ids, ntok, E, padding_idx, (cudaStream_t)stream);
}

size_t b200tts_bilstm_saved_bytes(const b200tts_bilstm_shape* s) { return s ? bilstm_saved_floats(*s) * sizeof(float) : 0; }
size_t b200tts_bilstm_workspace_bytes(const b200tts_bilstm_shape* s) { return s ? bilstm_workspace_floats(*s) * sizeof(float) : 0; }

int b200tts_bilstm_forward(const b200tts_bilstm_shape* shape, const b200tts_bilstm_params* params, const float* x,
                           const int32_t* lengths, float* out, void* saved, void* workspace, void* stream) {
    B200_REQUIRE(shape && params && x && lengths && out && saved && workspace, "bilstm_forward: null argument");
    B200_TRY(require_device());
    return bilstm_forward_impl(*shape, *params, x, lengths, out, (float*)saved, (float*)workspace, (cudaStream_t)stream);
}

int b200tts_bilstm_backward(const b200tts_bilstm_shape* shape, const b200tts_bilstm_params* params, const int32_t* lengths,
                            const void* saved, const float* dout, float* dx, const b200tts_bilstm_params* d_params, void* workspace,
                            void* stream) {
    B200_REQUIRE(shape && params && lengths && saved && dout && d_params && workspace, "bilstm_backward: null argument");
    B200_TRY(require_device());
    return bilstm_backward_impl(*shape, *params, lengths, (const float*)saved, dout, dx, *d_params, (float*)workspace, (cudaStream_t)stream);
}

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
    const unsigned long long key = mix64(seed ^ 0xD6E8FEB86659FD93ull) ^ (stream_id * 0xA24BAED4963EE407ull);
    size_t quads = (n + 15) / 16;
    int blocks = (int)((quads + 255) / 256 > NUM_SMS * 16 ? NUM_SMS * 16 : (quads + 255) / 256);
    if (blocks < 1) blocks = 1;
    fill_keep_mask_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(mask, n, threshold, key, g_mask_epoch);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

size_t b200tts_loss_workspace_bytes(void) { return loss_workspace_floats() * sizeof(float); }
int b200tts_tacotron_loss_forward(const b200tts_loss_shape* shape, const float* pre, const float* pre_target, const float* post,
                                  const float* post_target, const float* stop, const float* stop_target, const float* alignment,
                                  const int32_t* text_lengths, const int32_t* target_lengths, float* losses, void* workspace, void* stream) {
    B200_REQUIRE(shape && pre && pre_target && post && post_target && stop && stop_target && text_lengths && target_lengths && losses && workspace,
                 "tacotron_loss_forward: null argument");
    B200_REQUIRE(alignment || !shape->guided, "tacotron_loss_forward: guided attention needs the alignments");
    B200_TRY(require_device());
    return loss_forward_impl(*shape, pre, pre_target, post, post_target, stop, stop_target, alignment, text_lengths, target_lengths, losses,
                             (float*)workspace, (cudaStream_t)stream);
}
int b200tts_tacotron_loss_backward(const b200tts_loss_shape* shape, const float* pre, const float* pre_target, const float* post,
                                   const float* post_target, const float* stop, const float* stop_target, const int32_t* text_lengths,
                                   const int32_t* target_lengths, const float* grad_losses, float* d_pre, float* d_post, float* d_stop,
                                   float* d_alignment, void* stream) {
    B200_REQUIRE(shape && pre && pre_target && post && post_target && stop && stop_target && text_lengths && target_lengths && grad_losses,
                 "tacotron_loss_backward: null argument");
    B200_TRY(require_device());
    return loss_backward_impl(*shape, pre, pre_target, post, post_target, stop, stop_target, text_lengths, target_lengths, grad_losses, d_pre,
                              d_post, d_stop, d_alignment, (cudaStream_t)stream);
}

size_t b200tts_adam_clip_scratch_floats(void) { return adam_clip_scratch_floats(); }
int b200tts_adam_clip_step(float* p, float* g, float* m, float* v, size_t n, float lr, float beta1, float beta2, float eps,
                           float weight_decay, float max_norm, int step, float* scratch, void* stream) {
    B200_TRY(require_device());
    return adam_clip_step_impl(p, g, m, v, n, lr, beta1, beta2, eps, weight_decay, max_norm, step, scratch, (cudaStream_t)stream);
}

}  // extern "C"
