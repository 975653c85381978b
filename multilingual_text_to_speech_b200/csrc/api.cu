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
int decoder_state_reset_rows_check(const b200tts_decoder_shape& s, const b200tts_decoder_state& state, const int* rows, int count);
int decoder_state_reset_rows_impl(const b200tts_decoder_shape& s, const b200tts_decoder_state& state, const int* rows, int count,
                                  cudaStream_t st);
int decoder_backward_impl(const b200tts_decoder_shape& s, const b200tts_decoder_params& w, const b200tts_decoder_inputs& in,
                          const b200tts_decoder_outputs& fwd_out, const b200tts_decoder_output_grads& dout, const float* fws,
                          float* bws, size_t bws_bytes, const b200tts_decoder_params& dw, float* d_memory, cudaStream_t st);
size_t decoder_bwd_workspace_floats(const b200tts_decoder_shape& s);
size_t attention_step_backward_workspace_elems(int B, int M, int A, int C, int K);
int attention_step_backward_validate(int B, int L, int M, int A, int C, int K);
int attention_backward_chunk(int L, int M, int A, int C, int K);
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
                           float* out, float* saved, float* ws, cudaStream_t st, const int32_t* lengths = nullptr,
                           const int32_t* counts = nullptr);
int convblock_backward_impl(const b200tts_convblock_shape& s, const float* x, const float* weight, const float* gamma,
                            const float* beta, int affine_gstride, const uint8_t* keep, const float* saved, const float* dout,
                            float* dx, float* dweight, float* dgamma, float* dbeta, float* ws, cudaStream_t st,
                            const int32_t* counts = nullptr);
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
void bilstm_view_offsets(const b200tts_bilstm_shape& s, size_t* v);
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
size_t vocoder_workspace_bytes(const b200tts_vocoder_shape& s);
int vocoder_fft_plan(int N, int* radices, int capacity);
int spectrogram_magnitude_impl(const b200tts_vocoder_shape& s, const float* log_spec, const float* mel_basis, const float* mel_pinv_t,
                               float nnls_step, float* S, cudaStream_t st);
int griffinlim_impl(const b200tts_vocoder_shape& s, const float* S, const int* off, float* angles, float* rebuilt, int first, int iters,
                    float* wave, void* ws, size_t ws_bytes, cudaStream_t st);
int deemphasis_normalize_impl(const b200tts_vocoder_shape& s, float* wave, const int* off, cudaStream_t st);
size_t gl_stream_workspace_bytes(const b200tts_gl_stream_shape& s);
int gl_stream_reset_check(const b200tts_gl_stream_shape& s, void* ws, size_t ws_bytes, const int* list, int count);
int gl_stream_reset_impl(const b200tts_gl_stream_shape& s, void* ws, const int* list, int count, cudaStream_t st);
int gl_stream_run_check(const b200tts_gl_stream_shape& s, const b200tts_gl_stream_row* rows, int count, void* ws, size_t ws_bytes);
int gl_stream_run_impl(const b200tts_gl_stream_shape& s, const b200tts_gl_stream_row* rows, int count, const float* S_new, float* wave, void* ws,
                       cudaStream_t st);
size_t analysis_workspace_bytes(const b200tts_analysis_shape& s);
int stft_magnitude_impl(const b200tts_analysis_shape& s, const float* wave, const int* soff, const int* off, const float* mel_basis, float* out,
                        void* ws, size_t ws_bytes, cudaStream_t st);
int amplitude_to_db_impl(const b200tts_analysis_shape& s, const float* S, const int* off, float* out, cudaStream_t st);
int mel_cepstrum_validate(int total_frames, int n_mels, int n_mfcc);
int mcd_validate(int B, int n_mfcc, int mode);
int mel_cepstrum_impl(int total_frames, int n_mels, int n_mfcc, const float* mel_db, float* out, cudaStream_t st);
int mel_cepstral_distortion_impl(int B, int n_mfcc, int mode, const float* cep_a, const int* off_a, const float* cep_b, const int* off_b,
                                 double* mcd, int* path_len, cudaStream_t st);
int align_validate(const b200tts_align_shape& s);
int monotonic_alignment_impl(const b200tts_align_shape& s, const float* P, const int* text_lengths, const int* step_lengths, int* durations,
                             double* path_logp, int* path, cudaStream_t st);
int alignment_scores_impl(const b200tts_align_shape& s, const float* P, const int* text_lengths, const int* step_lengths, float* focus,
                          float* coverage, int* max_jump, int* moves_back, cudaStream_t st);
int wavernn_upsample_layer_check(int C, int len, int scale);
int wavernn_upsample_layer_impl(int C, int len, int scale, const float* fir, const float* in, float* out, cudaStream_t st);
int wavernn_fold_check(const b200tts_wavernn_fold_shape& s, int t0, int nsteps);
int wavernn_fold_impl(const b200tts_wavernn_fold_shape& s, const float* mel_up, const long long* mel_off, const int* frames, const int* row_utt,
                      const int* row_fold, const float* fir, const float* aux, int t0, int nsteps, float* feat, cudaStream_t st);
int wavernn_window_check(const b200tts_wavernn_window_shape& s, long long s0, int nsteps);
int wavernn_run_stream_impl(const b200tts_wavernn_shape& s, const b200tts_wavernn_params& p, const b200tts_wavernn_cond& cond, long long t,
                            int nsteps, const float* uniforms, float* out, void* ws, size_t ws_bytes, cudaStream_t st);
size_t wavernn_workspace_bytes(const b200tts_wavernn_shape& s);
int wavernn_check(const b200tts_wavernn_shape& s, void* ws, size_t ws_bytes);
int wavernn_prepare_impl(const b200tts_wavernn_shape& s, const b200tts_wavernn_params& p, void* ws, size_t ws_bytes, cudaStream_t st);
int wavernn_run_impl(const b200tts_wavernn_shape& s, const b200tts_wavernn_params& p, const b200tts_wavernn_cond& cond, int t0, int nsteps,
                     const float* uniforms, float* out, float* dbg, void* ws, size_t ws_bytes, cudaStream_t st);
int wavernn_run_rows_check(const b200tts_wavernn_shape& s, int active_rows, int nsteps);
int wavernn_run_rows_impl(const b200tts_wavernn_shape& s, const b200tts_wavernn_params& p, const b200tts_wavernn_cond& cond, const long long* row_t,
                          const int* row_n, int active_rows, int nsteps, const float* uniforms, float* out, void* ws, size_t ws_bytes,
                          cudaStream_t st);
int wavernn_reset_rows_check(const b200tts_wavernn_shape& s, const int* rows, int count);
int wavernn_reset_rows_impl(const b200tts_wavernn_shape& s, void* ws, size_t ws_bytes, const int* rows, int count, cudaStream_t st);
int wavernn_window_rows_check(const b200tts_wavernn_window_row* rows, int active_rows, int nsteps);
int wavernn_window_rows_impl(const b200tts_wavernn_window_row* rows, int active_rows, int nsteps, const float* mel, const float* fir,
                             const float* aux, float* feat, cudaStream_t st);
int wavernn_upsample_segments_check(int C, int nseg, const int* lens, int scale);
int wavernn_upsample_segments_impl(int C, int nseg, const int* lens, int scale, const float* fir, const float* in, float* out, cudaStream_t st);
int wavernn_aborted_impl(const b200tts_wavernn_shape& s, const void* ws, size_t ws_bytes, int* aborted, cudaStream_t st);
int wavernn_deemphasis_check(int rows, int len, int mu, float a);
int wavernn_deemphasis_impl(int rows, int len, int mu, float a, float* y, cudaStream_t st);
int wavernn_unfold_check(int B, int hop, int target, int overlap, int mu);
int wavernn_unfold_impl(int B, int hop, int target, int overlap, int mu, const int* frames, const int* row_off, const long long* wave_off,
                        long long total, const float* y, float* wave, cudaStream_t st);
int wavernn_unfold_streams_check(int nstreams, int hop, int target, int overlap, int mu, const b200tts_wavernn_unfold_stream* streams,
                                 int nsrc, long long total);
int wavernn_unfold_streams_impl(int nstreams, int hop, int target, int overlap, int mu, const b200tts_wavernn_unfold_stream* streams,
                                const long long* base, const int* period, int nsrc, long long total, const float* y, float* wave,
                                cudaStream_t st);
size_t gru_seq_saved_bytes(const b200tts_gru_seq_shape& s);
size_t gru_seq_workspace_bytes(const b200tts_gru_seq_shape& s);
int gru_seq_check(const b200tts_gru_seq_shape& s, void* ws, size_t ws_bytes);
int gru_seq_forward_impl(const b200tts_gru_seq_shape& s, const float* gi, const float* w_hh, const float* b_hh, float* h, void* saved, void* ws,
                         size_t ws_bytes, cudaStream_t st);
int gru_seq_backward_impl(const b200tts_gru_seq_shape& s, const float* w_hh, const float* h, const void* saved, const float* dh_ext, float* dgi,
                          float* dgh, float* dh_dbg, void* ws, size_t ws_bytes, cudaStream_t st);
int gru_seq_aborted_impl(const b200tts_gru_seq_shape& s, const void* ws, size_t ws_bytes, int* aborted, cudaStream_t st);
int gru_seq_abort_flag_copy_impl(const b200tts_gru_seq_shape& s, const void* ws, size_t ws_bytes, int* dst, cudaStream_t st);
int wavernn_cut_windows_check(int mode, int bits, int B, int feat, int seq_len, int pad, int hop, long long total_frames);
int wavernn_cut_windows_impl(int mode, int bits, int B, int feat, int seq_len, int pad, int hop, const float* mels, long long total_frames,
                             const long long* frame_start, const unsigned short* labels, const long long* sample_start, const int* table,
                             float* x, void* y, float* m, cudaStream_t st);
size_t wavernn_upsample_layer_backward_workspace_bytes(int C, int len, int scale);
int wavernn_upsample_layer_backward_impl(int C, int len, int scale, const float* fir, const float* in, const float* dout, float* din, float* dfir,
                                         void* ws, size_t ws_bytes, cudaStream_t st);
int wavernn_stretch_backward_check(int B, int F, int C, int hop);
int wavernn_stretch_backward_impl(int B, int F, int C, int hop, const float* dup, float* daux, cudaStream_t st);
int wavernn_loss_check(int mode, long long N, int n_out);
size_t wavernn_loss_workspace_bytes(long long N);
size_t column_sum_workspace_bytes(int cols);
int column_sum_check(long long rows, int cols);
int column_sum_impl(long long rows, int cols, const float* x, float* out, void* ws, size_t ws_bytes, cudaStream_t st);
int wavernn_loss_impl(int mode, long long N, int n_out, const float* logits, const void* target, float* loss, float* dlogits, void* ws,
                      size_t ws_bytes, cudaStream_t st);
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
int b200tts_debug_decoder_geometry(const b200tts_decoder_shape* shape, int* out, int n) {
    if (!shape || !out || validate_decoder_shape(*shape) != B200TTS_OK) return 0;
    const b200tts_decoder_shape s = step_shape(*shape);
    const TcPersistGeom g = tc_persist_geom(s);
    const AttBwdGeom ab = att_bwd_geom(s);
    const int v[14] = {b200tts_decoder_path(shape), g.grid, g.NBH, g.slot_kb_att, g.ch_h_att, g.ch_h_att ? g.nkb_h / g.ch_h_att : 0, g.ch_c_att,
                       g.n_c_att, g.alias_att, g.use_btab, g.slot_gen, g.ch_h_gen, ab.UN, ab.grid};
    const int m = n < 14 ? n : 14;
    for (int k = 0; k < m; ++k) out[k] = v[k];
    return m;
}
int b200tts_debug_bilstm_layout(const b200tts_bilstm_shape* shape, size_t* out, int n) {
    if (!shape || !out || shape->B <= 0 || shape->L <= 0 || shape->E <= 0 || shape->H <= 0) return 0;
    size_t v[10];
    bilstm_view_offsets(*shape, v);
    const int m = n < 10 ? n : 10;
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

static_assert(sizeof(b200tts_gemm_desc) == sizeof(GemmDesc), "b200tts_gemm_desc must list the fields of GemmDesc");
int b200tts_debug_gemm(const b200tts_gemm_desc* desc, int route, float* partial, size_t partial_elems, void* stream) {
    B200_REQUIRE(desc, "debug_gemm: null descriptor");
    B200_REQUIRE(route == 0 || route == 1, "debug_gemm: unknown route %d", route);
    B200_TRY(require_device());
    const b200tts_gemm_desc& s = *desc;
    GemmDesc d;
    d.A = s.A; d.B = s.B; d.C = s.C; d.bias = s.bias;
    d.M = s.M; d.N = s.N; d.K = s.K; d.lda = s.lda; d.ldb = s.ldb; d.ldc = s.ldc;
    d.transA = s.transA; d.transB = s.transB; d.alpha = s.alpha; d.beta = s.beta;
    d.batch = s.batch; d.strideA = s.strideA; d.strideB = s.strideB; d.strideC = s.strideC; d.a_batch_mod = s.a_batch_mod;
    d.splitk = s.splitk; d.partial = s.partial; d.keep_partials = s.keep_partials;
    d.A16 = s.A16; d.lda16 = s.lda16; d.B16 = s.B16; d.ldb16 = s.ldb16;
    d.kin = s.kin; d.kosA = s.kosA; d.kosB = s.kosB;
    if (route == 0) return gemm_run(d, (cudaStream_t)stream);
    return gemm_run_auto(d, partial, partial ? partial_elems : 0, (cudaStream_t)stream);
}

int b200tts_debug_gemm_pack_cache(int open) {
    if (open) tc_pack_cache_begin();
    else tc_pack_cache_end();
    return B200TTS_OK;
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

static bool forced_inputs(const b200tts_decoder_inputs& in) { return in.forced_count != 0 || in.forced_rows || in.forced_alignment; }

int b200tts_decoder_forward(const b200tts_decoder_shape* shape, const b200tts_decoder_params* params,
                            const b200tts_decoder_inputs* in, const b200tts_decoder_outputs* out, void* workspace,
                            size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && params && in && out, "decoder_forward: null argument");
    B200_REQUIRE(shape->att_window_back == 0 && shape->att_window_ahead == 0,
                 "decoder_forward: an attention window is for synthesis only (b200tts_decoder_forward_chunk)");
    B200_REQUIRE(!forced_inputs(*in), "decoder_forward: forced attention rows are for synthesis only (b200tts_decoder_forward_chunk)");
    B200_TRY(require_device());
    return decoder_forward_impl(*shape, *params, *in, *out, (float*)workspace, workspace_bytes, (cudaStream_t)stream);
}

int b200tts_decoder_forward_chunk(const b200tts_decoder_shape* shape, const b200tts_decoder_params* params,
                                  const b200tts_decoder_inputs* in, const b200tts_decoder_outputs* out, b200tts_decoder_state* state,
                                  int first, void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && params && in && out && state, "decoder_forward_chunk: null argument");
    B200_REQUIRE(state->att_h && state->att_c && state->gen_h && state->gen_c && state->context && state->cum_weights && state->frame,
                 "decoder_forward_chunk: every state buffer is required");
    B200_REQUIRE(!attention_window(*shape) || state->attended, "decoder_forward_chunk: an attention window needs state->attended");
    B200_REQUIRE(in->forced_count >= 0 && in->forced_count <= shape->B,
                 "decoder_forward_chunk: forced_count %d outside [0, B=%d]", in->forced_count, shape->B);
    B200_REQUIRE(in->forced_count == 0 ? !in->forced_rows && !in->forced_alignment : in->forced_rows && in->forced_alignment,
                 "decoder_forward_chunk: forced_rows and forced_alignment are given exactly when forced_count > 0");
    B200_REQUIRE(shape->R < 0 || shape->T % frames_per_step(*shape) == 0,
                 "decoder_forward_chunk: a chunk holds whole decoder steps (T=%d is not a multiple of R=%d)", shape->T, shape->R);
    B200_TRY(require_device());
    return decoder_forward_impl(*shape, *params, *in, *out, (float*)workspace, workspace_bytes, (cudaStream_t)stream, state, first);
}

int b200tts_decoder_state_reset_rows(const b200tts_decoder_shape* shape, b200tts_decoder_state* state, const int32_t* rows, int count,
                                     void* stream) {
    B200_REQUIRE(shape && state, "decoder_state_reset_rows: null argument");
    B200_TRY(decoder_state_reset_rows_check(*shape, *state, rows, count));
    B200_TRY(require_device());
    return decoder_state_reset_rows_impl(*shape, *state, rows, count, (cudaStream_t)stream);
}

int b200tts_decoder_backward(const b200tts_decoder_shape* shape, const b200tts_decoder_params* params,
                             const b200tts_decoder_inputs* in, const b200tts_decoder_outputs* fwd_out,
                             const b200tts_decoder_output_grads* dout, const void* fwd_workspace, void* bwd_workspace,
                             size_t bwd_workspace_bytes, const b200tts_decoder_params* d_params, float* d_memory,
                             void* stream) {
    B200_REQUIRE(shape && params && in && fwd_out && dout && fwd_workspace && bwd_workspace && d_params,
                 "decoder_backward: null argument");
    B200_REQUIRE(shape->att_window_back == 0 && shape->att_window_ahead == 0,
                 "decoder_backward: an attention window is for synthesis only (b200tts_decoder_forward_chunk)");
    B200_REQUIRE(!forced_inputs(*in), "decoder_backward: forced attention rows are for synthesis only (b200tts_decoder_forward_chunk)");
    B200_TRY(require_device());
    return decoder_backward_impl(*shape, *params, *in, *fwd_out, *dout, (const float*)fwd_workspace, (float*)bwd_workspace,
                                 bwd_workspace_bytes, *d_params, d_memory, (cudaStream_t)stream);
}

size_t b200tts_attention_step_workspace_elems(int B, int L, int A) { return (size_t)B * A + (size_t)B * L; }

int b200tts_attention_step(int B, int L, int M, int D, int A, int C, int K, const float* query, const float* memory,
                           const float* memory_transform, const int32_t* text_lengths, const float* w_query,
                           const float* w_location, const float* w_loc_features, const float* bias, const float* w_energy,
                           float* cum_weights, float* context, float* weights, float* workspace, void* stream) {
    B200_REQUIRE(query && memory && memory_transform && text_lengths && w_query && w_location && w_loc_features && bias && w_energy &&
                 cum_weights && context && weights && workspace, "attention_step: null argument");
    B200_REQUIRE(B > 0 && L > 0 && M > 0 && D > 0 && A > 0 && C > 0 && K > 0,
                 "attention_step: non-positive dimension (B=%d L=%d M=%d D=%d A=%d C=%d K=%d)", B, L, M, D, A, C, K);
    B200_REQUIRE(A % 4 == 0, "attention_step: attention dimension %d must be a multiple of 4", A);
    B200_TRY(require_device());
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
    B200_REQUIRE(q && memory && memory_transform && text_lengths && w_location && w_loc_features && bias && w_energy && cum_prev && weights &&
                 d_context && d_cum && d_q && d_memory_transform && d_w_location && d_w_loc_features && d_w_energy && workspace,
                 "attention_step_backward: null argument");
    B200_TRY(attention_step_backward_validate(B, L, M, A, C, K));
    B200_TRY(require_device());
    return attention_step_backward_impl(B, L, M, A, C, K, q, memory, memory_transform, text_lengths, w_location, w_loc_features, bias,
                                        w_energy, cum_prev, weights, d_context, d_weights, d_cum, d_q, d_memory_transform, d_w_location,
                                        d_w_loc_features, d_w_energy, workspace, (cudaStream_t)stream);
}

int b200tts_debug_attention_backward_chunk(int L, int M, int A, int C, int K) { return attention_backward_chunk(L, M, A, C, K); }

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

int b200tts_convblock_forward_counts(const b200tts_convblock_shape* shape, const int32_t* counts, int G, int NB, const float* x,
                                     const float* weight, const float* gamma, const float* beta, int affine_gstride, float* running_mean,
                                     float* running_var, const uint8_t* keep, float* out, void* saved, void* workspace, void* stream) {
    B200_REQUIRE(shape && counts && x && out && saved && workspace, "convblock_forward_counts: null argument");
    B200_REQUIRE(G == shape->G && NB == shape->NB, "convblock_forward_counts: counts are for G=%d, NB=%d but the shape has G=%d, NB=%d", G, NB,
                 shape->G, shape->NB);
    B200_REQUIRE((weight || shape->stage == 2) && ((gamma && beta) || shape->stage == 1), "convblock_forward_counts: null parameter");
    B200_TRY(require_device());
    return convblock_forward_impl(*shape, x, weight, gamma, beta, affine_gstride, running_mean, running_var, keep, out, (float*)saved,
                                  (float*)workspace, (cudaStream_t)stream, nullptr, counts);
}

int b200tts_convblock_backward_counts(const b200tts_convblock_shape* shape, const int32_t* counts, int G, int NB, const float* x,
                                      const float* weight, const float* gamma, const float* beta, int affine_gstride, const uint8_t* keep,
                                      const void* saved, const float* dout, float* dx, float* dweight, float* dgamma, float* dbeta,
                                      void* workspace, void* stream) {
    B200_REQUIRE(shape && counts && x && saved && dout && workspace, "convblock_backward_counts: null argument");
    B200_REQUIRE(G == shape->G && NB == shape->NB, "convblock_backward_counts: counts are for G=%d, NB=%d but the shape has G=%d, NB=%d", G, NB,
                 shape->G, shape->NB);
    B200_REQUIRE((weight || shape->stage == 2) && ((gamma && beta) || shape->stage == 1), "convblock_backward_counts: null parameter");
    B200_REQUIRE(dx || !shape->highway, "convblock_backward_counts: highway blocks need dx");
    B200_TRY(require_device());
    return convblock_backward_impl(*shape, x, weight, gamma, beta, affine_gstride, keep, (const float*)saved, dout, dx, dweight, dgamma,
                                   dbeta, (float*)workspace, (cudaStream_t)stream, counts);
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
    B200_REQUIRE(cell_kind == B200TTS_CELL_DROPOUT || cell_kind == B200TTS_CELL_ZONEOUT, "lstm_cell_backward: bad cell kind %d", cell_kind);
    B200_REQUIRE(rate_h >= 0.f && rate_h < 1.f && rate_c >= 0.f && rate_c < 1.f, "lstm_cell_backward: rates must be in [0, 1)");
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

size_t b200tts_vocoder_workspace_bytes(const b200tts_vocoder_shape* shape) {
    if (!shape) { set_last_error("vocoder_workspace_bytes: null shape"); return 0; }
    return vocoder_workspace_bytes(*shape);
}
int b200tts_vocoder_fft_plan(int N, int* radices, int capacity) {
    B200_REQUIRE(radices || capacity == 0, "vocoder_fft_plan: null radices");
    return vocoder_fft_plan(N, radices, capacity);
}
int b200tts_spectrogram_magnitude(const b200tts_vocoder_shape* shape, const float* log_spec, const float* mel_basis, const float* mel_pinv_t,
                                  float nnls_step, float* S_out, void* stream) {
    B200_REQUIRE(shape && log_spec && S_out, "spectrogram_magnitude: null argument");
    B200_TRY(require_device());
    return spectrogram_magnitude_impl(*shape, log_spec, mel_basis, mel_pinv_t, nnls_step, S_out, (cudaStream_t)stream);
}
int b200tts_griffinlim(const b200tts_vocoder_shape* shape, const float* S, const int32_t* off, float* angles, float* rebuilt, int first,
                       int iters, float* wave, void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && S && off && angles && rebuilt, "griffinlim: null argument");
    B200_TRY(require_device());
    return griffinlim_impl(*shape, S, off, angles, rebuilt, first, iters, wave, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_deemphasis_normalize(const b200tts_vocoder_shape* shape, float* wave, const int32_t* off, void* stream) {
    B200_REQUIRE(shape && wave && off, "deemphasis_normalize: null argument");
    B200_TRY(require_device());
    return deemphasis_normalize_impl(*shape, wave, off, (cudaStream_t)stream);
}

size_t b200tts_gl_stream_workspace_bytes(const b200tts_gl_stream_shape* shape) {
    if (!shape) { set_last_error("gl_stream_workspace_bytes: null shape"); return 0; }
    return gl_stream_workspace_bytes(*shape);
}
int b200tts_gl_stream_reset(const b200tts_gl_stream_shape* shape, void* workspace, size_t workspace_bytes, const int32_t* slots, int count,
                            void* stream) {
    B200_REQUIRE(shape, "gl_stream_reset: null argument");
    B200_TRY(gl_stream_reset_check(*shape, workspace, workspace_bytes, slots, count));
    B200_TRY(require_device());
    return gl_stream_reset_impl(*shape, workspace, slots, count, (cudaStream_t)stream);
}
int b200tts_gl_stream_run(const b200tts_gl_stream_shape* shape, const b200tts_gl_stream_row* rows, int count, const float* S_new, float* wave,
                          void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && S_new && wave, "gl_stream_run: null argument");
    B200_TRY(gl_stream_run_check(*shape, rows, count, workspace, workspace_bytes));
    B200_TRY(require_device());
    return gl_stream_run_impl(*shape, rows, count, S_new, wave, workspace, (cudaStream_t)stream);
}

size_t b200tts_analysis_workspace_bytes(const b200tts_analysis_shape* shape) {
    if (!shape) { set_last_error("analysis_workspace_bytes: null shape"); return 0; }
    return analysis_workspace_bytes(*shape);
}
int b200tts_stft_magnitude(const b200tts_analysis_shape* shape, const float* wave, const int32_t* soff, const int32_t* off,
                           const float* mel_basis, float* out, void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && wave && soff && off && out, "stft_magnitude: null argument");
    B200_TRY(require_device());
    return stft_magnitude_impl(*shape, wave, soff, off, mel_basis, out, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_amplitude_to_db(const b200tts_analysis_shape* shape, const float* S, const int32_t* off, float* out, void* stream) {
    B200_REQUIRE(shape && S && off && out, "amplitude_to_db: null argument");
    B200_TRY(require_device());
    return amplitude_to_db_impl(*shape, S, off, out, (cudaStream_t)stream);
}
int b200tts_mel_cepstrum(int total_frames, int n_mels, int n_mfcc, const float* mel_db, float* out, void* stream) {
    B200_REQUIRE(mel_db && out, "mel_cepstrum: null argument");
    B200_TRY(mel_cepstrum_validate(total_frames, n_mels, n_mfcc));
    B200_TRY(require_device());
    return mel_cepstrum_impl(total_frames, n_mels, n_mfcc, mel_db, out, (cudaStream_t)stream);
}
int b200tts_mel_cepstral_distortion(int B, int n_mfcc, int mode, const float* cep_a, const int32_t* off_a, const float* cep_b,
                                    const int32_t* off_b, double* mcd_out, int32_t* path_len_out, void* stream) {
    B200_REQUIRE(cep_a && off_a && cep_b && off_b && mcd_out, "mel_cepstral_distortion: null argument");
    B200_TRY(mcd_validate(B, n_mfcc, mode));
    B200_TRY(require_device());
    return mel_cepstral_distortion_impl(B, n_mfcc, mode, cep_a, off_a, cep_b, off_b, mcd_out, path_len_out, (cudaStream_t)stream);
}

int b200tts_monotonic_alignment(const b200tts_align_shape* shape, const float* P, const int32_t* text_lengths, const int32_t* step_lengths,
                                int32_t* durations_out, double* path_logp_out, int32_t* path_out, void* stream) {
    B200_REQUIRE(shape && P && text_lengths && step_lengths && durations_out && path_logp_out, "monotonic_alignment: null argument");
    B200_TRY(align_validate(*shape));
    B200_TRY(require_device());
    return monotonic_alignment_impl(*shape, P, text_lengths, step_lengths, durations_out, path_logp_out, path_out, (cudaStream_t)stream);
}
int b200tts_alignment_scores(const b200tts_align_shape* shape, const float* P, const int32_t* text_lengths, const int32_t* step_lengths,
                             float* focus_out, float* coverage_out, int32_t* max_jump_out, int32_t* moves_back_out, void* stream) {
    B200_REQUIRE(shape && P && text_lengths && step_lengths && focus_out && coverage_out && max_jump_out && moves_back_out,
                 "alignment_scores: null argument");
    B200_TRY(align_validate(*shape));
    B200_TRY(require_device());
    return alignment_scores_impl(*shape, P, text_lengths, step_lengths, focus_out, coverage_out, max_jump_out, moves_back_out,
                                 (cudaStream_t)stream);
}

int b200tts_wavernn_upsample_layer(int C, int len, int scale, const float* fir, const float* in, float* out, void* stream) {
    B200_REQUIRE(fir && in && out, "wavernn_upsample_layer: null argument");
    B200_TRY(wavernn_upsample_layer_check(C, len, scale));
    B200_TRY(require_device());
    return wavernn_upsample_layer_impl(C, len, scale, fir, in, out, (cudaStream_t)stream);
}
int b200tts_wavernn_fold(const b200tts_wavernn_fold_shape* shape, const float* mel_up, const int64_t* mel_off, const int32_t* frames,
                         const int32_t* row_utt, const int32_t* row_fold, const float* fir, const float* aux, int t0, int nsteps, float* feat,
                         void* stream) {
    B200_REQUIRE(shape && mel_up && mel_off && frames && row_utt && row_fold && fir && feat, "wavernn_fold: null argument");
    B200_REQUIRE(aux || shape->aux_dims == 0, "wavernn_fold: null aux");
    B200_TRY(wavernn_fold_check(*shape, t0, nsteps));
    B200_TRY(require_device());
    return wavernn_fold_impl(*shape, mel_up, reinterpret_cast<const long long*>(mel_off), frames, row_utt, row_fold, fir, aux, t0, nsteps, feat,
                             (cudaStream_t)stream);
}
size_t b200tts_wavernn_workspace_bytes(const b200tts_wavernn_shape* shape) {
    if (!shape) { set_last_error("wavernn_workspace_bytes: null shape"); return 0; }
    return wavernn_workspace_bytes(*shape);
}
int b200tts_wavernn_prepare(const b200tts_wavernn_shape* shape, const b200tts_wavernn_params* params, void* workspace, size_t workspace_bytes,
                            void* stream) {
    B200_REQUIRE(shape && params, "wavernn_prepare: null argument");
    B200_TRY(wavernn_check(*shape, workspace, workspace_bytes));
    B200_TRY(require_device());
    return wavernn_prepare_impl(*shape, *params, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_wavernn_run(const b200tts_wavernn_shape* shape, const b200tts_wavernn_params* params, const b200tts_wavernn_cond* cond, int t0,
                        int nsteps, const float* uniforms, float* out, float* dbg, void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && params && cond, "wavernn_run: null argument");
    B200_TRY(wavernn_check(*shape, workspace, workspace_bytes));
    B200_TRY(require_device());
    return wavernn_run_impl(*shape, *params, *cond, t0, nsteps, uniforms, out, dbg, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_wavernn_run_stream(const b200tts_wavernn_shape* shape, const b200tts_wavernn_params* params, const b200tts_wavernn_cond* cond,
                               long long t, int nsteps, const float* uniforms, float* out, void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && params && cond, "wavernn_run_stream: null argument");
    B200_TRY(wavernn_check(*shape, workspace, workspace_bytes));
    B200_TRY(require_device());
    return wavernn_run_stream_impl(*shape, *params, *cond, t, nsteps, uniforms, out, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_wavernn_run_rows(const b200tts_wavernn_shape* shape, const b200tts_wavernn_params* params, const b200tts_wavernn_cond* cond,
                             const int64_t* row_t, const int32_t* row_n, int active_rows, int nsteps, const float* uniforms, float* out,
                             void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && params && cond, "wavernn_run_rows: null argument");
    B200_REQUIRE(row_t && row_n && uniforms && out, "wavernn_run_rows: null row_t, row_n, uniforms or output");
    B200_TRY(wavernn_check(*shape, workspace, workspace_bytes));
    B200_TRY(wavernn_run_rows_check(*shape, active_rows, nsteps));
    B200_TRY(require_device());
    return wavernn_run_rows_impl(*shape, *params, *cond, reinterpret_cast<const long long*>(row_t), row_n, active_rows, nsteps, uniforms, out,
                                 workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_wavernn_reset_rows(const b200tts_wavernn_shape* shape, void* workspace, size_t workspace_bytes, const int32_t* rows, int count,
                               void* stream) {
    B200_REQUIRE(shape, "wavernn_reset_rows: null argument");
    B200_TRY(wavernn_check(*shape, workspace, workspace_bytes));
    B200_TRY(wavernn_reset_rows_check(*shape, rows, count));
    B200_TRY(require_device());
    return wavernn_reset_rows_impl(*shape, workspace, workspace_bytes, rows, count, (cudaStream_t)stream);
}
int b200tts_wavernn_window_rows(const b200tts_wavernn_window_row* rows, int active_rows, int nsteps, const float* mel, const float* fir,
                                const float* aux, float* feat, void* stream) {
    B200_REQUIRE(mel && fir && feat, "wavernn_window_rows: null argument");
    B200_TRY(wavernn_window_rows_check(rows, active_rows, nsteps));
    B200_REQUIRE(aux || rows[0].w.aux_dims == 0, "wavernn_window_rows: null aux");
    B200_TRY(require_device());
    return wavernn_window_rows_impl(rows, active_rows, nsteps, mel, fir, aux, feat, (cudaStream_t)stream);
}
int b200tts_wavernn_upsample_segments(int C, int nseg, const int32_t* lens, int scale, const float* fir, const float* in, float* out,
                                      void* stream) {
    B200_REQUIRE(fir && in && out, "wavernn_upsample_segments: null argument");
    B200_TRY(wavernn_upsample_segments_check(C, nseg, lens, scale));
    B200_TRY(require_device());
    return wavernn_upsample_segments_impl(C, nseg, lens, scale, fir, in, out, (cudaStream_t)stream);
}
int b200tts_wavernn_aborted(const b200tts_wavernn_shape* shape, const void* workspace, size_t workspace_bytes, int* aborted, void* stream) {
    B200_REQUIRE(shape && aborted, "wavernn_aborted: null argument");
    B200_TRY(require_device());
    return wavernn_aborted_impl(*shape, workspace, workspace_bytes, aborted, (cudaStream_t)stream);
}
int b200tts_wavernn_deemphasis(int rows, int len, int mu, float a, float* y, void* stream) {
    B200_REQUIRE(y, "wavernn_deemphasis: null argument");
    B200_TRY(wavernn_deemphasis_check(rows, len, mu, a));
    B200_TRY(require_device());
    return wavernn_deemphasis_impl(rows, len, mu, a, y, (cudaStream_t)stream);
}
int b200tts_wavernn_unfold(int B, int hop, int target, int overlap, int mu, const int32_t* frames, const int32_t* row_off, const int64_t* wave_off,
                           long long total, const float* y, float* wave, void* stream) {
    B200_REQUIRE(frames && row_off && wave_off && y && wave, "wavernn_unfold: null argument");
    B200_TRY(wavernn_unfold_check(B, hop, target, overlap, mu));
    B200_TRY(require_device());
    return wavernn_unfold_impl(B, hop, target, overlap, mu, frames, row_off, reinterpret_cast<const long long*>(wave_off), total, y, wave,
                               (cudaStream_t)stream);
}
int b200tts_wavernn_unfold_streams(int nstreams, int hop, int target, int overlap, int mu, const b200tts_wavernn_unfold_stream* streams,
                                   const int64_t* base, const int32_t* period, int nsrc, long long total, const float* y, float* wave,
                                   void* stream) {
    B200_REQUIRE(base && period && y && wave, "wavernn_unfold_streams: null argument");
    B200_TRY(wavernn_unfold_streams_check(nstreams, hop, target, overlap, mu, streams, nsrc, total));
    B200_TRY(require_device());
    return wavernn_unfold_streams_impl(nstreams, hop, target, overlap, mu, streams, reinterpret_cast<const long long*>(base), period, nsrc,
                                       total, y, wave, (cudaStream_t)stream);
}

size_t b200tts_gru_seq_saved_bytes(const b200tts_gru_seq_shape* shape) {
    if (!shape) { set_last_error("gru_seq_saved_bytes: null shape"); return 0; }
    return gru_seq_saved_bytes(*shape);
}
size_t b200tts_gru_seq_workspace_bytes(const b200tts_gru_seq_shape* shape) {
    if (!shape) { set_last_error("gru_seq_workspace_bytes: null shape"); return 0; }
    return gru_seq_workspace_bytes(*shape);
}
int b200tts_gru_seq_forward(const b200tts_gru_seq_shape* shape, const float* gi, const float* w_hh, const float* b_hh, float* h, void* saved,
                            void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && gi && w_hh && b_hh && h && saved, "gru_seq_forward: null argument");
    B200_TRY(gru_seq_check(*shape, workspace, workspace_bytes));
    B200_TRY(require_device());
    return gru_seq_forward_impl(*shape, gi, w_hh, b_hh, h, saved, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_gru_seq_backward(const b200tts_gru_seq_shape* shape, const float* w_hh, const float* h, const void* saved, const float* dh_ext,
                             float* dgi, float* dgh, float* dh_dbg, void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(shape && w_hh && h && saved && dh_ext && dgi && dgh, "gru_seq_backward: null argument");
    B200_TRY(gru_seq_check(*shape, workspace, workspace_bytes));
    B200_TRY(require_device());
    return gru_seq_backward_impl(*shape, w_hh, h, saved, dh_ext, dgi, dgh, dh_dbg, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_gru_seq_aborted(const b200tts_gru_seq_shape* shape, const void* workspace, size_t workspace_bytes, int* aborted, void* stream) {
    B200_REQUIRE(shape && aborted, "gru_seq_aborted: null argument");
    B200_TRY(require_device());
    return gru_seq_aborted_impl(*shape, workspace, workspace_bytes, aborted, (cudaStream_t)stream);
}
int b200tts_gru_seq_abort_flag_copy(const b200tts_gru_seq_shape* shape, const void* workspace, size_t workspace_bytes, int* dst, void* stream) {
    B200_REQUIRE(shape && dst, "gru_seq_abort_flag_copy: null argument");
    B200_TRY(gru_seq_check(*shape, const_cast<void*>(workspace), workspace_bytes));
    B200_TRY(require_device());
    return gru_seq_abort_flag_copy_impl(*shape, workspace, workspace_bytes, dst, (cudaStream_t)stream);
}
int b200tts_wavernn_cut_windows(int mode, int bits, int B, int feat, int seq_len, int pad, int hop, const float* mels, long long total_frames,
                                const int64_t* frame_start, const uint16_t* labels, const int64_t* sample_start, const int32_t* table, float* x,
                                void* y, float* m, void* stream) {
    B200_REQUIRE(mels && frame_start && labels && sample_start && table && x && y && m, "wavernn_cut_windows: null argument");
    B200_TRY(wavernn_cut_windows_check(mode, bits, B, feat, seq_len, pad, hop, total_frames));
    B200_TRY(require_device());
    return wavernn_cut_windows_impl(mode, bits, B, feat, seq_len, pad, hop, mels, total_frames, reinterpret_cast<const long long*>(frame_start),
                                    labels, reinterpret_cast<const long long*>(sample_start), table, x, y, m, (cudaStream_t)stream);
}
size_t b200tts_wavernn_upsample_layer_backward_workspace_bytes(int C, int len, int scale) {
    return wavernn_upsample_layer_backward_workspace_bytes(C, len, scale);
}
int b200tts_wavernn_upsample_layer_backward(int C, int len, int scale, const float* fir, const float* in, const float* dout, float* din,
                                            float* dfir, void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(fir && dout && (din || dfir), "wavernn_upsample_layer_backward: null argument");
    B200_TRY(wavernn_upsample_layer_check(C, len, scale));
    B200_TRY(require_device());
    return wavernn_upsample_layer_backward_impl(C, len, scale, fir, in, dout, din, dfir, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_wavernn_stretch_backward(int B, int F, int C, int hop, const float* dup, float* daux, void* stream) {
    B200_REQUIRE(dup && daux, "wavernn_stretch_backward: null argument");
    B200_TRY(wavernn_stretch_backward_check(B, F, C, hop));
    B200_TRY(require_device());
    return wavernn_stretch_backward_impl(B, F, C, hop, dup, daux, (cudaStream_t)stream);
}
size_t b200tts_wavernn_loss_workspace_bytes(long long N) { return wavernn_loss_workspace_bytes(N); }
size_t b200tts_column_sum_workspace_bytes(int cols) { return column_sum_workspace_bytes(cols); }
int b200tts_column_sum(long long rows, int cols, const float* x, float* out, void* workspace, size_t workspace_bytes, void* stream) {
    B200_REQUIRE(x && out, "column_sum: null argument");
    B200_TRY(column_sum_check(rows, cols));
    B200_TRY(require_device());
    return column_sum_impl(rows, cols, x, out, workspace, workspace_bytes, (cudaStream_t)stream);
}
int b200tts_wavernn_loss(int mode, long long N, int n_out, const float* logits, const void* target, float* loss, float* dlogits, void* workspace,
                         size_t workspace_bytes, void* stream) {
    B200_REQUIRE(logits && target && loss && dlogits, "wavernn_loss: null argument");
    B200_TRY(wavernn_loss_check(mode, N, n_out));
    B200_TRY(require_device());
    return wavernn_loss_impl(mode, N, n_out, logits, target, loss, dlogits, workspace, workspace_bytes, (cudaStream_t)stream);
}

}  // extern "C"
