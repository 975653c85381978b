/*
 * b200tts -- C ABI of the Hopper-native Tacotron-2 training hot path (sm_90a only; the b200tts prefix is historical).
 *
 * The reference (Tomiinek/Multilingual_Text_to_Speech) has no FFI / plugin layer: its boundary for this
 * path is the Python nn.Module surface (SURVEY.md section 8b).  This header is the boundary a native
 * binding would use instead; every entry point names the reference code it replaces.  The Python
 * host package (multilingual_text_to_speech_b200) binds it with ctypes and re-exposes the
 * reference's module classes on top.
 *
 * Conventions
 *   - plain pointers + sizes only; all tensors are dense row-major fp32 DEVICE pointers unless
 *     marked [host]; integer ids / lengths are int32; dropout keep-masks are uint8 (1 = keep).
 *   - the library never allocates: outputs and workspaces are caller-owned, sizes come from the
 *     *_workspace_bytes() queries (256-byte aligned base pointers expected).
 *   - every call enqueues work on `stream` (a cudaStream_t passed as void*) and returns
 *     immediately; 0 = ok, negative = error, message via b200tts_last_error().
 *   - there is NO CPU fallback: every entry point that needs the device fails with B200TTS_ERR_CUDA when
 *     no CUDA device is present and with B200TTS_ERR_UNSUPPORTED when it is not an sm_90 (H100) device.
 */
#ifndef B200TTS_H_
#define B200TTS_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200TTS_OK 0
#define B200TTS_ERR_INVALID (-1)
#define B200TTS_ERR_CUDA (-2)
#define B200TTS_ERR_UNSUPPORTED (-3)
#define B200TTS_ERR_WORKSPACE (-4)

#define B200TTS_CELL_DROPOUT 0 /* DropoutLSTMCell  modules/layers.py:37-47 */
#define B200TTS_CELL_ZONEOUT 1 /* ZoneoutLSTMCell  modules/layers.py:18-34 */

#define B200TTS_ATT_LOCATION 0 /* LocationSensitiveAttention  modules/attention.py:48-86 (hp.attention_type "location_sensitive") */
#define B200TTS_ATT_FORWARD 1  /* ForwardAttention            modules/attention.py:89-124 (hp.attention_type "forward") */

/* ---- library ---------------------------------------------------------------------------- */
const char* b200tts_last_error(void);
int b200tts_version(void);
/* Number of kernels this library has launched since load (bench.py's gpu_launches claim). */
unsigned long long b200tts_launch_count(void);

/* Live kernel timing for bench.py's per-kernel roofline: while enabled, the library brackets its dominant kernels (the four persistent
 * decoder loops, the attention post pass, the wgmma GEMM) with CUDA events on the launching stream.  enable != 0 starts a fresh
 * collection, 0 stops and clears.  After a device synchronize, kernel_timing_read(index, ...) returns the index-th distinct kernel
 * name with the summed duration and the number of launches; it returns 1 past the end of the list.                           */
int b200tts_kernel_timing(int enable);
int b200tts_kernel_timing_read(int index, char* name, int name_capacity, float* total_ms, int* count);

/* Arithmetic mode of every contraction in the library.  FP32: exact fp32 FFMA kernels (parity gate rtol 1e-3 /
 * atol 1e-4 against the reference).  BF16: operands rounded to bf16, fp32 accumulation on the tensor cores, fp32
 * master weights / states / outputs (BASELINE.json configs[1] "bf16 fwd / fp32 master"; gate: mel L1 < 1e-3).     */
#define B200TTS_PRECISION_FP32 0
#define B200TTS_PRECISION_BF16 1
int b200tts_set_precision(int mode);
int b200tts_get_precision(void);
/* Caller-owned device scratch (1024-byte aligned) for the bf16 operand packing of the wgmma GEMM path; without it (or when a
 * problem does not fit) the bf16 mode uses the mma.sync kernel.  ~1.5 GB covers the BASELINE shapes.  NULL releases it. */
int b200tts_set_scratch(void* ptr, size_t bytes);
/* Debug / A-B switch: 0 forces the mma.sync bf16 GEMM even when the wgmma path is applicable. */
int b200tts_set_tensor_core_gemm(int enabled);

/* ---- generic dense contraction (the time-batched GEMMs of the path) ----------------------- */
/* C = alpha * op(A) . op(B) + beta * C + bias[n];  op(A)(m,k) = transA ? A[k*lda+m] : A[m*lda+k],
 * op(B)(k,n) = transB ? B[n*ldb+k] : B[k*ldb+n].  Replaces the torch.nn.Linear / cuBLAS call sites
 * K8, K9, K15 of SURVEY.md section 2.3.  `workspace` (floats) is needed for splitk > 1.        */
int b200tts_gemm_f32(int transA, int transB, int M, int N, int K, float alpha, const float* A, int lda,
                     const float* B, int ldb, float beta, float* C, int ldc, const float* bias, int batch,
                     long long strideA, long long strideB, long long strideC, int splitk, float* workspace,
                     void* stream);

/* Debug: the library's whole GEMM descriptor (GemmDesc in csrc/common.cuh: the same fields in the same order, the same meaning),
 * so that tests can drive every feature of the dense contraction directly: batch strides, a_batch_mod, explicit split-K with
 * keep_partials, bf16 operands read in place (A16 / B16) and the two-level K (kin, kosA, kosB). */
typedef struct {
    const float* A;
    const float* B;
    float* C;
    const float* bias;
    int M, N, K;
    int lda, ldb, ldc;
    int transA, transB;
    float alpha, beta;
    int batch;
    long long strideA, strideB, strideC;
    int a_batch_mod;
    int splitk;
    float* partial;
    int keep_partials;
    const void* A16;
    int lda16;
    const void* B16;
    int ldb16;
    int kin;
    long long kosA, kosB;
} b200tts_gemm_desc;
/* route 0: the precision-mode dispatch (fp32 SIMT kernel, or the bf16 kernels: wgmma when it takes the shape, else mma.sync); the
 * descriptor's splitk / partial / keep_partials are used as given.  route 1: the auto-split dispatch, which picks the split-K factor
 * itself within `partial` (partial_elems floats; NULL = no split).  Returns a B200TTS_* status. */
int b200tts_debug_gemm(const b200tts_gemm_desc* desc, int route, float* partial, size_t partial_elems, void* stream);
/* Debug: open (1) or close (0) a pack-cache scope of the wgmma GEMM: inside it, bf16 operand packs are kept in the scratch and
 * reused by later products that read the same source view (the source buffers must not change while it is open). */
int b200tts_debug_gemm_pack_cache(int open);

/* ---- decoder: Decoder._decode, modules/tacotron2.py:148-209 -------------------------------- */
typedef struct {
    int B, L, T;            /* batch, padded text length, mel frames */
    int M, D, P, A, C, K, N; /* memory dim, decoder dim, prenet dim, attention dim, location channels,
                                location kernel size, mel channels */
    int cell_kind;          /* B200TTS_CELL_* */
    int training;           /* nn.Module.training of the cells (prenet dropout is always on) */
    float rate_h, rate_c;   /* dropout_hidden | (zoneout_hidden, zoneout_cell) */
    float prenet_rate;      /* hp.dropout used by the prenet */
    int att_kind;           /* B200TTS_ATT_*; 0 (location-sensitive) in a zero-initialised shape.  B200TTS_ATT_FORWARD: C and K
                               are ignored, params.attn_location / attn_loc_features must be NULL, the cumulative-weight rows of
                               the workspace (and b200tts_decoder_state.cum_weights) hold the forward variable alpha, and every
                               recurrence runs on the per-step kernel chains in both precision modes (b200tts_decoder_path = 0) */
    int att_extent;         /* forward attention only (location-sensitive attention ignores it).  0 in a zero-initialised shape: the
                               transition softmax, the 1e-6 floor, the normalisation and the context run over all L positions, padding
                               included (the reference's training semantics).  1: over each utterance's own text length; weights at
                               l >= length are 0, so a padded batch decodes every utterance as it decodes alone.  Forward and chunk
                               entry points only: b200tts_decoder_backward rejects 1. */
    int R;                  /* frames per decoder step (reduction factor, hp.outputs_per_step); 0 in a zero-initialised shape means 1.
                               T keeps counting target frames; the decode runs S = ceil(T / R) steps, and step i is fed frame i*R - 1
                               (zeros at step 0).  Arrays with S rows (one per step): the keep masks, `teacher`, `alignments` /
                               `d_alignments` and every per-step row of both workspaces.  Arrays with T frames: target, spectrogram,
                               stop and their gradients; frames of the last step past T are dropped (zero gradient).  The parameters
                               predict R frames per step: frame_w [R*N, D+M], frame_b [R*N], stop_w [R, D+M], stop_b [R], row block j
                               (rows j*N .. j*N+N-1 of frame_w, row j of stop_w) = frame j of the step.  Negative R is rejected. */
    int att_window_back, att_window_ahead;  /* windowed synthesis, location-sensitive attention and b200tts_decoder_forward_chunk only;
                               ahead = 0 (a zero-initialised shape) is off.  Otherwise (back >= 0, ahead >= 1) each step of utterance b
                               gives energies only to positions [c - back, c + ahead] within [0, length_b), where c is
                               b200tts_decoder_state.attended[b]; the softmax and the context run over those positions, every other
                               weight is exactly 0, and after the step c becomes the lowest position of the row's largest weight.
                               b200tts_decoder_forward and _backward, and forward attention, reject a window. */
} b200tts_decoder_shape;

/* Parameter block in the reference's own layouts ([out, in] Linear weights; names = state_dict keys). */
typedef struct {
    float* prenet_w0;   /* _prenet._layers.0.weight [P, N] */
    float* prenet_b0;   /* [P] */
    float* prenet_w1;   /* _prenet._layers.1.weight [P, P] */
    float* prenet_b1;   /* [P] */
    float* att_w_ih;    /* _decoder._attention_lstm.weight_ih [4D, P+M]  (gate order i,f,g,o) */
    float* att_w_hh;    /* [4D, D] */
    float* att_b_ih;    /* [4D] */
    float* att_b_hh;    /* [4D] */
    float* gen_w_ih;    /* _decoder._generator_lstm.weight_ih [4D, D+M] */
    float* gen_w_hh;    /* [4D, D] */
    float* gen_b_ih;    /* [4D] */
    float* gen_b_hh;    /* [4D] */
    float* attn_query;  /* _attention._query.weight [A, D] */
    float* attn_memory; /* _attention._memory.weight [A, M] */
    float* attn_location;     /* _attention._location.weight [A, C] */
    float* attn_loc_features; /* _attention._loc_features.weight [C, 1, K] */
    float* attn_bias;   /* _attention._bias [1, A] */
    float* attn_energy; /* _attention._energy.weight [1, A] */
    float* frame_w;     /* _decoder._frame_prediction.weight [N, D+M] */
    float* frame_b;     /* [N] */
    float* stop_w;      /* _decoder._stop_prediction.weight [1, D+M] */
    float* stop_b;      /* [1] */
} b200tts_decoder_params;

typedef struct {
    const float* memory;          /* [B, L, M] encoder output ++ speaker/language embeddings */
    const int32_t* text_lengths;  /* [B] */
    const float* target;          /* [B, N, T] ground-truth mel frames */
    const uint8_t* teacher;       /* [host] [S] 1 = ground truth fed at step i (tacotron2.py:171,181); NULL = all 1.  0 = free-running:
                                     step i is fed the last frame predicted at step i-1 (zeros at step 0), and the backward
                                     differentiates through that frame (no detach, as in the reference) */
    /* keep masks, NULL = no dropout at that site.  Time-major: row i belongs to decoder step i (S = ceil(T / R) rows). */
    const uint8_t* mask_prenet0;  /* [S, B, P] */
    const uint8_t* mask_prenet1;  /* [S, B, P] */
    const uint8_t* mask_att_h;    /* [S, B, D]; 8-byte aligned on the persistent attention reverse loop */
    const uint8_t* mask_att_c;    /* [S, B, D] zoneout only; 8-byte aligned there too */
    const uint8_t* mask_gen_h;    /* [S, B, D] */
    const uint8_t* mask_gen_c;    /* [S, B, D] zoneout only */
    const uint8_t* mask_step_prenet0; /* [S, B, P] prenet masks of free-running steps */
    const uint8_t* mask_step_prenet1; /* [S, B, P] */
    /* forced synthesis, b200tts_decoder_forward_chunk only; forced_count = 0 (a zero-initialised struct) is off.  Otherwise the
       forced_count (F, 1 <= F <= B) distinct rows forced_rows[0 .. F) (device int32, each in [0, B)) take each step's attention weights
       from forced_alignment (device [S, F, L], time-major: row [i, k] is step i of utterance forced_rows[k]) instead of computing them.
       For such an utterance b at step i: the alignment row is the supplied row with exact zeros at l >= length_b; location-sensitive
       attention carries cum_weights + that row, forward attention carries that row as alpha; the context is the sum over l < length_b
       of w[l] * memory[b, l, :], in the order the computed step sums it (from position 0, or with a window from the row's first
       non-zero weight).  No query, location feature, energy or softmax is computed for the row.  When F < B the computed step runs over
       every row first (a window applies to it) and the forced step then overwrites the forced rows; when F = B only the forced step
       runs.  b200tts_decoder_forward and _backward reject forced rows. */
    const int32_t* forced_rows;
    int forced_count;
    const float* forced_alignment;
} b200tts_decoder_inputs;

typedef struct {
    float* spectrogram; /* [B, T, N] */
    float* stop;        /* [B, T]   logits */
    float* alignments;  /* [B, S, L]  one row per decoder step */
} b200tts_decoder_outputs;

/* Bytes of the forward workspace; it also carries everything the backward pass re-reads. */
size_t b200tts_decoder_workspace_bytes(const b200tts_decoder_shape* shape);
size_t b200tts_decoder_bwd_workspace_bytes(const b200tts_decoder_shape* shape);
/* Which kernels a bf16-mode training step with every decoder step teacher-forced runs on for this shape (pure host arithmetic, no
 * device needed; a decode with a free-running step runs the per-step kernel chains, forward and backward): bit 0 = persistent
 * forward loops, bit 1 = their TMA + wgmma variant, bit 2 = persistent generator reverse loop, bit 3 = its wgmma
 * variant, bit 4 = persistent attention reverse loop, bit 5 = its wgmma product.  0 = the per-step kernel chains.
 * Every persistent loop is a TMA + wgmma kernel, so each variant bit (1, 3, 5) is set exactly when its loop bit (0, 2, 4)
 * is; a pass whose loop bit is clear runs the per-step kernel chains.  Forward attention (att_kind = B200TTS_ATT_FORWARD) always gives 0.
 * (The reference has no such limit anywhere: modules/attention.py:67-74 takes any length.) */
int b200tts_decoder_path(const b200tts_decoder_shape* shape);
/* Debug: byte offset, inside the decoder forward workspace, of the per-CTA phase cycle counters the persistent
 * kernels leave behind ([2][132][8] int64, one row per SM: attention loop, generator loop). */
size_t b200tts_debug_persist_profile_offset(const b200tts_decoder_shape* shape);
/* Same for the backward workspace: which = 0 generator loop, 1 attention loop ([132][8] int64 each). */
size_t b200tts_debug_persist_bwd_profile_offset(const b200tts_decoder_shape* shape, int which);
/* Debug: where a decoder call keeps its per-step state, so that tests can check every step of a decode.  Fills out[0 .. n) with
 * byte offsets, in this order:
 *   forward workspace:  ai, ca, hg, cg, ga, gg, q, cum, memT, fs, p1, aib, hgb
 *   backward workspace: dfs, dhgd, dctxs, dgg, dhas, dga, dq, dctxt, dmemT, dggb, dgab
 *   row strides (in elements) of aib and hgb: Kp_att, Kp_gen
 *   forward workspace:  xtm (prenet input, row i = the frame fed to step i), p0 (first prenet layer)
 *   backward workspace: dp1, dp0 (prenet layer gradients after the relu / dropout backward)
 * Every per-step view has one row per decoder step (S = ceil(T / R)); fs and dfs are R (N + 1) wide.
 * Returns the number of values written (30 when n >= 30), 0 for a rejected shape. */
int b200tts_debug_decoder_views(const b200tts_decoder_shape* shape, size_t* out, int n);
/* Debug (pure host arithmetic, no device needed): the geometry the persistent loops would run this shape with.  Fills out[0 .. n) in
 * this order:
 *   b200tts_decoder_path of the shape;
 *   forward loops: grid (CTAs), NBH (batch halves of 32 utterances), slot_kb (TMA ring slot of the attention loop, in 64-column
 *     k-blocks), ch_h and n_h (k-blocks per TMA load and loads of the h part), ch_c and n_c (same for the context part), alias (1: the
 *     accumulator staging shares the ring slot), use_btab (1: the context product's B fragments come from a shared table), the generator
 *     loop's slot and ch_h;
 *   attention reverse loop: UN (outputs per n-block), grid.
 * The geometry is reported whatever the path; only the loops the path bits select run with it.  Returns the number of values written
 * (14 when n >= 14), 0 for a rejected shape. */
int b200tts_debug_decoder_geometry(const b200tts_decoder_shape* shape, int* out, int n);

int b200tts_decoder_forward(const b200tts_decoder_shape* shape, const b200tts_decoder_params* params,
                            const b200tts_decoder_inputs* in, const b200tts_decoder_outputs* out, void* workspace,
                            size_t workspace_bytes, void* stream);

/* Decoder state carried between chunks of one decode (all device pointers, fp32 but `attended`; every field but `attended` required): lets a caller decode in
 * chunks of T frames and stop early, as the reference's inference loop does (Decoder.inference, tacotron2.py:201-207,216-219). */
typedef struct {
    float* att_h; float* att_c; /* [B, D] attention-LSTM state */
    float* gen_h; float* gen_c; /* [B, D] generator-LSTM state */
    float* context;             /* [B, M] last attention context */
    float* cum_weights;         /* [B, L] cumulative attention weights (forward attention: the last alignment = alpha) */
    float* frame;               /* [B, N] last predicted frame, the last of the last step's R (input of the next free-running step) */
    int32_t* attended;          /* [B] window centre: the first argmax of the last alignment row, 0 before step 0.  Read and written only
                                   with a window (shape->att_window_ahead >= 1); may be NULL without one */
} b200tts_decoder_state;

/* b200tts_decoder_forward on a chunk of T frames: `first` != 0 starts from the zero state (tacotron2.py:164-168), otherwise from
 * `state`; on return `state` holds the state after the chunk's last step.  Uses the per-step kernels (any precision mode).  A chunk
 * holds whole steps: T % R != 0 is rejected. */
int b200tts_decoder_forward_chunk(const b200tts_decoder_shape* shape, const b200tts_decoder_params* params,
                                  const b200tts_decoder_inputs* in, const b200tts_decoder_outputs* out, b200tts_decoder_state* state,
                                  int first, void* workspace, size_t workspace_bytes, void* stream);

/* Rows of a b200tts_decoder_state listed per launch of b200tts_decoder_state_reset_rows (more are split over several launches). */
#define B200TTS_DECODER_RESET_MAX_ROWS 64
/* Writes the initial state of a decode into the `count` listed rows (host int32, each in [0, shape->B)) of `state`, whose buffers hold
 * shape->B rows of width L, M, D and N: zeros, and for forward attention (shape->att_kind) the one-hot alpha_0 in cum_weights.  A chunk
 * with `first` = 0 then continues such a row exactly as a chunk with `first` != 0 starts a fresh decode: both write the state through the
 * same kernel.  The other rows are untouched, so texts can join a running decode.  Only B, L, M, D, N and att_kind of `shape` are read.
 * A non-NULL state->attended gets 0 in the listed rows. */
int b200tts_decoder_state_reset_rows(const b200tts_decoder_shape* shape, b200tts_decoder_state* state, const int32_t* rows, int count,
                                     void* stream);

typedef struct {
    const float* d_spectrogram; /* [B, T, N] or NULL */
    const float* d_stop;        /* [B, T]    or NULL */
    const float* d_alignments;  /* [B, S, L] or NULL */
} b200tts_decoder_output_grads;

/* Backward of the decode (autograd replay of tacotron2.py:148-209, train.py:83), free-running steps included: their gradient
 * flows back through the fed-back frame into the previous step's frame projection, generator LSTM and attention.
 * `fwd_workspace` is the buffer the matching forward call filled and `fwd_out` its outputs (the
 * alignments are re-read).  Parameter gradients are ACCUMULATED into `d_params` (+=, like autograd
 * .grad); `d_memory` [B, L, M] is overwritten (may be NULL). */
int b200tts_decoder_backward(const b200tts_decoder_shape* shape, const b200tts_decoder_params* params,
                             const b200tts_decoder_inputs* in, const b200tts_decoder_outputs* fwd_out,
                             const b200tts_decoder_output_grads* dout, const void* fwd_workspace, void* bwd_workspace,
                             size_t bwd_workspace_bytes, const b200tts_decoder_params* d_params, float* d_memory,
                             void* stream);

/* ---- single attention step: LocationSensitiveAttention.forward, modules/attention.py:39-45,67-86 ---- */
/* query [B, D]; memory [B, L, M]; memory_transform [B, L, A] (= AttentionBase.reset, attention.py:25);
 * cum_weights [B, L] is read and updated in place; context [B, M], weights [B, L] written.
 * workspace floats: b200tts_attention_step_workspace_elems(B, L, A).                           */
size_t b200tts_attention_step_workspace_elems(int B, int L, int A);
int b200tts_attention_step(int B, int L, int M, int D, int A, int C, int K, const float* query, const float* memory,
                           const float* memory_transform, const int32_t* text_lengths, const float* w_query,
                           const float* w_location, const float* w_loc_features, const float* bias,
                           const float* w_energy, float* cum_weights, float* context, float* weights,
                           float* workspace, void* stream);


/* Backward of one attention step (autograd of attention.py:39-45,67-86 for the module-level API; the training path runs the fused
 * decoder backward instead).  q [B, A] = query . Wq^T as the forward computed it (the head of its workspace); cum_prev [B, L] the
 * cumulative weights the step CONSUMED; weights [B, L] its output.  d_cum [B, L]: in = gradient of the UPDATED cumulative weights,
 * out = gradient of cum_prev.  d_q [B, A] out (the caller forms d query = d_q . Wq, d Wq += d_q^T . query, d bias += sum_b d_q);
 * d_memory_transform [B, L, A], d_w_location [A, C], d_w_loc_features [C, K], d_w_energy [A] are ACCUMULATED (+=).
 * workspace floats: b200tts_attention_step_backward_workspace_elems(B, M, A, C, K).                                              */
size_t b200tts_attention_step_backward_workspace_elems(int B, int M, int A, int C, int K);
int b200tts_attention_step_backward(int B, int L, int M, int A, int C, int K, const float* q, const float* memory,
                                    const float* memory_transform, const int32_t* text_lengths, const float* w_location,
                                    const float* w_loc_features, const float* bias, const float* w_energy, const float* cum_prev,
                                    const float* weights, const float* d_context, const float* d_weights, float* d_cum, float* d_q,
                                    float* d_memory_transform, float* d_w_location, float* d_w_loc_features, float* d_w_energy,
                                    float* workspace, void* stream);
/* The per-chunk position count LC the attention backward kernel runs (L, M, A, C, K) with: it processes each utterance's positions in
 * chunks of LC, the largest multiple of 4 (at most L rounded up to 4) whose shared memory fits in 220 KB.  0 for dims the backward
 * rejects, including an L for which not even 4-row chunks fit in the 227 KB limit.  Host only. */
int b200tts_debug_attention_backward_chunk(int L, int M, int A, int C, int K);

/* ---- single forward-attention step: ForwardAttention.forward, modules/attention.py:23-45,89-124 ----
 * e = v . tanh(query . Wq^T + memory_transform + bias) over ALL L positions; s = softmax(e) (padding included);
 * a[l] = (alpha[l] + alpha[l-1]) * s[l]; a[l] = 0 for l >= text_lengths; w = clamp(a, 1e-6) / sum; context = w . memory.
 * alpha [B, L] is read and replaced by w in place (ForwardAttention.reset sets alpha[:, 0] = 1); context [B, M], weights [B, L]
 * written.  workspace floats: b200tts_forward_attention_step_workspace_elems(B, L, A); its head holds q = query . Wq^T [B, A]. */
size_t b200tts_forward_attention_step_workspace_elems(int B, int L, int A);
int b200tts_forward_attention_step(int B, int L, int M, int D, int A, const float* query, const float* memory,
                                   const float* memory_transform, const int32_t* text_lengths, const float* w_query,
                                   const float* bias, const float* w_energy, float* alpha, float* context, float* weights,
                                   float* workspace, void* stream);
/* Backward of one forward-attention step.  q [B, A] as the forward left it; alpha_prev [B, L] the alpha the step CONSUMED; weights
 * [B, L] its output.  d_alpha [B, L]: in = gradient of the new alpha (= weights), out = gradient of alpha_prev.  d_q [B, A] out (the
 * caller forms d query, d Wq and d bias = sum_b d_q); d_memory_transform [B, L, A] and d_w_energy [A] are ACCUMULATED (+=), the latter
 * from per-utterance partials reduced over the batch in a fixed order.
 * workspace floats: b200tts_forward_attention_step_backward_workspace_elems(B, M, A).                                             */
size_t b200tts_forward_attention_step_backward_workspace_elems(int B, int M, int A);
int b200tts_forward_attention_step_backward(int B, int L, int M, int A, const float* q, const float* memory, const float* memory_transform,
                                            const int32_t* text_lengths, const float* bias, const float* w_energy, const float* alpha_prev,
                                            const float* weights, const float* d_context, const float* d_weights, float* d_alpha,
                                            float* d_q, float* d_memory_transform, float* d_w_energy, float* workspace, void* stream);

/* ---- convolution block: ConvBlock / HighwayConvBlock / ConvBlockGenerated / HighwayConvBlockGenerated ----
 * modules/layers.py:50-178.  x [NB, G*Cin, L] -> pad((k-1)*dil/2) -> grouped Conv1d(no bias) -> BatchNorm1d
 * (batch statistics over (NB, L) incl. padded positions when training) -> activation -> Dropout ->
 * optional highway gate  out = h2 * sigmoid(h1) + x * (1 - sigmoid(h1)).
 * weight [G*Cout, Cin, k] is either an nn.Conv1d weight or the output of b200tts_generator_forward.
 * gamma / beta: element (g, o) at ptr[g*affine_gstride + o] (plain BN: stride Cout; generated BN:
 * ptr = affine, affine + Cout with stride 2*Cout, modules/generated.py:83-84).                       */
typedef struct {
    int NB, G, Cin, Cout, L; /* Cout = per-group conv output channels (2*Cin for highway blocks) */
    int k, dilation;
    int activation;          /* 0 identity, 1 relu, 2 tanh */
    int highway;
    int training;
    float eps, momentum, dropout;
    int stage;               /* 0: whole block.  1: convolution only = Conv1dGenerated.forward / nn.Conv1d (modules/generated.py:34-42;
                                gamma / beta / keep ignored, out [NB, G*Cout, L]).  2: batch norm (+ activation, dropout) only, applied to
                                x [NB, G*Cout, L] = BatchNorm1dGenerated.forward (modules/generated.py:71-96; weight ignored, Cin == Cout) */
} b200tts_convblock_shape;

size_t b200tts_convblock_saved_bytes(const b200tts_convblock_shape* shape);
size_t b200tts_convblock_workspace_bytes(const b200tts_convblock_shape* shape);
/* running_mean / running_var [G*Cout] are updated in place when training (may be NULL then). keep: uint8
 * [NB, G*Cout, L] or NULL.  out [NB, G*Cf, L] with Cf = highway ? Cout/2 : Cout.
 * saved (fp32, n = NB*G*Cout*L, Ct = G*Cout, a64(m) = m rounded up to a multiple of 64): floats [0, n) hold the convolution
 * product before batch norm (stage 0; unused by stages 1 and 2), then mean [Ct] at a64(n) and invstd [Ct] at a64(n) + a64(Ct):
 * the batch statistics when training, running_mean and 1/sqrt(running_var + eps) in eval.                                       */
int b200tts_convblock_forward(const b200tts_convblock_shape* shape, const float* x, const float* weight,
                              const float* gamma, const float* beta, int affine_gstride, float* running_mean,
                              float* running_var, const uint8_t* keep, float* out, void* saved, void* workspace,
                              void* stream);
/* The same for a padded batch of utterances in eval mode, whole block (stage 0) only: lengths [NB] int32 (device); every output at a
 * position l >= lengths[n] of sample n is written as 0 by the fused epilogue.  Fed a zero-padded input, each sample's output then
 * equals running the block on that sample alone (conv1d pads with zeros); with every length == L it is bit-identical to
 * b200tts_convblock_forward.  Training or stage 1 / 2 is rejected.                                                                */
int b200tts_convblock_forward_masked(const b200tts_convblock_shape* shape, const int32_t* lengths, const float* x, const float* weight,
                                     const float* gamma, const float* beta, int affine_gstride, float* running_mean,
                                     float* running_var, const uint8_t* keep, float* out, void* saved, void* workspace,
                                     void* stream);
/* dx overwritten; dweight / dgamma / dbeta accumulated (+=).                                         */
int b200tts_convblock_backward(const b200tts_convblock_shape* shape, const float* x, const float* weight,
                               const float* gamma, const float* beta, int affine_gstride, const uint8_t* keep,
                               const void* saved, const float* dout, float* dx, float* dweight, float* dgamma,
                               float* dbeta, void* workspace, void* stream);
/* The same pair for a batch whose channel blocks hold different numbers of utterances (every stage, training and eval):
 * counts [G] int32 (device).  Rows nb < counts[g] of channel block g are occupied, rows nb >= counts[g] are vacant.
 * - Batch-norm statistics of block g run over its occupied rows only (n = counts[g] * L); the running statistics of a block
 *   with counts[g] == 0 are left unchanged, and its gamma / beta (and, through the zero dz, its weights) get exactly 0.
 * - Vacant rows of out (every stage), of the batch-norm input gradient and of dx are written as exact 0.  Vacant rows of x
 *   must be finite: the weight-gradient products add 0 * x for them.
 * - G and NB restate what the counts were derived for and must equal shape->G / shape->NB.  A device-side count outside
 *   [0, NB] is clamped into it (no row outside the tensor is ever addressed).
 * With every count == NB the results are bit-identical to b200tts_convblock_forward / b200tts_convblock_backward.      */
int b200tts_convblock_forward_counts(const b200tts_convblock_shape* shape, const int32_t* counts, int G, int NB, const float* x,
                                     const float* weight, const float* gamma, const float* beta, int affine_gstride,
                                     float* running_mean, float* running_var, const uint8_t* keep, float* out, void* saved,
                                     void* workspace, void* stream);
int b200tts_convblock_backward_counts(const b200tts_convblock_shape* shape, const int32_t* counts, int G, int NB, const float* x,
                                      const float* weight, const float* gamma, const float* beta, int affine_gstride,
                                      const uint8_t* keep, const void* saved, const float* dout, float* dx, float* dweight,
                                      float* dgamma, float* dbeta, void* workspace, void* stream);

/* ---- one LSTM cell step: ZoneoutLSTMCell.forward / DropoutLSTMCell.forward, modules/layers.py:26-34,44-47 ----
 * gates [B, 4D]: in = x . W_ih^T + b_ih + h . W_hh^T + b_hh (order i, f, g, o), out = the activated gates (saved for the backward);
 * h_prev / c_prev / h_out / c_out [B, D]; keep masks uint8 [B, D] or NULL (zoneout: both, dropout cell: mask_h only).            */
int b200tts_lstm_cell_forward(int B, int D, int cell_kind, int training, float rate_h, float rate_c, float* gates, const float* h_prev,
                              const float* c_prev, const uint8_t* mask_h, const uint8_t* mask_c, float* h_out, float* c_out, void* stream);
/* d_h [B, D] gradient of h_out; d_c [B, D] in: gradient of c_out, out: gradient of c_prev; d_h_prev [B, D] out: the DIRECT gradient of
 * h_prev (zoneout carry; zeros for the dropout cell; the part through the gates is d_gates . W_hh); d_gates [B, 4D] out (pre-activation). */
int b200tts_lstm_cell_backward(int B, int D, int cell_kind, int training, float rate_h, float rate_c, const float* gates, const float* c_prev,
                               const uint8_t* mask_h, const uint8_t* mask_c, const float* d_h, float* d_c, float* d_h_prev, float* d_gates,
                               void* stream);

/* ---- parameter generator: Conv1dGenerated / BatchNorm1dGenerated weight synthesis, modules/generated.py:38-39,81-82 ----
 * out[g, :] = (e[g] . Wb^T + bb) . Wk^T + bk;   e [G, gd], Wb [bn, gd], Wk [R, bn]; eb [G, bn] is saved. */
size_t b200tts_generator_workspace_bytes(int G, int bn);
int b200tts_generator_forward(int G, int gd, int bn, long long R, const float* e, const float* Wb, const float* bb,
                              const float* Wk, const float* bk, float* eb, float* out, void* stream);
/* all gradients accumulated (+=). */
int b200tts_generator_backward(int G, int gd, int bn, long long R, const float* e, const float* Wb, const float* Wk,
                               const float* eb, const float* dout, float* de, float* dWb, float* dbb, float* dWk,
                               float* dbk, void* workspace, void* stream);

/* ---- embeddings: nn.Embedding gather (tacotron2.py:237-239,363; :121-124,143-146) ---- */
/* out[t, 0:E] = table[ids[t], :] for ntok tokens, output row stride ldo (lets the caller write a column block). */
int b200tts_embedding_forward(float* out, int ldo, const float* table, const int32_t* ids, long long ntok, int E, void* stream);
/* dtable[v, :] += sum_{t: ids[t]==v} dout[t, 0:E]; rows equal to padding_idx (or -1 for none) are skipped. */
int b200tts_embedding_backward(float* dtable, int V, const float* dout, int ldo, const int32_t* ids, long long ntok, int E,
                               int padding_idx, void* stream);

/* ---- packed bidirectional LSTM of the vanilla encoder: modules/encoder.py:33,41-44 ---- */
typedef struct { int B, L, E, H; } b200tts_bilstm_shape;
typedef struct {
    float *w_ih, *w_hh, *b_ih, *b_hh;                                 /* _lstm.weight_ih_l0 [4H, E] ... */
    float *w_ih_reverse, *w_hh_reverse, *b_ih_reverse, *b_hh_reverse; /* _lstm.*_l0_reverse */
} b200tts_bilstm_params;
size_t b200tts_bilstm_saved_bytes(const b200tts_bilstm_shape* shape);
size_t b200tts_bilstm_workspace_bytes(const b200tts_bilstm_shape* shape);
/* x [B, L, E], lengths [B] -> out [B, L, 2H] (zeros at positions >= length). */
int b200tts_bilstm_forward(const b200tts_bilstm_shape* shape, const b200tts_bilstm_params* params, const float* x,
                           const int32_t* lengths, float* out, void* saved, void* workspace, void* stream);
int b200tts_bilstm_backward(const b200tts_bilstm_shape* shape, const b200tts_bilstm_params* params,
                            const int32_t* lengths, const void* saved, const float* dout, float* dx,
                            const b200tts_bilstm_params* d_params, void* workspace, void* stream);
/* Debug: where the bi-LSTM keeps its per-step state, so that tests can check every step of both directions (pure host arithmetic,
 * no device needed).  Fills out[0 .. n) in this order:
 *   saved (byte offsets):     xp [2][L][B][E], gates [2][L][B][4H], hs [2][L + 1][B][H], cs [2][L + 1][B][H], bsum [2][4H]
 *   workspace (byte offsets): dg [2][L][B][4H], dxp [2][L][B][E]
 *   split-K factors of the per-step chain's recurrent products (forward, backward), 1 if the persistent kernel runs the recurrence
 * Direction-major, in processing order (step j is position j forward, L-1-j reverse).  The persistent kernel reads
 * B200TTS_BILSTM_CHAIN as the forward and backward calls do.  Returns the number of values written (10 when n >= 10), 0 for a
 * rejected shape. */
int b200tts_debug_bilstm_layout(const b200tts_bilstm_shape* shape, size_t* out, int n);

/* ---- loss: TacotronLoss.forward, modules/tacotron2.py:439-485 (guided attention :439-457 in closed form) ----
 * pre / post / targets [B, N, T]; stop (logits, padded positions already filled as in tacotron2.py:380) / stop_target [B, T]; alignment
 * [B, S, L] with S = ceil(T / R); lengths int32 [B].  losses[4] (device) = { 2*MSE(pre), MSE(post), BCEWithLogits(pos_weight)/(N+2),
 * guided attention }.  The guided term runs on the step grid: utterance b has ceil(target_lengths[b] / R) steps, which take the place of
 * its frame count in the weight and the division (R = 1: the reference's formula).  The four mel buffers need no more than float
 * alignment: the forward reads them four floats at a time with 16-byte loads when all four are 16-byte aligned and with scalar loads
 * otherwise, in the same order and with the same arithmetic, so the result does not depend on their alignment.                     */
typedef struct {
    int B, N, T, L;
    int guided;            /* hp.guided_attention_loss and guided_att_steps > 0 */
    float guided_g;        /* current variance (TacotronLoss._g) */
    float stop_pos_weight; /* 100 in the reference (tacotron2.py:465) */
    int R;                 /* frames per decoder step of the alignment rows; 0 in a zero-initialised shape means 1 */
} b200tts_loss_shape;
size_t b200tts_loss_workspace_bytes(void);
int b200tts_tacotron_loss_forward(const b200tts_loss_shape* shape, const float* pre, const float* pre_target, const float* post,
                                  const float* post_target, const float* stop, const float* stop_target, const float* alignment,
                                  const int32_t* text_lengths, const int32_t* target_lengths, float* losses, void* workspace, void* stream);
/* grad_losses[4] (device): upstream gradient of each term.  Any of d_pre / d_post / d_stop / d_alignment may be NULL; all are overwritten. */
int b200tts_tacotron_loss_backward(const b200tts_loss_shape* shape, const float* pre, const float* pre_target, const float* post,
                                   const float* post_target, const float* stop, const float* stop_target, const int32_t* text_lengths,
                                   const int32_t* target_lengths, const float* grad_losses, float* d_pre, float* d_post, float* d_stop,
                                   float* d_alignment, void* stream);

/* ---- dropout-mask generation (counter-based RNG; replaces the Philox draws inside F.dropout) ---- */
int b200tts_fill_keep_mask(uint8_t* mask, size_t n, float drop_rate, uint64_t seed, uint64_t stream_id, void* stream);
/* Optional DEVICE-side epoch mixed into every mask key (NULL = off): a training step captured in a CUDA graph bakes the host seeds into
 * its kernel nodes, so the graph increments *epoch (a device uint64 the caller owns) once per replay and every replay draws new masks. */
int b200tts_set_mask_epoch(const uint64_t* device_epoch);
/* Per-row keep masks, time-major [steps, rows, width] (1 = keep), in one launch: element (i, r, p) is decision (step0[r] + i) * width + p
 * of the stream b200tts_fill_keep_mask draws for (seeds[r], stream_id).  So a row's masks over steps [0, S), however they are cut into
 * calls, are the rows of one b200tts_fill_keep_mask(n = S * width, seeds[r], stream_id) call.  seeds (uint64) and step0 (int64, >= 0)
 * are DEVICE arrays of `rows` entries.  The device epoch of b200tts_set_mask_epoch is NOT mixed in: the draws depend on the seed alone
 * (the equality above holds while no epoch is set). */
int b200tts_fill_keep_mask_rows(uint8_t* mask, int steps, int rows, int width, float drop_rate, const uint64_t* seeds, const int64_t* step0,
                                uint64_t stream_id, void* stream);
/* Per-row uniforms in [0, 1), [rows, nsteps, width] (the layout b200tts_wavernn_run_rows reads with width = uniforms per step), in one
 * launch: element (r, i, u) is draw (t0[r] + i) * width + u of the counter-based stream keyed by (seeds[r], stream_id): the top 24 bits
 * of splitmix64 over the key and the draw index, times 2^-24.  A row's draws do not depend on how its steps are split into calls.  seeds
 * (uint64) and t0 (int64, >= 0) are DEVICE arrays of `rows` entries.
 *
 * Stream ids under one request seed: B200TTS_SEED_STREAM_PRENET0 and _PRENET1 for the decoder's
 * two per-step prenet dropout sites (b200tts_fill_keep_mask_rows, width P, one step per decoder step), B200TTS_SEED_STREAM_VOCODER for
 * the WaveRNN sample loop's uniforms (b200tts_fill_uniform_rows, one step per sample). */
int b200tts_fill_uniform_rows(float* out, int rows, int nsteps, int width, const uint64_t* seeds, const int64_t* t0, uint64_t stream_id,
                              void* stream);
#define B200TTS_SEED_STREAM_PRENET0 0x5EED000000000001ull
#define B200TTS_SEED_STREAM_PRENET1 0x5EED000000000002ull
#define B200TTS_SEED_STREAM_VOCODER 0x5EED000000000003ull

/* ---- optimizer step on flat buffers: clip_grad_norm_ + torch.optim.Adam with coupled L2 decay (train.py:84-85, 260-271) ----
 * p, g, m, v: n fp32 elements each (the flat parameter buffer, the flat all-reduced gradient, Adam moments); g is overwritten with
 * the clipped gradient; max_norm <= 0 disables clipping; step counts from 1; scratch holds b200tts_adam_clip_scratch_floats()
 * floats, scratch[0] = gradient norm before clipping, scratch[1] = applied clip coefficient (device values after the call). */
size_t b200tts_adam_clip_scratch_floats(void);
int b200tts_adam_clip_step(float* p, float* g, float* m, float* v, size_t n, float lr, float beta1, float beta2, float eps,
                           float weight_decay, float max_norm, int step, float* scratch, void* stream);

/* ---- Griffin-Lim vocoder: audio.inverse_spectrogram, reference utils/audio.py:88-97 (librosa 0.7.0) ----
 * Packed ragged layout, frame-major: utterance b owns frames [off[b], off[b+1]) (off: int32 [B+1], device, off[0] = 0, F_b >= 2);
 * K = N/2 + 1 bins.  Magnitudes S [total_frames, K] fp32; angles and rebuilt [total_frames, K] complex64 (re, im pairs); waveforms
 * packed at hop * (off[b] - b) with hop * (F_b - 1) samples each.  No utterance reads another's data and nothing uses atomics: every
 * result is bit-reproducible and independent of the batch it is computed in.  fp32 whatever b200tts_set_precision says.
 * Supported: even N <= 2048 whose N/2 has no prime factor above 31, 1 <= win <= N (periodic Hann centre-padded to N), 1 <= hop <= win. */
typedef struct {
    int B, total_frames;
    int N, hop, win;
    int n_mels;          /* 0: the input is a linear log spectrogram [total_frames, K]; > 0: a log-mel spectrogram [total_frames, n_mels] */
    float power;         /* magnitude exponent before Griffin-Lim (hp.griffin_lim_power) */
    float momentum;      /* Griffin-Lim momentum (librosa 0.7.0: 0.99) */
    float preemphasis;   /* de-emphasis coefficient; 0 = off */
    int nnls_iters;      /* FISTA steps of the mel inversion */
} b200tts_vocoder_shape;
/* Host only: the griffinlim workspace (twiddles, window, frame buffer [total_frames, N]); 0 for an invalid shape (message set). */
size_t b200tts_vocoder_workspace_bytes(const b200tts_vocoder_shape* shape);
/* Host only: the radices of the complex FFT of length N/2, in stage order, into radices[0:capacity]; returns the stage count, or a
 * negative status for an unsupported N. */
int b200tts_vocoder_fft_plan(int N, int* radices, int capacity);
/* S = db_to_amplitude(log_spec) = (10^(0.1 s))^0.5; mel input: S = nnls(mel_basis, S) by FISTA from clip(pinv(A) S, 0) with step
 * nnls_step (1 / ||A||_2^2); then S ** power.  mel_basis [n_mels, K] (every bin in at most two adjacent filters, as the Slaney basis is),
 * mel_pinv_t = pinv(mel_basis)^T [n_mels, K]; both NULL for a linear input. */
int b200tts_spectrogram_magnitude(const b200tts_vocoder_shape* shape, const float* log_spec, const float* mel_basis, const float* mel_pinv_t,
                                  float nnls_step, float* S_out, void* stream);
/* `iters` Griffin-Lim iterations from the given state (librosa.griffinlim):  inverse = istft(S * angles); rebuilt' = stft(inverse)
 * (centre reflect padding); angles = rebuilt' - momentum / (1 + momentum) * rebuilt; angles /= |angles| + 1e-16; rebuilt = rebuilt'.
 * first != 0: the previous rebuilt counts as 0 (it is not read).  Then, if wave != NULL, wave = istft(S * angles). */
int b200tts_griffinlim(const b200tts_vocoder_shape* shape, const float* S, const int32_t* off, float* angles, float* rebuilt, int first,
                       int iters, float* wave, void* workspace, size_t workspace_bytes, void* stream);
/* In place per utterance: wave = lfilter([1], [1, -preemphasis], wave) (skipped when preemphasis = 0), then wave /= max(wave) -- the
 * largest sample, not the largest magnitude, as the reference's Python max() is. */
int b200tts_deemphasis_normalize(const b200tts_vocoder_shape* shape, float* wave, const int32_t* off, void* stream);

/* ---- streaming Griffin-Lim: frame-by-frame phase reconstruction with look-ahead (RTISI-LA), audio.GriffinLimVocoder ----
 * Up to `slots` streams, each in its own workspace slot: the committed overlap-add c over the frames still open, the time-domain estimates
 * of the look-ahead set A = {m .. min(m + k, F - 1)}, their magnitudes, the frame counters and the de-emphasis carry.  Frame m is processed
 * once frame m + k has arrived or the stream has ended: the frames of A not yet in it are admitted in increasing j (x_j = irfft(S_j X / |X|),
 * X = rfft(w p_j), p_j = (c + the overlap-add of the frames of A before j) / e over frame j's span, phase 1 where X = 0), then `iters`
 * Jacobi iterations project every frame of A against p_j = (c + the overlap-add of all of A) / e, then c += w x_m.  e is the one-sided
 * envelope sum_{i >= 0} w^2(n - i hop) (0 where it is 0).  The samples of the trimmed output (z[N/2 .. N/2 + hop (F - 1)) of the untrimmed
 * signal z) below (m + 1) hop, or all of them after the last frame, are released divided by the window sum-square of frames 0..m where that
 * exceeds tiny(float32), then de-emphasised (y = x + preemphasis y_prev, carried across calls; 0 = off).  No peak normalisation.  fp32. */
#define B200TTS_GL_STREAM_MAX_LOOKAHEAD 7
typedef struct {
    int N, hop, win;     /* as in b200tts_vocoder_shape: periodic Hann of win samples centre-padded to N */
    int lookahead;       /* k, 0 to B200TTS_GL_STREAM_MAX_LOOKAHEAD */
    int iters;           /* Jacobi iterations per processed frame, >= 1 */
    int slots;           /* streams of the workspace, 1 to 64 */
    float preemphasis;   /* in (-1, 1) */
} b200tts_gl_stream_shape;
typedef struct {
    int slot;            /* the stream's workspace slot; each slot at most once per call */
    int frames;          /* frames the stream has received, this call's included (never fewer than the previous call's) */
    int ended;           /* nonzero: `frames` is the stream's length F (>= 2) */
    long long s_off;     /* row of S_new holding the first frame received since the previous call */
    long long wave_off;  /* where the samples this call releases go in `wave` */
} b200tts_gl_stream_row;
/* Host only: the workspace (twiddles, window and `slots` slots); 0 for an invalid shape (message set). */
size_t b200tts_gl_stream_workspace_bytes(const b200tts_gl_stream_shape* shape);
/* Resets the `count` listed slots (host int32, distinct, each in [0, slots)) to an empty stream, and writes the FFT tables: a workspace is
 * run only after its first reset.  One launch. */
int b200tts_gl_stream_reset(const b200tts_gl_stream_shape* shape, void* workspace, size_t workspace_bytes, const int32_t* slots, int count,
                            void* stream);
/* One call over `count` rows (host descriptors, 1 to 64): row r's stream takes its new frames' magnitudes from S_new [rows, N/2 + 1] (fp32,
 * b200tts_spectrogram_magnitude's output), processes every frame that is ready, in order, and writes the samples it releases to
 * wave + wave_off.  S_new and wave are required even when no row has new frames or releases samples.  The frame count a slot has
 * received lives on the device, so the call cannot check that S_new holds rows [s_off, s_off + frames - that count) for every row, nor
 * that wave is long enough: the caller keeps that count (frames of its previous call, 0 after a reset), as for any device buffer.  One CTA per row, one launch; no slot is read by another row's CTA, so a stream's bits do not depend on its company or on
 * how its frames were cut into calls. */
int b200tts_gl_stream_run(const b200tts_gl_stream_shape* shape, const b200tts_gl_stream_row* rows, int count, const float* S_new, float* wave,
                          void* workspace, size_t workspace_bytes, void* stream);

/* ---- audio analysis: audio.spectrogram and mel_cepstral_distorision, reference utils/audio.py:66-78, 117-161 (librosa 0.7.0) ----
 * Packed ragged layout: utterance b owns samples [soff[b], soff[b+1]) of an fp32 waveform (L_b >= 1) and frames [off[b], off[b+1]) with
 * F_b = 1 + L_b / hop (soff, off: int32 [B+1], device, both starting at 0; the caller keeps them consistent).  Spectra are frame-major
 * [total_frames, bins] fp32 with bins = K = N/2 + 1 (linear) or n_mels.  No utterance reads another's data and nothing uses atomics: every
 * result is bit-reproducible and independent of the batch it is computed in.  Supported: even N <= 2048 whose N/2 has no prime factor
 * above 31, 1 <= win <= N (periodic Hann centre-padded to N), hop >= 1. */
typedef struct {
    int B, total_samples, total_frames;
    int N, hop, win;
    int n_mels;          /* 0: linear magnitudes [total_frames, K]; > 0: mel magnitudes [total_frames, n_mels] */
    double preemphasis;  /* pre-emphasis coefficient a: y[n] - a y[n-1] before the padding; 0 = off */
} b200tts_analysis_shape;
/* Host only: the stft_magnitude workspace (fp64 twiddles and window, mel filter ranges); 0 for an invalid shape (message set). */
size_t b200tts_analysis_workspace_bytes(const b200tts_analysis_shape* shape);
/* |stft(preemphasis(y), center=True, pad_mode='reflect', window='hann')| per utterance: the transform in fp64, rounded to complex64, the
 * magnitude in fp32; np.pad's repeated reflection when L_b < N/2.  mel_basis [n_mels, K] (NULL when n_mels = 0): out = mel_basis . |X|,
 * each filter summing its nonzero bins in ascending order in fp32.  workspace: 256-byte aligned, b200tts_analysis_workspace_bytes. */
int b200tts_stft_magnitude(const b200tts_analysis_shape* shape, const float* wave, const int32_t* soff, const int32_t* off,
                           const float* mel_basis, float* out, void* workspace, size_t workspace_bytes, void* stream);
/* librosa amplitude_to_db(S, ref=np.max, amin=1e-5, top_db=None) per utterance, fp32: 10 log10(max(1e-10, S^2)) minus the same of the
 * utterance's largest |S|.  S and out [total_frames, bins] (bins from shape->n_mels); out may be S. */
int b200tts_amplitude_to_db(const b200tts_analysis_shape* shape, const float* S, const int32_t* off, float* out, void* stream);
/* librosa mfcc(S = mel_db / 10, n_mfcc): scipy.fftpack.dct(type=2, norm='ortho') over the n_mels axis, the first n_mfcc coefficients
 * (c0 included).  mel_db [total_frames, n_mels] -> out [total_frames, n_mfcc], fp32 (the DCT matrix from fp64, rounded to fp32). */
int b200tts_mel_cepstrum(int total_frames, int n_mels, int n_mfcc, const float* mel_db, float* out, void* stream);
#define B200TTS_MCD_CUT 0
#define B200TTS_MCD_STRETCH 1
#define B200TTS_MCD_DTW 2
/* DTW keeps three anti-diagonals of (fp64, int32) in shared memory: the shorter sequence of a pair may have at most this many frames. */
#define B200TTS_DTW_MAX_FRAMES 6455
/* Mel cepstral distortion of B pairs (reference mel_cepstral_distorision): pair b is cep_a frames [off_a[b], off_a[b+1]) against cep_b
 * frames [off_b[b], off_b[b+1]) (each [frames, n_mfcc] fp32; off_a, off_b int32 [B+1], device; every sequence non-empty).  The frame
 * distance is the Euclidean distance over coefficients 1..n_mfcc-1, summed in index order in fp32; means and costs accumulate in fp64.
 * CUT: mean over the first min(F_a, F_b) frame pairs.  STRETCH: the shorter sequence indexed at i * n // m over the longer length m (the
 * first when the lengths are equal).  DTW: the exact dynamic-time-warping optimum (fastdtw's recurrence without its radius-1
 * approximation): path cost / path length.  mcd_out: double [B]; path_len_out: int32 [B] (pairs averaged over) or NULL.  A DTW pair whose
 * shorter side exceeds B200TTS_DTW_MAX_FRAMES gets NaN and path length -1. */
int b200tts_mel_cepstral_distortion(int B, int n_mfcc, int mode, const float* cep_a, const int32_t* off_a, const float* cep_b,
                                    const int32_t* off_b, double* mcd_out, int32_t* path_len_out, void* stream);

/* ---- forced alignment: monotonic alignment search over attention probabilities (no counterpart in the reference) ----
 * P: fp32 attention probabilities of B utterances, utterance b's weight of symbol l at decoder step s at P[b batch_stride + s ld + l]
 * (s < S, l < L: a padded [B, S, L] batch).  text_lengths, step_lengths: int32 [B], device; utterance b uses steps s < S_b and symbols
 * l < L_b.  No workspace.  One CTA per utterance: no utterance reads another's data and nothing uses global atomics, so every result is
 * bit-reproducible and independent of the batch it is computed in. */
typedef struct {
    int B, S, L;              /* utterances; padded steps and symbols (1 <= L <= B200TTS_ALIGN_MAX_SYMBOLS) */
    long long ld;             /* elements between consecutive steps of one utterance (>= L) */
    long long batch_stride;   /* elements between consecutive utterances (>= 0) */
} b200tts_align_shape;
/* The search keeps two fp64 rows of L values and one back-pointer bit per cell in shared memory (227 KB): an utterance may have at most
 * this many symbols, and S_b L_b at most this many cells (1,688 steps at 1,024 symbols; 5,761 steps at 300). */
#define B200TTS_ALIGN_MAX_SYMBOLS 1024
#define B200TTS_ALIGN_MAX_CELLS 1728512
/* Monotonic alignment search (Glow-TTS MAS) per utterance: the path l_0 = 0, l_{S_b - 1} = L_b - 1, l_{s+1} - l_s in {0, 1} that maximises
 * sum_s log(max(P[s, l_s], 1e-8)), accumulated in fp64 (log of the fp32 weight widened to fp64).  Recurrence Q[s][l] = log max(P[s, l],
 * 1e-8) + max(Q[s-1][l], Q[s-1][l-1]).  Tie rule: the path advances from symbol l - 1 to l at step s only when Q[s-1][l-1] > Q[s-1][l]
 * strictly; on equal values it stays on symbol l.  durations_out int32 [B, L]: steps per symbol (each >= 1 below L_b, summing to S_b;
 * 0 from L_b on); path_logp_out double [B]: the path's sum; path_out int32 [B, S] or NULL: the symbol of each step (-1 from S_b on).
 * Requires 1 <= L_b <= S_b <= S, L_b <= L and S_b L_b <= B200TTS_ALIGN_MAX_CELLS: lengths live on the device, so the caller checks them;
 * an utterance outside these gets durations -1, path -1 and a NaN path_logp. */
int b200tts_monotonic_alignment(const b200tts_align_shape* shape, const float* P, const int32_t* text_lengths, const int32_t* step_lengths,
                                int32_t* durations_out, double* path_logp_out, int32_t* path_out, void* stream);
/* Alignment quality per utterance over steps s < S_b and symbols l < L_b (fp64 sums, fp32 results): focus_out, the mean over steps of the
 * step's largest weight; coverage_out, the fraction of symbols whose weights summed over the steps reach 0.5; max_jump_out (int32), the
 * largest forward move of the per-step argmax (the first index on equal weights) between consecutive steps, 0 if it never moves forward;
 * moves_back_out (int32), 1 if it ever moves backwards.  Requires 1 <= L_b <= L and 1 <= S_b <= S; an utterance outside these gets NaN
 * scores and -1 moves. */
int b200tts_alignment_scores(const b200tts_align_shape* shape, const float* P, const int32_t* text_lengths, const int32_t* step_lengths,
                             float* focus_out, float* coverage_out, int32_t* max_jump_out, int32_t* moves_back_out, void* stream);

/* ---- pitch analysis: probabilistic YIN F0 tracks (librosa 0.10 librosa.pyin; no counterpart in the reference) ----
 * Packed ragged layout as the analysis entry points: utterance b owns samples [soff[b], soff[b+1]) of an fp32 waveform (L_b >= 1) and
 * frames [off[b], off[b+1]) with F_b = 1 + L_b / hop (soff, off: int32 [B+1], device).  Frame t of utterance b is the frame_length samples
 * y[0 .. frame_length) starting at sample t hop - frame_length / 2, zero outside [0, L_b) (center=True, constant padding, no
 * pre-emphasis).  The host computes every derived quantity below once, with numpy, and passes it in the shape.  No utterance reads another's
 * data, sums run in a fixed order and nothing uses atomics: every result is bit-reproducible and independent of the batch it is computed in.
 * fp64 whatever b200tts_set_precision says. */
#define B200TTS_PITCH_THRESHOLDS 100
/* The Viterbi keeps two fp64 rows of 2 n states plus prefix and suffix maxima of both halves in shared memory, and uint16 back-pointers. */
#define B200TTS_PITCH_MAX_BINS 1201
#define B200TTS_PITCH_MAX_FRAME_LENGTH 2048
typedef struct {
    int B, total_samples, total_frames;
    int frame_length, win_length, hop; /* even frame_length <= B200TTS_PITCH_MAX_FRAME_LENGTH, win_length = frame_length / 2, hop >= 1 */
    int min_period, max_period;        /* floor(sr / fmax), min(ceil(sr / fmin), frame_length - win_length - 1); K = max - min + 1 >= 2 */
    int n_bins;                        /* n = floor(120 log2(fmax / fmin)) + 1 pitch bins, 1 <= n <= B200TTS_PITCH_MAX_BINS */
    int transition_width;              /* W = round(35.92 * 12 hop / sr) * 10 + 1, odd, 1 <= W <= n */
    double sr, fmin;
    double log_tiny;                   /* log(DBL_MIN): an out-of-band transition and a zero observation */
    double log_init;                   /* log(1 / n + DBL_MIN): the start probability of each unvoiced state */
    double thresholds[B200TTS_PITCH_THRESHOLDS];   /* linspace(0, 1, 101)[1:] */
    double beta_probs[B200TTS_PITCH_THRESHOLDS];   /* diff(scipy.stats.beta.cdf(linspace(0, 1, 101), 2, 18)) */
} b200tts_pitch_shape;
/* Host only: the bytes of b200tts_pitch_viterbi's back-pointers (uint16 [total_frames, 2 n]); 0 for an invalid shape (message set). */
size_t b200tts_pitch_workspace_bytes(const b200tts_pitch_shape* shape);
/* Stage A, the cumulative mean normalised difference per frame, in fp64 from the fp32 samples (direct sums in index order):
 *   acf(tau) = sum_{i=1}^{win} y_i y_{i+tau},  e(tau) = sum_{i=tau+1}^{tau+win} y_i^2, each set to 0 where its magnitude is below 1e-6;
 *   d(tau) = (e(0) + e(tau)) - 2 acf(tau);  d'(tau) = d(tau) / (c(tau) / tau + DBL_MIN), c(tau) = d(1) + ... + d(tau) summed in order.
 * cmnd_out: double [total_frames, K], entry k = d'(min_period + k). */
int b200tts_pitch_cmnd(const b200tts_pitch_shape* shape, const float* wave, const int32_t* soff, const int32_t* off, double* cmnd_out,
                       void* stream);
/* Stage B, pYIN observation probabilities from d' [total_frames, K].  Troughs: k = 0 iff d'[0] < d'[1]; 0 < k < K - 1 iff d'[k] < d'[k-1]
 * and d'[k] <= d'[k+1]; k = K - 1 iff d'[K-1] < d'[K-2].  For threshold j with N_j troughs below thresholds[j], a trough below it at
 * position p among them gets prior (1 - e^-2) / (1 - e^(-2 N_j)) e^(-2 p) (Boltzmann, lambda 2); its probability is sum_j prior_j
 * beta_probs[j].  The first lowest trough also gets 0.01 sum beta_probs[j] over the thresholds it is not below.  A trough with nonzero
 * probability maps to bin rint(120 log2(sr / (min_period + k + s) / fmin)) clipped to [0, n] (half to even), with the parabolic shift
 * s = -b / a (a = d'[k+1] + d'[k-1] - 2 d'[k], b = (d'[k+1] - d'[k-1]) / 2; s = 0 when |b| >= |a| and at both ends).  Of troughs sharing a
 * bin the larger lag wins; bin n is dropped.  obs_out: double [total_frames, n], zero elsewhere; voiced_prob_out: double [total_frames],
 * clip(sum of obs_out's row, 0, 1). */
int b200tts_pitch_observations(const b200tts_pitch_shape* shape, const double* cmnd, double* obs_out, double* voiced_prob_out, void* stream);
/* Stage C, librosa.sequence.viterbi over 2 n states (voiced bins, then unvoiced bins), one CTA per utterance.  Log observations:
 * log(obs + DBL_MIN) for voiced state i, log((1 - voiced_prob) / n + DBL_MIN) for every unvoiced state.  Start: log_tiny on the voiced
 * states, log_init on the unvoiced ones.  log_trans: double [2, W, n] (device), log_trans[s, q, i] = log(S_s T[i - h + q, i] + DBL_MIN)
 * for the source bin i - h + q in [0, n) (h = W / 2; other entries unread), T the row-normalised triangular band of librosa's
 * transition_local(n, W, 'triangle', wrap=False), S_0 = 1 - 0.01 (same voicing) and S_1 = 1 - S_0 (switch).  Every transition outside the
 * band costs log_tiny, as in the dense kron(transition_loop(2, 1 - 0.01), T).  Ties go to the lowest source state, and the final state is the
 * first best.  state_out: int32 [total_frames], the decoded state (bin i voiced when < n, bin state - n unvoiced).  workspace: at least
 * b200tts_pitch_workspace_bytes. */
int b200tts_pitch_viterbi(const b200tts_pitch_shape* shape, const double* obs, const double* voiced_prob, const int32_t* off,
                          const double* log_trans, int32_t* state_out, void* workspace, size_t workspace_bytes, void* stream);

/* ---- pitch modification: TD-PSOLA pitch shifting (no counterpart in the reference; tests/psola_oracle.py states the contract) ----
 * The packed ragged layout of the pitch entry points: utterance b owns samples [soff[b], soff[b+1]) of an fp32 waveform (L_b >= 1) and
 * frames [off[b], off[b+1]) with F_b = 1 + L_b / hop.  Sample n is in frame min(F_b - 1, (n + hop / 2) / hop); per frame, f0 (fp32 Hz, NaN
 * unvoiced) and r (fp32, new F0 / old F0).  P(n) = rint(sr / f0) in fp64 (half to even); U = unvoiced_spacing.
 *   Analysis marks m_0 < m_1 < ... in [0, L_b): m_0 = argmax x over [0, min(L, P(0))) when sample 0 is voiced, else 0.  From a voiced mark
 *   (p = P(m)): c = m + p, stop when c >= L; next = argmax x over [c - p/4, min(L - 1, c + p/4)] when c is voiced, else c.  From an
 *   unvoiced mark, o = the first voiced sample after it (L if none): next = m + U when m + U < o (stop when >= L), else argmax x over
 *   [o, min(L, o + P(o))) (stop when o = L).  argmax is over signed x, first index on ties.  d_k = m_{k+1} - m_k; the last mark's d is its
 *   nominal period (P voiced, U unvoiced).
 *   Synthesis marks: t_0 = m_0, t_{j+1} = t_j + q_j in fp64, c_j = rint(t_j) until c_j >= L; k(j) the analysis mark nearest c_j (lower on
 *   ties); q_j = d_k / r[frame(c_j)] when mark k is voiced, else d_k.
 *   Overlap-add: grain j reads x around m_{k(j)}, writes around c_j, half-widths a = d_{k-1} (grain of mark 0: max(its nominal period, m_0))
 *   and b = d_k, weight (1 + cos(pi u / (a + 1))) / 2 for -a <= u <= 0 and (1 + cos(pi u / (b + 1))) / 2 for 0 <= u <= b, except 1 on the
 *   left half of mark 0's grains and the right half of the last mark's.  y(n) = sum w x[m + n - c_j] / max(1, sum w) over the grains
 *   covering n whose source index is in [0, L), both sums fp64 in increasing j; y = 0 where no grain covers n.  At r = 1, y = x.
 * Workspace (b200tts_psola_workspace_bytes): int32 info [B, 4] = {analysis marks K_b, synthesis marks J_b, grain 0's left half-width,
 * W_b = the largest half-width}, then int32 [total_samples] each of marks, d, centres c and k, then uint8 [total_samples] voiced flags of
 * the marks; utterance b's entries start at soff[b] (K_b, J_b <= L_b).  No utterance reads another's data, sums run in a fixed order and
 * nothing uses atomics: results are bit-identical in any batch.  fp64 whatever b200tts_set_precision says.  The host checks f0 and r (voiced
 * periods in [2, B200TTS_PSOLA_MAX_PERIOD], ratios finite in [0.5, 2]); the kernels clamp both into those ranges, so no input can make a
 * walk run away. */
#define B200TTS_PSOLA_MAX_PERIOD 1024
typedef struct {
    int B, total_samples, total_frames;
    int hop;                           /* frames of the f0 and ratio tracks: F_b = 1 + L_b / hop, hop >= 1 */
    int unvoiced_spacing;              /* U, in [1, B200TTS_PSOLA_MAX_PERIOD] */
    double sr;                         /* sample rate in Hz */
} b200tts_psola_shape;
/* Host only: the workspace bytes of a batch; 0 for an invalid shape (message set). */
size_t b200tts_psola_workspace_bytes(const b200tts_psola_shape* shape);
/* Analysis and synthesis marks, one warp per utterance: wave fp32 [total_samples], f0 and ratio fp32 [total_frames] -> workspace. */
int b200tts_psola_marks(const b200tts_psola_shape* shape, const float* wave, const int32_t* soff, const float* f0, const float* ratio,
                        const int32_t* off, void* workspace, size_t workspace_bytes, void* stream);
/* Overlap-add from the marks b200tts_psola_marks wrote, as a gather: each output sample sums the grains whose centre lies within W_b of it.
 * out: fp32 [total_samples], not aliasing wave. */
int b200tts_psola_overlap_add(const b200tts_psola_shape* shape, const float* wave, const int32_t* soff, const void* workspace,
                              size_t workspace_bytes, float* out, void* stream);

/* ---- time-scale modification: WSOLA time stretching (no counterpart in the reference; tests/wsola_oracle.py states the contract) ----
 * The packed ragged layout of the pitch entry points: utterance b owns input samples [soff[b], soff[b+1]) of an fp32 waveform x (L >= 1,
 * read as 0 outside [0, L)), output samples [ooff[b], ooff[b+1]) (L' >= 1) and synthesis frames [foff[b], foff[b+1]), K = (L' - 1) / H + 2
 * of them.  H = hop, N = 2H, D = tolerance.  Frame k is centred on output sample kH; warp[k] is its input position tau_k (fp64).
 *   Nominal positions: a_k = rint(clamp(tau_k, 0, L)) (half to even; NaN reads as 0).
 *   Search: p_0 = a_0.  For k >= 1, u_m = x[p_{k-1} + H + m] (the natural continuation of frame k - 1) and v_{d,m} = x[a_k + d + m] for m in
 *   [-H, H) and d in [-D, D].  C(d) = sum u v and E(d) = sum v v, each an fp64 sum of the exact fp64 products of fp32 samples, accumulated
 *   one term at a time in increasing m from 0.0 (C = fma(u, v, C)).  s(d) = C / sqrt(E), IEEE fp64, and s = 0 where E = 0.
 *   p_k = a_k + the d of largest s; on exact ties the smallest |d| wins, then the negative d.  At tau_k = kH, d = 0 is the Cauchy-Schwarz
 *   maximum, so y = x up to rounding; silence (every s = 0) copies the nominal positions.
 *   Overlap-add: y[n] = sum over k in {n / H, n / H + 1} (frames the utterance has) of w(n - kH + H) x[p_k + n - kH], summed in fp64 in
 *   increasing k and rounded to fp32, with w(i) = 0.5 - 0.5 cos(pi i / H), the periodic Hann window of length 2H.  w(i) + w(i + H) = 1,
 *   so there is no normalisation.
 * No workspace and no atomics; no utterance reads another's data, so results are bit-identical in any batch.  fp64 whatever
 * b200tts_set_precision says.  total_samples <= INT_MAX - B200TTS_WSOLA_MAX_TOLERANCE, so every position fits in int32. */
#define B200TTS_WSOLA_MAX_HOP 1024
#define B200TTS_WSOLA_MAX_TOLERANCE 1024
typedef struct {
    int B, total_samples, total_out_samples, total_frames;
    int hop;                           /* H in [1, B200TTS_WSOLA_MAX_HOP] */
    int tolerance;                     /* D in [0, B200TTS_WSOLA_MAX_TOLERANCE] */
} b200tts_wsola_shape;
/* The frame positions p, one CTA per utterance walking its frames in order: wave fp32 [total_samples], warp fp64 [total_frames] ->
 * positions int32 [total_frames]. */
int b200tts_wsola_positions(const b200tts_wsola_shape* shape, const float* wave, const int32_t* soff, const double* warp,
                            const int32_t* foff, int32_t* positions, void* stream);
/* The overlap-add of the frames at the positions b200tts_wsola_positions wrote, one thread per output sample: out fp32
 * [total_out_samples], not aliasing wave. */
int b200tts_wsola_overlap_add(const b200tts_wsola_shape* shape, const float* wave, const int32_t* soff, const int32_t* positions,
                              const int32_t* foff, const int32_t* ooff, float* out, void* stream);

/* ---- polyphase resampling: scipy.signal.resample_poly(x, up, down) with its defaults (tests/resample_oracle.py restates it) ----
 * The packed ragged layout of the WSOLA entry points: utterance b owns input samples [soff[b], soff[b+1]) of an fp32 waveform x (L >= 1)
 * and output samples [ooff[b], ooff[b+1]), L' = ceil(L up / down) of them.  plan int32 [B][4], 16-byte aligned, holds (up, down, h_len,
 * table offset) per utterance, up / down the rate ratio in lowest terms, m = max(up, down) <= max_factor, h_len = 10 m.
 *   Filter: h[j] = up w[j] / sum(w), j in [0, 2 h_len], w[j] = (1/m) sinc((j - h_len) / m) kaiser(2 h_len + 1, beta 5)[j] (scipy's
 *   firwin(2 h_len + 1, 1 / m, window=('kaiser', 5.0))), built by the caller in fp64.
 *   Table: taps[offset + phase T + i] = h[phase + i up] for phase in [0, up) and i in [0, T), T = ceil((2 h_len + 1) / up), 0 where
 *   phase + i up > 2 h_len: each phase's taps are contiguous.
 *   Output: with t = h_len + n down (64-bit), k0 = t / up and phase = t mod up,
 *   y[n] = sum over i in [0, T) with phase + i up <= 2 h_len and k0 - i in [0, L) of x[k0 - i] taps[offset + phase T + i], that is
 *   y[n] = sum_k x[k] h[h_len + n down - k up] over the k whose h index lies in [0, 2 h_len].  The sum is fp64, accumulated by fma in
 *   increasing i from 0.0, and rounded to fp32 once.
 * One thread per output sample; no workspace and no atomics, and no utterance reads another's data, so results are bit-identical in any
 * batch.  fp64 whatever b200tts_set_precision says.  out fp32 [total_out_samples] must not alias wave or taps. */
#define B200TTS_RESAMPLE_MAX_FACTOR 2048
typedef struct {
    int B, total_samples, total_out_samples;
    int total_taps;                    /* doubles in taps: every plan's offset + up T lies within it */
    int max_factor;                    /* the largest max(up, down) of the plan, in [1, B200TTS_RESAMPLE_MAX_FACTOR] */
} b200tts_resample_shape;
int b200tts_resample(const b200tts_resample_shape* shape, const float* wave, const int32_t* soff, const int32_t* ooff, const int32_t* plan,
                     const double* taps, float* out, void* stream);

/* ---- silence trimming: librosa 0.7.0 effects.trim(x, top_db, frame_length, hop_length) (tests/resample_oracle.py restates it) ----
 * The packed ragged layout: utterance b owns samples [soff[b], soff[b+1]) of an fp32 waveform x (L >= 1, already cropped by any margin)
 * and frames [foff[b], foff[b+1]), F = 1 + (L + 2 (W / 2) - W) / hop of them, W = frame_length.
 *   Frame power: p_f = sum_{j < W} x_pad[f hop + j]^2 / W in fp64, x_pad the signal reflect-padded by W / 2 on both sides with numpy's
 *   repeated reflection (period 2 (L - 1); a single sample repeats).  Each frame is summed by one warp in a fixed order.
 *   Decision: db_f = 10 log10(max(1e-10, p_f)) - 10 log10(max(1e-10, max_f p_f)); frame f is non-silent when db_f > -top_db.
 *   Bounds: with a and b the first and last non-silent frames, (start, end) = (a hop, min(L, (b + 1) hop)); (0, 0) when none is.
 * Two kernels: one warp per frame for p, then one CTA per utterance for the maximum and the bounds.  No atomics, so results are the same
 * in any batch.  power fp64 [total_frames] (the frame powers p) and bounds int32 [B][2] are written; fp64 whatever b200tts_set_precision
 * says. */
typedef struct {
    int B, total_samples, total_frames;
    int frame_length;                  /* W >= 1 */
    int hop;                           /* >= 1 */
    double top_db;                     /* finite */
} b200tts_trim_shape;
int b200tts_trim_silence(const b200tts_trim_shape* shape, const float* wave, const int32_t* soff, const int32_t* foff, double* power,
                         int32_t* bounds, void* stream);

/* ---- WaveRNN vocoder (fatchord architecture): mel -> waveform, one GRU step per sample over fold rows ----
 * The MelResNet and the time-batched conditioning products run on the convolution-block and GEMM entry points; these entry points add
 * the mel upsampling layers, the folding, the persistent sample loop and the unfolding.  Fold rows: utterance b's F_b hop sample
 * positions are cut into folds of fold_len = target + 2 overlap samples starting every target + overlap (fold_with_overlap, the tail
 * zero-padded); the rows of all utterances are numbered consecutively.  These entry points are fp32 whatever b200tts_set_precision
 * says, except the loop's recurrent products (bf16 operands, fp32 accumulation and state); the convolution-block and GEMM stages follow
 * the precision mode, which WaveRNN.generate_batch sets to fp32 for the duration of a call. */
#define B200TTS_WAVERNN_RAW 0
#define B200TTS_WAVERNN_MOL 1
/* out[c, i] = sum_{k=-s..s} fir[k + s] in[c, (i + k) / s] over 0 <= i + k < len s: nearest stretch x s, then the FIR of 2s+1 taps with zero
 * padding s (an upsampling layer pair).  in [C, len], out [C, len s], fp32. */
int b200tts_wavernn_upsample_layer(int C, int len, int scale, const float* fir, const float* in, float* out, void* stream);
typedef struct {
    int B, rows;          /* utterances; fold rows of all of them */
    int n_mels, aux_dims; /* feature columns: the mel path, then the MelResNet output (all four quarters) */
    int hop, pad, scale;  /* hop = the product of the upsampling factors; pad frames on each side; scale = the last factor */
    int target, overlap;
    int max_frames;       /* aux is [B, max_frames, aux_dims] */
} b200tts_wavernn_fold_shape;
/* feat [nsteps, rows, n_mels + aux_dims] for the loop steps [t0, t0 + nsteps): row r (utterance row_utt[r], fold row_fold[r]) at step t is
 * sample position q = fold (target + overlap) + t; zero for q >= F_b hop.  Mel columns: the last upsampling layer (taps fir [2 scale + 1])
 * at the uncut position q + pad hop, from mel_up + mel_off[b], the penultimate layer [n_mels, (F_b + 2 pad) hop / scale] of the padded
 * mel; aux columns: aux[b, q / hop, :].  frames, row_utt, row_fold: int32; mel_off: int64 element offsets; all on the device. */
int b200tts_wavernn_fold(const b200tts_wavernn_fold_shape* shape, const float* mel_up, const int64_t* mel_off, const int32_t* frames,
                         const int32_t* row_utt, const int32_t* row_fold, const float* fir, const float* aux, int t0, int nsteps, float* feat,
                         void* stream);
typedef struct {
    int n_mels, aux_dims; /* feature columns, as in b200tts_wavernn_fold_shape */
    int hop, pad, scale;
    int frames;           /* the mel's frame count F once it is known (positions from F hop on are 0), 0 while the mel is still arriving */
    long long m0;         /* the mel window holds samples [m0, m0 + mel_len) of the penultimate layer of the padded mel */
    int mel_len;
    int a0, aux_len;      /* the aux window holds frames [a0, a0 + aux_len) */
} b200tts_wavernn_window_shape;
/* Rows of one call of b200tts_wavernn_window_rows and segments of b200tts_wavernn_upsample_segments: at most this many. */
#define B200TTS_WAVERNN_MAX_STREAMS 64
typedef struct {
    b200tts_wavernn_window_shape w;   /* the row's windows; n_mels, aux_dims, hop, pad, scale equal in every row */
    long long s0;                     /* the row's first position (its steps run so far) */
    long long mel_off, aux_off;       /* element offsets of the row's mel and aux windows in the packed buffers */
    int n;                            /* positions [s0, s0 + n), 0 to nsteps */
} b200tts_wavernn_window_row;
/* feat [nsteps, active_rows, n_mels + aux_dims] of active_rows unfolded rows (one utterance each, no folds) in one launch: row r's step i
 * holds the features of sample position q = rows[r].s0 + i for i < rows[r].n, zero past it.  They are the columns b200tts_wavernn_fold
 * writes for q, with the same arithmetic (zero for q >= F hop once F = w.frames is known), read from the row's windows: mel + mel_off
 * [n_mels, mel_len] holds the penultimate layer's samples [m0, m0 + mel_len) (equal to the whole padded mel's wherever they are read),
 * aux + aux_off [aux_len, aux_dims] the MelResNet output's frames [a0, a0 + aux_len).  rows: host descriptors.  B200TTS_ERR_INVALID when a
 * read of a row with n > 0 would fall outside its windows. */
int b200tts_wavernn_window_rows(const b200tts_wavernn_window_row* rows, int active_rows, int nsteps, const float* mel, const float* fir,
                                const float* aux, float* feat, void* stream);
/* b200tts_wavernn_upsample_layer over nseg packed segments (1 to B200TTS_WAVERNN_MAX_STREAMS): segment g is in [C, lens[g]] right after
 * segment g - 1 and goes to out [C, lens[g] scale] at scale times its input offset; each equal to its own b200tts_wavernn_upsample_layer.
 * lens: host int32. */
int b200tts_wavernn_upsample_segments(int C, int nseg, const int32_t* lens, int scale, const float* fir, const float* in, float* out,
                                      void* stream);
typedef struct {
    int rows;             /* fold rows of one loop */
    int rnn_dims;         /* R: a multiple of 128, at most 640 */
    int fc_dims;          /* a multiple of 128, at most 2048 */
    int n_out;            /* fc3 outputs: RAW 2^bits (2..2048 classes), MOL 3 x mixtures (mixtures <= 32) */
    int mode;             /* B200TTS_WAVERNN_RAW / _MOL */
    int fold_len;         /* steps of a fold row: the row length of the uniform tape and of the output */
} b200tts_wavernn_shape;
/* fp32, row-major, on the device.  The loop multiplies bf16 copies of w_hh1, w_ih2x, w_hh2, w_fc1x, w_fc2x and w_fc3. */
typedef struct {
    const float* w_hh1;   /* rnn1.weight_hh_l0 [3R, R] */
    const float* b_hh1;   /* [3R] */
    const float* u1;      /* rnn1.weight_ih_l0 . I.weight[:, 0] [3R]: the previous sample's share of GRU1's input gates */
    const float* w_prev;  /* I.weight[:, 0] [R] */
    const float* w_ih2x;  /* rnn2.weight_ih_l0[:, :R] [3R, R] */
    const float* w_hh2;   /* [3R, R] */
    const float* b_hh2;   /* [3R] */
    const float* w_fc1x;  /* fc1.weight[:, :R] [fc, R] */
    const float* w_fc2x;  /* fc2.weight[:, :fc] [fc, fc] */
    const float* w_fc3;   /* [n_out, fc] */
    const float* b_fc3;   /* [n_out] */
} b200tts_wavernn_params;
/* The products of one chunk of steps that do not depend on the previous sample, [nsteps, rows, width] fp32:
 *   c = I.weight[:, 1:] . [mel, a1] + I.bias (R);  g1 = rnn1.weight_ih_l0 . c + b_ih1 (3R);  c2 = rnn2.weight_ih_l0[:, R:] . a2 + b_ih2 (3R);
 *   p1 = fc1.weight[:, R:] . a3 + fc1.bias (fc);  p2 = fc2.weight[:, fc:] . a4 + fc2.bias (fc). */
typedef struct { const float *c, *g1, *c2, *p1, *p2; } b200tts_wavernn_cond;
/* Host only: the loop workspace (packed bf16 weights, state, activation rows, grid barrier); 0 for an invalid shape (message set). */
size_t b200tts_wavernn_workspace_bytes(const b200tts_wavernn_shape* shape);
/* Packs the weights into the workspace (256-byte aligned) and zeroes the state (h1 = h2 = 0, previous sample 0) and the abort flag. */
int b200tts_wavernn_prepare(const b200tts_wavernn_shape* shape, const b200tts_wavernn_params* params, void* workspace, size_t workspace_bytes,
                            void* stream);
/* Steps [t0, t0 + nsteps) of every row, one cooperative launch of 128 CTAs (B200TTS_ERR_INVALID when they cannot be co-resident), carrying
 * the state in the workspace from the previous call.  Per step: x = c + w_prev prev; h1 = GRU(x, h1); x += h1; h2 = GRU([x, a2], h2); x += h2;
 * x = relu(fc1 [x, a3]); x = relu(fc2 [x, a4]); logits = fc3 x (torch GRU gate order r, z, n).  Sampling from the uniform tape
 * uniforms [rows, fold_len, U]: RAW (U = 1): k = the smallest class whose softmax CDF exceeds u, sample 2k / (n_out - 1) - 1; MOL
 * (U = mixtures + 1): each u mapped to 1e-5 + (1 - 2e-5) u, the component argmax(logit - log(-log u_j)), sample mean + exp(max(log_scale,
 * log 1e-14)) (log u - log(1 - u)) clamped to [-1, 1].  The sample is the next step's prev and goes to out[row, t] ([rows, fold_len]).
 * dbg (NULL: off) [nsteps, rows, 4R + 2 fc + n_out] receives each step's h1, bf16(x after GRU1), h2, bf16(x after GRU2), bf16(y1),
 * bf16(y2) and the logits.  A grid-barrier timeout (about 2 s) raises the abort flag and ends the launch: see b200tts_wavernn_aborted. */
int b200tts_wavernn_run(const b200tts_wavernn_shape* shape, const b200tts_wavernn_params* params, const b200tts_wavernn_cond* cond, int t0,
                        int nsteps, const float* uniforms, float* out, float* dbg, void* workspace, size_t workspace_bytes, void* stream);
/* A stream of unknown length: nsteps (at most shape->fold_len) more steps of every row after the t steps run since the last prepare, from the
 * state left in the workspace, exactly as b200tts_wavernn_run would run steps [t, t + nsteps).  uniforms [rows, nsteps, U] and out
 * [rows, nsteps] hold this call's steps only; cond as for b200tts_wavernn_run. */
int b200tts_wavernn_run_stream(const b200tts_wavernn_shape* shape, const b200tts_wavernn_params* params, const b200tts_wavernn_cond* cond,
                               long long t, int nsteps, const float* uniforms, float* out, void* workspace, size_t workspace_bytes, void* stream);
/* Concurrent streams, one per row of one loop: row r has run row_t[r] steps since it was last reset (or prepared) and runs row_n[r] (0 to
 * nsteps) more in this call, exactly as b200tts_wavernn_run_stream would run them on that row alone: its step i reads cond[i, r],
 * uniforms[r, i] and writes out[r, i], with the h1 / h2 slot parity of step row_t[r] + i.  Past its budget a row writes nothing (state,
 * previous sample, activation rows and out columns keep their values).  Only the first active_rows rows (at most shape->rows) are computed;
 * cond is [nsteps, active_rows, width], uniforms [active_rows, nsteps, U], out [active_rows, nsteps]; nsteps at most shape->fold_len.
 * row_t int64, row_n int32, both [active_rows] on the device. */
int b200tts_wavernn_run_rows(const b200tts_wavernn_shape* shape, const b200tts_wavernn_params* params, const b200tts_wavernn_cond* cond,
                             const int64_t* row_t, const int32_t* row_n, int active_rows, int nsteps, const float* uniforms, float* out,
                             void* workspace, size_t workspace_bytes, void* stream);
/* Zeroes h1, h2, both h1 / h2 activation slots and the previous sample of the `count` listed rows (host int32, each in [0, shape->rows)),
 * as b200tts_wavernn_prepare leaves them, so that a row can start a new stream without a prepare. */
int b200tts_wavernn_reset_rows(const b200tts_wavernn_shape* shape, void* workspace, size_t workspace_bytes, const int32_t* rows, int count,
                               void* stream);
/* Synchronises the stream and sets *aborted to the loop's abort flag (nonzero: a launch since the last prepare timed out). */
int b200tts_wavernn_aborted(const b200tts_wavernn_shape* shape, const void* workspace, size_t workspace_bytes, int* aborted, void* stream);
/* Optional de-emphasis of the loop's folded samples, in place, before b200tts_wavernn_unfold: each of `rows` rows of `len` samples is
 * mu-law decoded when mu > 0 (fp64, then fp32; pass mu = 0 to unfold afterwards), then filtered by lfilter([1], [1, -a]) on the Griffin-Lim
 * de-emphasis scan (fp32, without its normalisation).  a in (-1, 1); a = 0 only decodes. */
int b200tts_wavernn_deemphasis(int rows, int len, int mu, float a, float* y, void* stream);
/* Utterance b's (F_b - 1) hop samples at wave + wave_off[b] from its folds y[row_off[b] .. row_off[b + 1]) ([rows, target + 2 overlap]):
 * mu-law decoded when mu > 0 (sign(y) / mu ((1 + mu)^|y| - 1)), the first and last `overlap` samples of each fold multiplied by
 * [overlap / 2 zeros, sqrt(0.5 (1 + t))] and [sqrt(0.5 (1 - t)), zeros] (t = linspace(-1, 1, overlap - overlap / 2)), overlap-added in fold
 * order, and the last 20 hop samples multiplied by linspace(1, 0, 20 hop).  fp64 arithmetic, fp32 output; total = sum (F_b - 1) hop. */
int b200tts_wavernn_unfold(int B, int hop, int target, int overlap, int mu, const int32_t* frames, const int32_t* row_off, const int64_t* wave_off,
                           long long total, const float* y, float* wave, void* stream);
/* One stream of b200tts_wavernn_unfold_streams: the output positions [q0, q1) of its utterance, written at wave + wave_off (each stream right
 * after the previous one, the first at 0).  Fold f of the utterance (f in [fold0, fold0 + nfolds), every fold that covers a position of the
 * range) reads its samples through source entry src + f - fold0. */
typedef struct {
    long long q0, q1, wave_off;
    int frames;           /* F once it is known (the fade-out lands on the 20 hops before (F - 1) hop; q1 <= (F - 1) hop), 0 while unknown */
    int fold0, nfolds, src;
} b200tts_wavernn_unfold_stream;
/* Incremental unfold of up to B200TTS_WAVERNN_MAX_STREAMS folded streams in one launch, with b200tts_wavernn_unfold's fp64 arithmetic (the
 * same device functions): position q of a stream sums, over the folds f with 0 <= j = q - f (target + overlap) < target + 2 overlap in
 * ascending order, fold f's sample j, mu-law decoded when mu > 0 and cross-faded; an absent fold (base[e] < 0) adds nothing.  Times the
 * linear fade-out when frames > 0.  Fold sample j of source entry e is y[base[e] + j mod period[e]] (a slot of pool-owned storage; period
 * >= 1).  So the positions of an utterance whose folds all exist, cut into ranges of any size, equal b200tts_wavernn_unfold of the whole
 * utterance bit for bit.  streams: host descriptors, checked without a device; base (int64) and period (int32): nsrc entries on the
 * device; total = the sum of q1 - q0. */
int b200tts_wavernn_unfold_streams(int nstreams, int hop, int target, int overlap, int mu, const b200tts_wavernn_unfold_stream* streams,
                                   const int64_t* base, const int32_t* period, int nsrc, long long total, const float* y, float* wave,
                                   void* stream);

/* ---- WaveRNN training: the teacher-forced forward, the loss and the backward ----
 * The MelResNet, the input products of the GRUs, the fully connected layers and every weight gradient run on the convolution-block and
 * GEMM entry points (they follow the precision mode); these entry points add the GRU sequence loops (fp32 in both precision modes), the
 * adjoints of the upsampling layers and of the aux stretch, and the losses.  All fp32, row-major, on the device, stream-ordered. */
typedef struct {
    int B;                /* utterances: 1 to 64 */
    int T;                /* steps: 1 to 4400 (16 hops of 275 samples) */
    int R;                /* hidden size: a multiple of 128, at most 640 */
} b200tts_gru_seq_shape;
/* Host only: bytes of the forward's saved state ([B, T, 4R]: r, z, n, W_hn h + b_hn of every step) and of the loops' workspace (grid
 * barrier, abort flag, the reverse loop's carry); 0 for an invalid shape (message set).  The workspace must be 256-byte aligned and zeroed by
 * the caller before its first loop; after that, loops of one shape (both GRUs of a model, forward and reverse) may share it in stream
 * order, and its abort flag collects a timeout of any of them. */
size_t b200tts_gru_seq_saved_bytes(const b200tts_gru_seq_shape* shape);
size_t b200tts_gru_seq_workspace_bytes(const b200tts_gru_seq_shape* shape);
/* torch.nn.GRU (batch_first, one layer, gate order r, z, n, h0 = 0) given its input products gi = x W_ih^T + b_ih [B, T, 3R]:
 * r = s(gi_r + W_hr h + b_hr), z = s(gi_z + W_hz h + b_hz), n = tanh(gi_n + r (W_hn h + b_hn)), h' = (1 - z) n + z h.  h [B, T, R]: every
 * step's output.  One cooperative launch of 128 CTAs (B200TTS_ERR_INVALID when they cannot be co-resident); a grid-barrier timeout
 * (about 2 s) raises the abort flag and ends the launch: see b200tts_gru_seq_aborted.  The flag is never cleared by the loops. */
int b200tts_gru_seq_forward(const b200tts_gru_seq_shape* shape, const float* gi, const float* w_hh, const float* b_hh, float* h, void* saved,
                            void* workspace, size_t workspace_bytes, void* stream);
/* The reverse of b200tts_gru_seq_forward (same w_hh, h and saved state) for the external gradient dh_ext [B, T, R] of every step's output:
 * dgi [B, T, 3R] = the gradient of gi = [dr^, dz^, dn^] and dgh [B, T, 3R] = the gradient of W_hh h + b_hh = [dr^, dz^, r dn^] (both
 * overwritten), from which the caller forms d W_ih, d b_ih, d x, d W_hh = sum_t dgh_t^T h_{t-1} and d b_hh.  dh_dbg (NULL: off) [B, T, R]
 * receives every step's total dh = dh_ext + z dh_next + W_hh^T dgh_next.  One cooperative launch of 128 CTAs. */
int b200tts_gru_seq_backward(const b200tts_gru_seq_shape* shape, const float* w_hh, const float* h, const void* saved, const float* dh_ext,
                             float* dgi, float* dgh, float* dh_dbg, void* workspace, size_t workspace_bytes, void* stream);
/* Synchronises the stream and sets *aborted to the loops' abort flag (nonzero: a loop on this workspace timed out since it was zeroed). */
int b200tts_gru_seq_aborted(const b200tts_gru_seq_shape* shape, const void* workspace, size_t workspace_bytes, int* aborted, void* stream);
/* Enqueues a copy of the loops' abort flag (one int) to dst (pinned host or device memory) on the stream, without synchronising: the caller
 * reads *dst once the work enqueued before it has completed (an event recorded after the call).  For a training step captured in a CUDA
 * graph, whose flag is read after the replay instead of inside it. */
int b200tts_gru_seq_abort_flag_copy(const b200tts_gru_seq_shape* shape, const void* workspace, size_t workspace_bytes, int* dst, void* stream);
/* Training windows from a corpus in device memory, one launch: fatchord's collate_vocoder with explicit offsets.
 *   mels: fp32 [feat, total_frames], the utterances' mels side by side (utterance u's frames from frame_start[u]);
 *   labels: uint16 [sum N_u] (utterance u's samples from sample_start[u]); frame_start, sample_start: int64, one per utterance;
 *   table: int32 [B, 2] of (utterance u, mel offset o);
 *   m [B, feat, mel_win] = mel_u[:, o : o + mel_win] with mel_win = seq_len / hop + 2 pad; the label window lab = labels_u[(o + pad) hop :
 *   (o + pad) hop + seq_len + 1]; x [B, seq_len] fp32 = label_2_float(lab[:seq_len], MOL ? 16 : bits); y [B, seq_len] = lab[1:] as int64
 *   (RAW) or label_2_float(lab[1:], 16) as fp32 (MOL).  label_2_float(v, b) = 2 v / (2^b - 1) - 1, each fp32 operation IEEE-rounded.
 * Limits, checked on the host: mode RAW or MOL, bits 1 to 16, B 1 to 64, seq_len a positive multiple of the hop and at most 16 hops, pad 0 to
 * 64, feat 1 to 1024.  The table is NOT checked: every window must lie inside its utterance's mel and labels (the caller validates it). */
int b200tts_wavernn_cut_windows(int mode, int bits, int B, int feat, int seq_len, int pad, int hop, const float* mels, long long total_frames,
                                const int64_t* frame_start, const uint16_t* labels, const int64_t* sample_start, const int32_t* table, float* x,
                                void* y, float* m, void* stream);
/* The adjoint of b200tts_wavernn_upsample_layer (C, len, scale, fir, in as there) for dout [C, len scale]: din [C, len] (overwritten; NULL:
 * not formed) and dfir [2 scale + 1] += the FIR gradient (NULL: not formed; needs `in` and the workspace, summed in a fixed order). */
size_t b200tts_wavernn_upsample_layer_backward_workspace_bytes(int C, int len, int scale);
int b200tts_wavernn_upsample_layer_backward(int C, int len, int scale, const float* fir, const float* in, const float* dout, float* din,
                                            float* dfir, void* workspace, size_t workspace_bytes, void* stream);
/* The adjoint of the aux stretch aux_up[b, t, c] = aux[b, t / hop, c]: daux[b, f, c] = sum_{q < hop} dup[b, f hop + q, c] (overwritten).
 * dup [B, F hop, C], daux [B, F, C]. */
int b200tts_wavernn_stretch_backward(int B, int F, int C, int hop, const float* dup, float* daux, void* stream);
/* Mean loss over N rows of logits [N, n_out] into loss[0], and dlogits [N, n_out] = its gradient (both overwritten), summed in a fixed order.
 * RAW: cross entropy against int32 labels [N] (a label outside [0, n_out) gives NaN).  MOL: fatchord's discretized_mix_logistic_loss
 * (65536 classes, log scales clamped below at log 1e-14) against fp32 targets [N] in [-1, 1]; n_out = 3 x mixtures. */
size_t b200tts_wavernn_loss_workspace_bytes(long long N);
/* out[c] += sum over the rows of x [rows, cols] (fp32, summed in a fixed order of 64 row chunks): the bias gradients of the GRUs. */
size_t b200tts_column_sum_workspace_bytes(int cols);
int b200tts_column_sum(long long rows, int cols, const float* x, float* out, void* workspace, size_t workspace_bytes, void* stream);
int b200tts_wavernn_loss(int mode, long long N, int n_out, const float* logits, const void* target, float* loss, float* dlogits, void* workspace,
                         size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200TTS_H_ */
