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
 * Returns the number of values written (26 when n >= 26), 0 for a rejected shape. */
int b200tts_debug_decoder_views(const b200tts_decoder_shape* shape, size_t* out, int n);

int b200tts_decoder_forward(const b200tts_decoder_shape* shape, const b200tts_decoder_params* params,
                            const b200tts_decoder_inputs* in, const b200tts_decoder_outputs* out, void* workspace,
                            size_t workspace_bytes, void* stream);

/* Decoder state carried between chunks of one decode (all device pointers, fp32; every field required): lets a caller decode in
 * chunks of T frames and stop early, as the reference's inference loop does (Decoder.inference, tacotron2.py:201-207,216-219). */
typedef struct {
    float* att_h; float* att_c; /* [B, D] attention-LSTM state */
    float* gen_h; float* gen_c; /* [B, D] generator-LSTM state */
    float* context;             /* [B, M] last attention context */
    float* cum_weights;         /* [B, L] cumulative attention weights (forward attention: the last alignment = alpha) */
    float* frame;               /* [B, N] last predicted frame, the last of the last step's R (input of the next free-running step) */
} b200tts_decoder_state;

/* b200tts_decoder_forward on a chunk of T frames: `first` != 0 starts from the zero state (tacotron2.py:164-168), otherwise from
 * `state`; on return `state` holds the state after the chunk's last step.  Uses the per-step kernels (any precision mode).  A chunk
 * holds whole steps: T % R != 0 is rejected. */
int b200tts_decoder_forward_chunk(const b200tts_decoder_shape* shape, const b200tts_decoder_params* params,
                                  const b200tts_decoder_inputs* in, const b200tts_decoder_outputs* out, b200tts_decoder_state* state,
                                  int first, void* workspace, size_t workspace_bytes, void* stream);

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
 * [NB, G*Cout, L] or NULL.  out [NB, G*Cf, L] with Cf = highway ? Cout/2 : Cout.                     */
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

/* ---- loss: TacotronLoss.forward, modules/tacotron2.py:439-485 (guided attention :439-457 in closed form) ----
 * pre / post / targets [B, N, T]; stop (logits, padded positions already filled as in tacotron2.py:380) / stop_target [B, T]; alignment
 * [B, S, L] with S = ceil(T / R); lengths int32 [B].  losses[4] (device) = { 2*MSE(pre), MSE(post), BCEWithLogits(pos_weight)/(N+2),
 * guided attention }.  The guided term runs on the step grid: utterance b has ceil(target_lengths[b] / R) steps, which take the place of
 * its frame count in the weight and the division (R = 1: the reference's formula).                                                     */
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

/* ---- optimizer step on flat buffers: clip_grad_norm_ + torch.optim.Adam with coupled L2 decay (train.py:84-85, 260-271) ----
 * p, g, m, v: n fp32 elements each (the flat parameter buffer, the flat all-reduced gradient, Adam moments); g is overwritten with
 * the clipped gradient; max_norm <= 0 disables clipping; step counts from 1; scratch holds b200tts_adam_clip_scratch_floats()
 * floats, scratch[0] = gradient norm before clipping, scratch[1] = applied clip coefficient (device values after the call). */
size_t b200tts_adam_clip_scratch_floats(void);
int b200tts_adam_clip_step(float* p, float* g, float* m, float* v, size_t n, float lr, float beta1, float beta2, float eps,
                           float weight_decay, float max_norm, int step, float* scratch, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200TTS_H_ */
