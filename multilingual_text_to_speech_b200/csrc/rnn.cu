// Packed bidirectional LSTM of the vanilla encoder (reference modules/encoder.py:33,41-44: nn.LSTM on a
// pack_padded_sequence).  Semantics restated: zero initial state, the state of utterance b is frozen
// and its output is exactly zero at positions >= lengths[b]; the reverse direction therefore starts at
// each utterance's own last token.  Input projections are time-batched GEMMs; the recurrence is a
// per-step GEMM + the shared LSTM cell kernel (decoder_fwd.cu / decoder_bwd.cu).
#include "decoder_internal.cuh"

namespace b200tts {

namespace {

inline int grid_for(size_t n) {
    size_t g = (n + 255) / 256;
    return (int)(g > NUM_SMS * 16 ? NUM_SMS * 16 : (g < 1 ? 1 : g));
}

// xp[dir][j, b, :] = x[b, t(dir, j), :]   with t(0, j) = j, t(1, j) = L-1-j
__global__ void to_processing_order_kernel(float* __restrict__ xp, const float* __restrict__ x, int B, int L, int E) {
    const size_t per = (size_t)L * B * E;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < 2 * per; idx += (size_t)gridDim.x * blockDim.x) {
        const int dir = idx / per;
        const size_t r = idx % per;
        const int e = r % E, b = (r / E) % B, j = r / ((size_t)E * B);
        const int t = dir ? L - 1 - j : j;
        xp[idx] = x[((size_t)b * L + t) * E + e];
    }
}
// dx[b, t, :] = dxp[0][t, b, :] + dxp[1][L-1-t, b, :]
__global__ void from_processing_order_kernel(float* __restrict__ dx, const float* __restrict__ dxp, int B, int L, int E) {
    const size_t per = (size_t)L * B * E;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < per; idx += (size_t)gridDim.x * blockDim.x) {
        const int e = idx % E, t = (idx / E) % L, b = idx / ((size_t)E * L);
        dx[idx] = dxp[((size_t)t * B + b) * E + e] + dxp[per + ((size_t)(L - 1 - t) * B + b) * E + e];
    }
}
__global__ void colsum_add2_kernel(float* __restrict__ d1, float* __restrict__ d2, const float* __restrict__ src, size_t rows, int cols) {
    __shared__ float sm[8][33];
    const int c = blockIdx.x * 32 + threadIdx.x;
    float acc = 0.f;
    if (c < cols)
        for (size_t r = threadIdx.y; r < rows; r += 8) acc += src[r * cols + c];
    sm[threadIdx.y][threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.y == 0 && c < cols) {
        float s = 0.f;
        for (int j = 0; j < 8; ++j) s += sm[j][threadIdx.x];
        d1[c] += s; d2[c] += s;
    }
}

struct RnnLayout {
    size_t xp, gates, hs, cs, bsum, total;        // saved
    size_t part, dg, dxp, dc, dhz, scratch, wtotal;   // workspace
    int split, split_b;
};
RnnLayout rnn_layout(const b200tts_bilstm_shape& s) {
    RnnLayout l;
    const size_t B = s.B, L = s.L, E = s.E, H = s.H;
    size_t off = 0;
    auto take = [&](size_t n) { size_t o = off; off = align_up_sz(off + n, 64); return o; };
    l.xp = take(2 * L * B * E);
    l.gates = take(2 * L * B * 4 * H);
    l.hs = take(2 * (L + 1) * B * H);
    l.cs = take(2 * (L + 1) * B * H);
    l.bsum = take(2 * 4 * H);
    l.total = off;
    off = 0;
    l.split = pick_splitk(s.B, 4 * s.H, s.H);
    l.split_b = pick_splitk(s.B, s.H, 4 * s.H);
    const size_t p1 = (size_t)l.split * B * 4 * H, p2 = (size_t)l.split_b * B * H;
    l.part = take(p1 > p2 ? p1 : p2);
    l.dg = take(2 * L * B * 4 * H);
    l.dxp = take(2 * L * B * E);
    l.dc = take(B * H);
    l.dhz = take(B * H);
    l.scratch = take((size_t)2 * 1024 * 1024);
    l.wtotal = off;
    return l;
}

}  // namespace

size_t bilstm_saved_floats(const b200tts_bilstm_shape& s) { return rnn_layout(s).total; }
size_t bilstm_workspace_floats(const b200tts_bilstm_shape& s) { return rnn_layout(s).wtotal; }

int bilstm_forward_impl(const b200tts_bilstm_shape& s, const b200tts_bilstm_params& w, const float* x, const int* lengths, float* out,
                        float* saved, float* ws, cudaStream_t st) {
    B200_REQUIRE(s.B > 0 && s.L > 0 && s.E > 0 && s.H > 0, "bilstm: non-positive dimension");
    const RnnLayout l = rnn_layout(s);
    const int B = s.B, L = s.L, E = s.E, H = s.H;
    const size_t BH = (size_t)B * H, B4H = 4 * BH;
    const bool persist = bilstm_persist_supported(s);
    to_processing_order_kernel<<<grid_for(2 * (size_t)L * B * E), 256, 0, st>>>(saved + l.xp, x, B, L, E);
    B200_LAUNCH_CHECK();
    for (int dir = 0; dir < 2; ++dir) {
        const float* w_ih = dir ? w.w_ih_reverse : w.w_ih; const float* w_hh = dir ? w.w_hh_reverse : w.w_hh;
        const float* b_ih = dir ? w.b_ih_reverse : w.b_ih; const float* b_hh = dir ? w.b_hh_reverse : w.b_hh;
        float* bsum = saved + l.bsum + (size_t)dir * 4 * H;
        B200_TRY(launch_add_vec(bsum, b_ih, b_hh, 4 * H, st));
        float* gates = saved + l.gates + (size_t)dir * L * B4H;
        float* hs = saved + l.hs + (size_t)dir * (L + 1) * BH;
        float* cs = saved + l.cs + (size_t)dir * (L + 1) * BH;
        GemmDesc g;
        g.A = saved + l.xp + (size_t)dir * L * B * E; g.lda = E; g.B = w_ih; g.ldb = E; g.transB = 1; g.C = gates; g.ldc = 4 * H;
        g.bias = bsum; g.M = L * B; g.N = 4 * H; g.K = E;
        B200_TRY(gemm_run(g, st));
        if (persist) continue;           // the recurrence of both directions runs in ONE persistent launch below
        B200_TRY(launch_fill(hs, 0.f, BH, st));
        B200_TRY(launch_fill(cs, 0.f, BH, st));
        for (int j = 0; j < L; ++j) {
            const int t = dir ? L - 1 - j : j;
            GemmDesc r;
            r.A = hs + (size_t)j * BH; r.lda = H; r.B = w_hh; r.ldb = H; r.transB = 1; r.M = B; r.N = 4 * H; r.K = H;
            r.splitk = l.split; r.partial = ws + l.part; r.keep_partials = 1;
            if (r.splitk == 1) { r.C = ws + l.part; r.ldc = 4 * H; r.keep_partials = 0; r.partial = nullptr; }
            B200_TRY(gemm_run(r, st));
            CellFwdArgs ca{};
            ca.xproj = gates + (size_t)j * B4H; ca.gates = gates + (size_t)j * B4H;
            ca.part = ws + l.part; ca.nsplit = l.split; ca.part_stride = B4H;
            ca.c_prev = cs + (size_t)j * BH; ca.h_prev = hs + (size_t)j * BH; ca.ld_hprev = H;
            ca.c_out = cs + (size_t)(j + 1) * BH; ca.h_out = hs + (size_t)(j + 1) * BH; ca.ld_hout = H;
            ca.kind = B200TTS_CELL_DROPOUT; ca.training = 0; ca.rate_h = 0.f; ca.rate_c = 0.f;
            ca.y_out = out + (size_t)t * 2 * H + (size_t)dir * H; ca.ld_y = L * 2 * H;
            ca.lengths = lengths; ca.step = t; ca.B = B; ca.D = H;
            B200_TRY(launch_cell_fwd(ca, st));
        }
    }
    if (persist)
        B200_TRY(bilstm_persist_forward(s, w.w_hh, w.w_hh_reverse, saved + l.gates, saved + l.hs, saved + l.cs, out, lengths, st));
    return B200TTS_OK;
}

int bilstm_backward_impl(const b200tts_bilstm_shape& s, const b200tts_bilstm_params& w, const int* lengths, const float* saved,
                         const float* dout, float* dx, const b200tts_bilstm_params& dw, float* ws, cudaStream_t st) {
    const RnnLayout l = rnn_layout(s);
    const int B = s.B, L = s.L, E = s.E, H = s.H;
    const size_t BH = (size_t)B * H, B4H = 4 * BH;
    const bool persist = bilstm_persist_supported(s);
    for (int dir = 0; dir < 2; ++dir) {
        const float* w_ih = dir ? w.w_ih_reverse : w.w_ih; const float* w_hh = dir ? w.w_hh_reverse : w.w_hh;
        float* dw_ih = dir ? dw.w_ih_reverse : dw.w_ih; float* dw_hh = dir ? dw.w_hh_reverse : dw.w_hh;
        float* db_ih = dir ? dw.b_ih_reverse : dw.b_ih; float* db_hh = dir ? dw.b_hh_reverse : dw.b_hh;
        const float* gates = saved + l.gates + (size_t)dir * L * B4H;
        const float* hs = saved + l.hs + (size_t)dir * (L + 1) * BH;
        const float* cs = saved + l.cs + (size_t)dir * (L + 1) * BH;
        float* dg = ws + l.dg + (size_t)dir * L * B4H;
        if (persist && dir == 0)         // gate gradients of BOTH directions in one persistent launch
            B200_TRY(bilstm_persist_backward(s, w.w_hh, w.w_hh_reverse, saved + l.gates, saved + l.cs, dout, ws + l.dg, lengths, st));
        for (int j = L - 1; j >= 0 && !persist; --j) {
            const int t = dir ? L - 1 - j : j;
            CellBwdArgs ca{};
            ca.gates = gates + (size_t)j * B4H; ca.c_prev = cs + (size_t)j * BH;
            ca.dh_static = dout + (size_t)t * 2 * H + (size_t)dir * H; ca.ld_dhs = L * 2 * H;
            ca.part = ws + l.part; ca.nsplit = l.split_b; ca.part_stride = BH; ca.ld_part = H; ca.part_col0 = 0;
            ca.dc_state = ws + l.dc; ca.dhz_state = ws + l.dhz;
            ca.kind = B200TTS_CELL_DROPOUT; ca.training = 0; ca.rate_h = 0.f; ca.rate_c = 0.f;
            ca.dgates = dg + (size_t)j * B4H; ca.lengths = lengths; ca.step = t; ca.B = B; ca.D = H; ca.last = (j == L - 1);
            B200_TRY(launch_cell_bwd(ca, st));
            if (j > 0) {
                GemmDesc r;
                r.A = ca.dgates; r.lda = 4 * H; r.B = w_hh; r.ldb = H; r.transB = 0; r.M = B; r.N = H; r.K = 4 * H;
                r.splitk = l.split_b; r.partial = ws + l.part; r.keep_partials = 1;
                if (r.splitk == 1) { r.C = ws + l.part; r.ldc = H; r.keep_partials = 0; r.partial = nullptr; }
                B200_TRY(gemm_run(r, st));
            }
        }
        const float* xp = saved + l.xp + (size_t)dir * L * B * E;
        GemmDesc a;   // dW_ih += dg^T . x
        a.A = dg; a.lda = 4 * H; a.transA = 1; a.B = xp; a.ldb = E; a.C = dw_ih; a.ldc = E; a.beta = 1.f; a.M = 4 * H; a.N = E; a.K = L * B;
        B200_TRY(gemm_run_auto(a, ws + l.scratch, (size_t)2 * 1024 * 1024, st));
        GemmDesc b;   // dW_hh += dg^T . h_prev
        b.A = dg; b.lda = 4 * H; b.transA = 1; b.B = hs; b.ldb = H; b.C = dw_hh; b.ldc = H; b.beta = 1.f; b.M = 4 * H; b.N = H; b.K = L * B;
        B200_TRY(gemm_run_auto(b, ws + l.scratch, (size_t)2 * 1024 * 1024, st));
        dim3 blk(32, 8);
        colsum_add2_kernel<<<cdiv(4 * H, 32), blk, 0, st>>>(db_ih, db_hh, dg, (size_t)L * B, 4 * H);
        B200_LAUNCH_CHECK();
        GemmDesc c;   // dx (processing order) = dg . W_ih
        c.A = dg; c.lda = 4 * H; c.B = w_ih; c.ldb = E; c.transB = 0; c.C = ws + l.dxp + (size_t)dir * L * B * E; c.ldc = E;
        c.M = L * B; c.N = E; c.K = 4 * H;
        B200_TRY(gemm_run(c, st));
    }
    if (dx) {
        from_processing_order_kernel<<<grid_for((size_t)L * B * E), 256, 0, st>>>(dx, ws + l.dxp, B, L, E);
        B200_LAUNCH_CHECK();
    }
    return B200TTS_OK;
}

}  // namespace b200tts
