// Fused TacotronLoss (reference modules/tacotron2.py:439-485): 2 x MSE(pre) + MSE(post) + pos-weighted stop BCE / (mels + 2) +
// guided attention, forward and backward.  The guided-attention weight  1 - exp(-(l / L_b - t / T_b)^2 / (2 g^2))  is evaluated in
// closed form per element: the reference's per-utterance Python loop (meshgrid, :449-451) and its [B, T, L] weight tensor never exist.
// Deterministic: block partials in a fixed grid, summed in a fixed order by one block (no atomics).
#include "common.cuh"

namespace b200tts {

namespace {

constexpr int LT = 256;
constexpr int LOSS_BLOCKS = NUM_SMS * 4;

struct LossArgs {
    int B, N, T, L;
    int R, S;               // frames per decoder step; alignment rows S = ceil(T / R) (the guided term's step grid)
    float inv2g2, pos_weight;
    int guided;
    const float* pre; const float* pre_t; const float* post; const float* post_t;
    const float* stop; const float* stop_t; const float* align;
    const int* text_len; const int* target_len;
};

__device__ __forceinline__ float stop_bce(float x, float y, float pw) {
    // F.binary_cross_entropy_with_logits(x, y, pos_weight = pw): (1 - y) x + (1 + (pw - 1) y) softplus(-x)
    const float sp = log1pf(expf(-fabsf(x))) + fmaxf(-x, 0.f);
    return (1.f - y) * x + (1.f + (pw - 1.f) * y) * sp;
}
__device__ __forceinline__ float guided_weight(int t, int l, int Tb, int Lb, float inv2g2) {
    const float d = (float)l / (float)Lb - (float)t / (float)Tb;
    return 1.f - expf(-d * d * inv2g2);
}

// four consecutive floats: one 16-byte load when the caller's buffers allow it, four scalar loads otherwise (same arithmetic after)
template <bool VEC>
__device__ __forceinline__ float4 load4(const float* p) {
    if constexpr (VEC) return *reinterpret_cast<const float4*>(p);
    else return make_float4(p[0], p[1], p[2], p[3]);
}

template <bool VEC>
__global__ void __launch_bounds__(LT) loss_partial_kernel(const LossArgs a, float* __restrict__ partial) {
    __shared__ float red[4][LT / 32];
    const size_t gid = (size_t)blockIdx.x * LT + threadIdx.x, gstride = (size_t)gridDim.x * LT;
    float s_pre = 0.f, s_post = 0.f, s_stop = 0.f, s_att = 0.f;
    const size_t nmel = (size_t)a.B * a.N * a.T;
    for (size_t i = gid * 4; i < nmel; i += gstride * 4) {
        if (i + 3 < nmel) {
            const float4 p = load4<VEC>(a.pre + i), pt = load4<VEC>(a.pre_t + i);
            const float4 q = load4<VEC>(a.post + i), qt = load4<VEC>(a.post_t + i);
            s_pre += (p.x - pt.x) * (p.x - pt.x) + (p.y - pt.y) * (p.y - pt.y) + (p.z - pt.z) * (p.z - pt.z) + (p.w - pt.w) * (p.w - pt.w);
            s_post += (q.x - qt.x) * (q.x - qt.x) + (q.y - qt.y) * (q.y - qt.y) + (q.z - qt.z) * (q.z - qt.z) + (q.w - qt.w) * (q.w - qt.w);
        } else {
            for (size_t j = i; j < nmel; ++j) {
                const float d0 = a.pre[j] - a.pre_t[j], d1 = a.post[j] - a.post_t[j];
                s_pre += d0 * d0; s_post += d1 * d1;
            }
        }
    }
    const size_t nstop = (size_t)a.B * a.T;
    for (size_t i = gid; i < nstop; i += gstride) s_stop += stop_bce(a.stop[i], a.stop_t[i], a.pos_weight);
    if (a.guided) {
        // one (b, step t) row per warp iteration: lanes stride over the text positions.  Utterance b has Tb = ceil(target_len / R) steps.
        const int lane = threadIdx.x & 31;
        const size_t wid = gid >> 5, wstride = gstride >> 5, nrows = (size_t)a.B * a.S;
        for (size_t row = wid; row < nrows; row += wstride) {
            const int b = (int)(row / a.S), t = (int)(row % a.S);
            const int Tb = (a.target_len[b] + a.R - 1) / a.R, Lb = min(a.text_len[b], a.L);
            if (t >= Tb) continue;
            const float* al = a.align + row * a.L;
            float acc = 0.f;
            for (int l = lane; l < Lb; l += 32) acc += guided_weight(t, l, Tb, Lb, a.inv2g2) * al[l];
            s_att += acc / (float)Tb;
        }
    }
    float v[4] = {s_pre, s_post, s_stop, s_att};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        v[k] = warp_sum(v[k]);
        if ((threadIdx.x & 31) == 0) red[k][threadIdx.x >> 5] = v[k];
    }
    __syncthreads();
    if (threadIdx.x < 4) {
        float t = 0.f;
        for (int w = 0; w < LT / 32; ++w) t += red[threadIdx.x][w];
        partial[(size_t)blockIdx.x * 4 + threadIdx.x] = t;
    }
}

__global__ void loss_final_kernel(const float* __restrict__ partial, int nblocks, float* __restrict__ losses, float s_pre, float s_post,
                                  float s_stop, float s_att) {
    // double accumulation in a fixed order: the 4 terms are sums of up to 10^8 squares
    if (threadIdx.x < 4) {
        double t = 0.0;
        for (int b = 0; b < nblocks; ++b) t += (double)partial[(size_t)b * 4 + threadIdx.x];
        const float scale = threadIdx.x == 0 ? s_pre : threadIdx.x == 1 ? s_post : threadIdx.x == 2 ? s_stop : s_att;
        losses[threadIdx.x] = (float)(t * (double)scale);
    }
}

__global__ void __launch_bounds__(LT) loss_backward_kernel(const LossArgs a, const float* __restrict__ gl, float* __restrict__ d_pre,
                                                           float* __restrict__ d_post, float* __restrict__ d_stop, float* __restrict__ d_align,
                                                           float c_pre, float c_post, float c_stop, float c_att) {
    const size_t gid = (size_t)blockIdx.x * LT + threadIdx.x, gstride = (size_t)gridDim.x * LT;
    const float g_pre = gl[0] * c_pre, g_post = gl[1] * c_post, g_stop = gl[2] * c_stop, g_att = gl[3] * c_att;
    const size_t nmel = (size_t)a.B * a.N * a.T;
    for (size_t i = gid; i < nmel; i += gstride) {
        if (d_pre) d_pre[i] = g_pre * (a.pre[i] - a.pre_t[i]);
        if (d_post) d_post[i] = g_post * (a.post[i] - a.post_t[i]);
    }
    const size_t nstop = (size_t)a.B * a.T;
    if (d_stop)
        for (size_t i = gid; i < nstop; i += gstride) {
            const float x = a.stop[i], y = a.stop_t[i];
            const float sneg = 1.f / (1.f + expf(x));                 // sigmoid(-x)
            d_stop[i] = g_stop * ((1.f - y) - (1.f + (a.pos_weight - 1.f) * y) * sneg);
        }
    if (d_align) {
        const size_t nal = (size_t)a.B * a.S * a.L;
        for (size_t i = gid; i < nal; i += gstride) {
            const size_t row = i / a.L;
            const int l = (int)(i % a.L), b = (int)(row / a.S), t = (int)(row % a.S);
            const int Tb = (a.target_len[b] + a.R - 1) / a.R, Lb = min(a.text_len[b], a.L);
            d_align[i] = (a.guided && t < Tb && l < Lb) ? g_att * guided_weight(t, l, Tb, Lb, a.inv2g2) / (float)Tb : 0.f;
        }
    }
}

}  // namespace

static LossArgs make_args(const b200tts_loss_shape& s, const float* pre, const float* pre_t, const float* post, const float* post_t,
                          const float* stop, const float* stop_t, const float* align, const int* text_len, const int* target_len) {
    LossArgs a{};
    a.B = s.B; a.N = s.N; a.T = s.T; a.L = s.L;
    a.R = s.R > 0 ? s.R : 1; a.S = (s.T + a.R - 1) / a.R;
    a.inv2g2 = 1.f / (2.f * s.guided_g * s.guided_g); a.pos_weight = s.stop_pos_weight; a.guided = s.guided;
    a.pre = pre; a.pre_t = pre_t; a.post = post; a.post_t = post_t; a.stop = stop; a.stop_t = stop_t; a.align = align;
    a.text_len = text_len; a.target_len = target_len;
    return a;
}

}  // namespace b200tts
using namespace b200tts;

extern "C" {

size_t b200tts_loss_workspace_bytes(void) { return (size_t)LOSS_BLOCKS * 4 * sizeof(float); }

int b200tts_tacotron_loss_forward(const b200tts_loss_shape* shape, const float* pre, const float* pre_target, const float* post,
                                  const float* post_target, const float* stop, const float* stop_target, const float* alignment,
                                  const int32_t* text_lengths, const int32_t* target_lengths, float* losses, void* workspace, void* stream) {
    B200_REQUIRE(shape && pre && pre_target && post && post_target && stop && stop_target && text_lengths && target_lengths && losses && workspace,
                 "tacotron_loss_forward: null argument");
    const b200tts_loss_shape& s = *shape;
    B200_REQUIRE(alignment || !s.guided, "tacotron_loss_forward: guided attention needs the alignments");
    B200_TRY(require_device());
    B200_REQUIRE(s.B > 0 && s.N > 0 && s.T > 0 && s.L > 0 && s.R >= 0, "loss_forward: bad shape");
    B200_REQUIRE(!s.guided || s.guided_g > 0.f, "loss_forward: guided attention needs a positive variance");
    cudaStream_t st = (cudaStream_t)stream;
    float* ws = (float*)workspace;
    const LossArgs a = make_args(s, pre, pre_target, post, post_target, stop, stop_target, alignment, text_lengths, target_lengths);
    const uintptr_t addr_bits = reinterpret_cast<uintptr_t>(pre) | reinterpret_cast<uintptr_t>(pre_target) | reinterpret_cast<uintptr_t>(post) |
                                reinterpret_cast<uintptr_t>(post_target);
    if ((addr_bits & 15) == 0)
        loss_partial_kernel<true><<<LOSS_BLOCKS, LT, 0, st>>>(a, ws);
    else
        loss_partial_kernel<false><<<LOSS_BLOCKS, LT, 0, st>>>(a, ws);
    B200_LAUNCH_CHECK();
    const double nmel = (double)s.B * s.N * s.T, nstop = (double)s.B * s.T;
    loss_final_kernel<<<1, 32, 0, st>>>(ws, LOSS_BLOCKS, losses, (float)(2.0 / nmel), (float)(1.0 / nmel), (float)(1.0 / (nstop * (s.N + 2))),
                                        (float)(1.0 / s.B));
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_tacotron_loss_backward(const b200tts_loss_shape* shape, const float* pre, const float* pre_target, const float* post,
                                   const float* post_target, const float* stop, const float* stop_target, const int32_t* text_lengths,
                                   const int32_t* target_lengths, const float* grad_losses, float* d_pre, float* d_post, float* d_stop,
                                   float* d_alignment, void* stream) {
    B200_REQUIRE(shape && pre && pre_target && post && post_target && stop && stop_target && text_lengths && target_lengths && grad_losses,
                 "tacotron_loss_backward: null argument");
    B200_TRY(require_device());
    const b200tts_loss_shape& s = *shape;
    B200_REQUIRE(s.R >= 0, "loss_backward: bad shape");
    const LossArgs a = make_args(s, pre, pre_target, post, post_target, stop, stop_target, nullptr, text_lengths, target_lengths);
    const double nmel = (double)s.B * s.N * s.T, nstop = (double)s.B * s.T;
    loss_backward_kernel<<<NUM_SMS * 8, LT, 0, (cudaStream_t)stream>>>(a, grad_losses, d_pre, d_post, d_stop, d_alignment, (float)(4.0 / nmel),
                                                                   (float)(2.0 / nmel), (float)(1.0 / (nstop * (s.N + 2))), (float)(1.0 / s.B));
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // extern "C"
