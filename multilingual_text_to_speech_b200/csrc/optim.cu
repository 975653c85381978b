// Fused gradient clipping + Adam step on the flat parameter / gradient buffers (reference train.py:84-85, 260-271):
//   clip_grad_norm_(parameters, max_norm)  then  torch.optim.Adam(lr, weight_decay) with COUPLED L2 decay (not AdamW).
// Three launches whatever the number of parameter tensors: squared-norm partials, fixed-order finish, fused update.
#include "common.cuh"

namespace b200tts {

namespace {

constexpr int NORM_BLOCKS = NUM_SMS * 8;

__global__ void __launch_bounds__(256) sqnorm_partial_kernel(const float* __restrict__ g, size_t n, float* __restrict__ partial) {
    __shared__ float red[64];
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    const size_t n4 = n / 4;
    const float4* g4 = reinterpret_cast<const float4*>(g);
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        const float4 v = g4[i];
        a0 = fmaf(v.x, v.x, a0); a1 = fmaf(v.y, v.y, a1); a2 = fmaf(v.z, v.z, a2); a3 = fmaf(v.w, v.w, a3);
    }
    if (blockIdx.x == 0)
        for (size_t i = n4 * 4 + threadIdx.x; i < n; i += blockDim.x) a0 = fmaf(g[i], g[i], a0);
    const float s = block_sum((a0 + a1) + (a2 + a3), red);
    if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

// norm[0] = sqrt(sum of partials) (fixed order), norm[1] = clip coefficient min(1, max_norm / (norm + 1e-6)) (1 when max_norm <= 0)
__global__ void __launch_bounds__(256) sqnorm_finish_kernel(const float* __restrict__ partial, int nblk, float max_norm, float* __restrict__ norm) {
    __shared__ float red[64];
    float s = 0.f;
    for (int i = threadIdx.x; i < nblk; i += blockDim.x) s += partial[i];
    s = block_sum(s, red);
    if (threadIdx.x == 0) {
        const float nrm = sqrtf(s);
        norm[0] = nrm;
        float coef = 1.f;
        if (max_norm > 0.f) { coef = max_norm / (nrm + 1e-6f); coef = coef < 1.f ? coef : 1.f; }
        norm[1] = coef;
    }
}

__global__ void __launch_bounds__(256) adam_clip_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                                        size_t n, float lr, float beta1, float beta2, float eps, float weight_decay,
                                                        float bc1, float bc2_sqrt, const float* __restrict__ norm) {
    const float coef = norm[1];
    const float step_size = lr / bc1;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float pi = p[i];
        const float gc = g[i] * coef;                       // clipped gradient (what clip_grad_norm_ leaves in .grad)
        g[i] = gc;
        const float gi = fmaf(weight_decay, pi, gc);         // coupled L2 decay
        const float mi = beta1 * m[i] + (1.f - beta1) * gi;
        const float vi = beta2 * v[i] + (1.f - beta2) * gi * gi;
        m[i] = mi; v[i] = vi;
        const float denom = sqrtf(vi) / bc2_sqrt + eps;
        p[i] = pi - step_size * (mi / denom);
    }
}

}  // namespace

}  // namespace b200tts
using namespace b200tts;

extern "C" {

size_t b200tts_adam_clip_scratch_floats(void) { return NORM_BLOCKS + 8; }

int b200tts_adam_clip_step(float* p, float* g, float* m, float* v, size_t n, float lr, float beta1, float beta2, float eps,
                           float weight_decay, float max_norm, int step, float* scratch, void* stream) {
    B200_TRY(require_device());
    B200_REQUIRE(p && g && m && v && scratch, "adam_clip_step: null argument");
    B200_REQUIRE(step >= 1 && beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f, "adam_clip_step: step must be >= 1 and betas in [0, 1)");
    B200_REQUIRE((reinterpret_cast<uintptr_t>(g) & 15) == 0, "adam_clip_step: the gradient buffer must be 16-byte aligned");
    if (n == 0) return B200TTS_OK;
    cudaStream_t st = (cudaStream_t)stream;
    float* norm = scratch;                  // [0] = norm, [1] = clip coefficient
    float* partial = scratch + 8;
    size_t want = (n / 4 + 255) / 256;
    const int nblk = (int)(want < 1 ? 1 : (want > NORM_BLOCKS ? NORM_BLOCKS : want));
    sqnorm_partial_kernel<<<nblk, 256, 0, st>>>(g, n, partial);
    B200_LAUNCH_CHECK();
    sqnorm_finish_kernel<<<1, 256, 0, st>>>(partial, nblk, max_norm, norm);
    B200_LAUNCH_CHECK();
    const double bc1 = 1.0 - pow((double)beta1, (double)step), bc2 = 1.0 - pow((double)beta2, (double)step);
    size_t ub = (n + 255) / 256;
    const int ublk = (int)(ub > NUM_SMS * 16 ? NUM_SMS * 16 : ub);
    adam_clip_kernel<<<ublk, 256, 0, st>>>(p, g, m, v, n, lr, beta1, beta2, eps, weight_decay, (float)bc1, (float)sqrt(bc2), norm);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // extern "C"
