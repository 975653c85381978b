// Encoder-side ops: (grouped, dilated) 1-D convolution block with batch-norm / activation / dropout /
// highway gate, the per-language parameter generator, and embedding gather / scatter.
//   reference: modules/layers.py:50-178 (ConvBlock*, HighwayConvBlock*), modules/generated.py:7-96,
//              modules/encoder.py:196-221, modules/tacotron2.py:237-239,363 (embedding), :143-146 (cond. embeddings)
// Convolutions run as im2col + the batched fp32 GEMM (one GEMM per (sample-row, language) pair, the
// generated per-language kernels shared across rows through GemmDesc::a_batch_mod).
#include "common.cuh"

namespace b200tts {

namespace {

// col[nb, i*k + t, l] = x[nb, i, l + t*dil - pad]  (zero outside)      nb runs over (row, group) pairs
__global__ void im2col1d_kernel(float* __restrict__ col, const float* __restrict__ x, size_t NBG, int Cin, int L, int k, int dil, int pad) {
    const size_t total = NBG * Cin * k * L;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int l = idx % L;
        const int t = (idx / L) % k;
        const size_t ni = idx / ((size_t)L * k);          // nb * Cin + i
        const int ls = l + t * dil - pad;
        col[idx] = (ls >= 0 && ls < L) ? x[ni * L + ls] : 0.f;
    }
}

// dx[nb, i, l] (+)= sum_t dcol[nb, i*k + t, l - t*dil + pad]
__global__ void col2im1d_kernel(float* __restrict__ dx, const float* __restrict__ dcol, size_t NBG, int Cin, int L, int k, int dil,
                                int pad, int accumulate) {
    const size_t total = NBG * Cin * L;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int l = idx % L;
        const size_t ni = idx / L;
        float acc = accumulate ? dx[idx] : 0.f;
        for (int t = 0; t < k; ++t) {
            const int lo = l - t * dil + pad;
            if (lo >= 0 && lo < L) acc += dcol[(ni * k + t) * L + lo];
        }
        dx[idx] = acc;
    }
}

// Sum over the (NB, L) slab of channel c of f(x).  The slab is NB rows of L contiguous values; the (row, 16-byte group) pairs are
// flattened over the 256 threads and walked four at a time, so that every thread keeps four independent 16-byte loads in flight whatever
// L is (a row of the encoder has only 45 such groups: walking row by row left 80 % of the block idle behind one load latency per row).
template <class F>
__device__ __forceinline__ float channel_sum(const float* __restrict__ x, int c, int NB, int Ct, int L, F f) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    const bool vec = (L & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
    if (vec) {
        const int L4 = L >> 2, total = NB * L4;
        for (int i0 = threadIdx.x; i0 < total; i0 += 4 * (int)blockDim.x) {
            float4 v[4]; int qq[4], ll[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int i = i0 + u * (int)blockDim.x;
                qq[u] = -1;
                if (i < total) {
                    const int q = i / L4, l4 = i - q * L4;
                    qq[u] = q; ll[u] = 4 * l4;
                    v[u] = reinterpret_cast<const float4*>(x + ((size_t)q * Ct + c) * L)[l4];
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (qq[u] >= 0) {
                    a0 += f(v[u].x, qq[u], ll[u]); a1 += f(v[u].y, qq[u], ll[u] + 1); a2 += f(v[u].z, qq[u], ll[u] + 2); a3 += f(v[u].w, qq[u], ll[u] + 3);
                }
        }
    } else {
        for (int q = 0; q < NB; ++q) {
            const float* row = x + ((size_t)q * Ct + c) * L;
            for (int l = threadIdx.x; l < L; l += blockDim.x) a0 += f(row[l], q, l);
        }
    }
    return (a0 + a1) + (a2 + a3);
}

// Rows of channel block g that hold utterances: counts[g] clamped to [0, NB], so that a count out of range never addresses a row
// outside the tensor (a count above NB reads as NB, a negative one as 0).  Without counts every row is occupied.
__device__ __forceinline__ int block_rows(const int* __restrict__ counts, int g, int NB) {
    if (!counts) return NB;
    const int n = counts[g];
    return n < 0 ? 0 : (n > NB ? NB : n);
}

// per-channel batch statistics over (NB, L); x [NB, Ct, L].  One CTA per channel, two passes (mean, then variance).
// counts (or null): channel block g = c / Cout takes its statistics over its occupied rows q < counts[g] only, summed in the same
// order as the whole slab; a block with no occupied row writes mean 0 / invstd 0 and leaves its running statistics as they are.
__global__ void __launch_bounds__(256) bn_stats_kernel(const float* __restrict__ x, float* __restrict__ mean, float* __restrict__ invstd,
                                                       float* __restrict__ running_mean, float* __restrict__ running_var, int NB,
                                                       int Ct, int L, float eps, float momentum, const int* __restrict__ counts, int Cout) {
    __shared__ float red[64];
    const int c = blockIdx.x;
    const int rows = block_rows(counts, c / Cout, NB);
    if (rows == 0) {
        if (threadIdx.x == 0) { mean[c] = 0.f; invstd[c] = 0.f; }
        return;
    }
    const int n = rows * L;
    const float s = channel_sum(x, c, rows, Ct, L, [](float v, int, int) { return v; });
    const float mu = block_sum(s, red) / (float)n;
    const float v = channel_sum(x, c, rows, Ct, L, [mu](float xv, int, int) { const float d = xv - mu; return d * d; });
    const float var = block_sum(v, red) / (float)n;
    if (threadIdx.x == 0) {
        mean[c] = mu;
        invstd[c] = 1.f / sqrtf(var + eps);
        if (running_mean) {
            const float unbiased = n > 1 ? var * ((float)n / (float)(n - 1)) : var;
            running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mu;
            running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
        }
    }
}

__global__ void bn_eval_stats_kernel(float* __restrict__ mean, float* __restrict__ invstd, const float* __restrict__ rm,
                                     const float* __restrict__ rv, int Ct, float eps) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < Ct) { mean[c] = rm[c]; invstd[c] = 1.f / sqrtf(rv[c] + eps); }
}

__device__ __forceinline__ float act_fwd(int kind, float z) { return kind == 1 ? fmaxf(z, 0.f) : (kind == 2 ? tanhf(z) : z); }
__device__ __forceinline__ float act_bwd(int kind, float z, float a) { return kind == 1 ? (z > 0.f ? 1.f : 0.f) : (kind == 2 ? 1.f - a * a : 1.f); }

struct BlockArgs {
    const float* conv;      // [NB, G*Cout, L] convolution output (pre batch-norm)
    const float* mean; const float* invstd;   // [G*Cout]
    const float* gamma; const float* beta; int affine_gstride;   // gamma[g*stride + o]
    const uint8_t* keep; float keep_scale;    // [NB, G*Cout, L] or null
    const float* xin;       // [NB, G*Cin, L] block input (highway only)
    int NB, G, Cout, L, act, highway;
    const int* lengths;     // [NB] or null (forward only): outputs at positions l >= lengths[nb] are written as 0
    const int* counts;      // [G] or null: rows nb >= counts[g] of channel block g are vacant; their outputs and gradients are written as 0
};

// idx -> (nb, g, c, l) of a [NB, G, Cf, L] tensor; 32-bit arithmetic whenever the tensor has fewer than 2^32 elements
__device__ __forceinline__ void split_index(size_t idx, bool small, int L, int Cf, int G, int& l, int& c, int& g, size_t& nb) {
    if (small) {
        const unsigned i = (unsigned)idx, r = i / (unsigned)L, r2 = r / (unsigned)Cf, r3 = r2 / (unsigned)G;
        l = (int)(i - r * (unsigned)L); c = (int)(r - r2 * (unsigned)Cf); g = (int)(r2 - r3 * (unsigned)G); nb = r3;
    } else {
        l = idx % L; c = (idx / L) % Cf; g = (idx / ((size_t)L * Cf)) % G; nb = idx / ((size_t)L * Cf * G);
    }
}

// y = dropout(act(bn(conv)));  highway: out[g, c] = y[g, C + c] * sigmoid(y[g, c]) + xin[g, c] * (1 - sigmoid(y[g, c]))
__global__ void block_fwd_kernel(const BlockArgs p, float* __restrict__ out) {
    const int Cf = p.highway ? p.Cout / 2 : p.Cout;
    const size_t total = (size_t)p.NB * p.G * Cf * p.L;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        int l, c, g; size_t nb;
        split_index(idx, total <= 0xffffffffull, p.L, Cf, p.G, l, c, g, nb);
        if (p.lengths && l >= p.lengths[nb]) { out[idx] = 0.f; continue; }
        if (p.counts && (int)nb >= block_rows(p.counts, g, p.NB)) { out[idx] = 0.f; continue; }
        auto value = [&](int o) {
            const int ch = g * p.Cout + o;
            const size_t ci = (nb * p.G * p.Cout + ch) * p.L + l;
            const float z = (p.conv[ci] - p.mean[ch]) * p.invstd[ch] * p.gamma[g * p.affine_gstride + o] + p.beta[g * p.affine_gstride + o];
            float a = act_fwd(p.act, z);
            if (p.keep) a = a * (float)p.keep[ci] * p.keep_scale;
            return a;
        };
        if (p.highway) {
            const float h1 = value(c), h2 = value(Cf + c);
            const float s = sigmoidf_acc(h1);
            out[idx] = h2 * s + p.xin[idx] * (1.f - s);
        } else {
            out[idx] = value(c);
        }
    }
}

// The same for 4 consecutive positions per thread (L % 4 == 0, 16-byte aligned tensors): one index split per 4 elements, 128-bit
// loads / stores, 32-bit keep-mask words.  Element arithmetic is identical to the scalar kernel.
__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ float4 keep4(const uint8_t* keep, size_t i, float scale) {
    const uint32_t w = *reinterpret_cast<const uint32_t*>(keep + i);
    return make_float4((float)(w & 0xffu) * scale, (float)((w >> 8) & 0xffu) * scale, (float)((w >> 16) & 0xffu) * scale, (float)(w >> 24) * scale);
}
__global__ void __launch_bounds__(256) block_fwd_vec4_kernel(const BlockArgs p, float* __restrict__ out) {
    const int Cf = p.highway ? p.Cout / 2 : p.Cout, L4 = p.L >> 2;
    const unsigned total = (unsigned)p.NB * p.G * Cf * L4;          // < 2^32 (checked by the launcher)
    for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
        const unsigned row = idx / (unsigned)L4, l4 = idx - row * (unsigned)L4;        // row = (nb * G + g) * Cf + c
        const unsigned r2 = row / (unsigned)Cf, c = row - r2 * (unsigned)Cf, nb = r2 / (unsigned)p.G, g = r2 - nb * (unsigned)p.G;
        auto value = [&](int o) {
            const int ch = g * p.Cout + o;
            const size_t ci = ((size_t)(nb * p.G * p.Cout + ch)) * p.L + 4 * l4;
            const float mu = p.mean[ch], be = p.beta[g * p.affine_gstride + o];
            const float is = p.invstd[ch], ga = p.gamma[g * p.affine_gstride + o];
            const float4 x = ld4(p.conv + ci);
            float4 a;
            a.x = act_fwd(p.act, (x.x - mu) * is * ga + be); a.y = act_fwd(p.act, (x.y - mu) * is * ga + be);
            a.z = act_fwd(p.act, (x.z - mu) * is * ga + be); a.w = act_fwd(p.act, (x.w - mu) * is * ga + be);

            if (p.keep) {
                const float4 k = keep4(p.keep, ci, p.keep_scale);
                a.x *= k.x; a.y *= k.y; a.z *= k.z; a.w *= k.w;
            }
            return a;
        };
        const size_t oi = (size_t)row * p.L + 4 * l4;
        // a float4 group may straddle the utterance's length: the lanes at or past it are zeroed one by one
        int valid = p.lengths ? p.lengths[nb] - 4 * (int)l4 : 4;
        if (p.counts && (int)nb >= block_rows(p.counts, (int)g, p.NB)) valid = 0;      // vacant row
        if (valid <= 0) { st4(out + oi, make_float4(0.f, 0.f, 0.f, 0.f)); continue; }
        float4 r;
        if (p.highway) {
            const float4 h1 = value(c), h2 = value(Cf + c), xi = ld4(p.xin + oi);
            const float s0 = sigmoidf_acc(h1.x), s1 = sigmoidf_acc(h1.y), s2 = sigmoidf_acc(h1.z), s3 = sigmoidf_acc(h1.w);
            r = make_float4(h2.x * s0 + xi.x * (1.f - s0), h2.y * s1 + xi.y * (1.f - s1), h2.z * s2 + xi.z * (1.f - s2),
                            h2.w * s3 + xi.w * (1.f - s3));
        } else {
            r = value(c);
        }
        if (valid < 4) {
            r.w = 0.f;
            if (valid < 3) r.z = 0.f;
            if (valid < 2) r.y = 0.f;
        }
        st4(out + oi, r);
    }
}

__global__ void __launch_bounds__(256) block_bwd_prep_vec4_kernel(const BlockArgs p, const float* __restrict__ dout, float* __restrict__ dz,
                                                                  float* __restrict__ dx_skip) {
    const int Cf = p.highway ? p.Cout / 2 : p.Cout, L4 = p.L >> 2;
    const unsigned total = (unsigned)p.NB * p.G * Cf * L4;
    for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
        const unsigned row = idx / (unsigned)L4, l4 = idx - row * (unsigned)L4;
        const unsigned r2 = row / (unsigned)Cf, c = row - r2 * (unsigned)Cf, nb = r2 / (unsigned)p.G, g = r2 - nb * (unsigned)p.G;
        const size_t oi = (size_t)row * p.L + 4 * l4;
        if (p.counts && (int)nb >= block_rows(p.counts, (int)g, p.NB)) {       // vacant row: no gradient anywhere
            const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
            const size_t ci = ((size_t)(nb * p.G * p.Cout + g * p.Cout + c)) * p.L + 4 * l4;
            st4(dz + ci, z);
            if (p.highway) { st4(dz + ci + (size_t)Cf * p.L, z); st4(dx_skip + oi, z); }
            continue;
        }
        const float4 go4 = ld4(dout + oi);
        const float go[4] = {go4.x, go4.y, go4.z, go4.w};
        float zs[2][4], as[2][4], ks[2][4];
        size_t cis[2];
        const int nch = p.highway ? 2 : 1;
        for (int j = 0; j < nch; ++j) {
            const int o = c + j * Cf, ch = g * p.Cout + o;
            cis[j] = ((size_t)(nb * p.G * p.Cout + ch)) * p.L + 4 * l4;
            const float mu = p.mean[ch], is = p.invstd[ch], ga = p.gamma[g * p.affine_gstride + o], be = p.beta[g * p.affine_gstride + o];
            const float4 x = ld4(p.conv + cis[j]);
            const float xs[4] = {x.x, x.y, x.z, x.w};
            float4 k4 = make_float4(1.f, 1.f, 1.f, 1.f);
            if (p.keep) k4 = keep4(p.keep, cis[j], p.keep_scale);
            const float kk[4] = {k4.x, k4.y, k4.z, k4.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                zs[j][e] = (xs[e] - mu) * is * ga + be;
                as[j][e] = act_fwd(p.act, zs[j][e]);
                ks[j][e] = kk[e];
            }
        }
        if (p.highway) {
            const float4 xi4 = ld4(p.xin + oi);
            const float xi[4] = {xi4.x, xi4.y, xi4.z, xi4.w};
            float d1[4], d2[4], dsk[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float h1 = as[0][e] * ks[0][e], h2 = as[1][e] * ks[1][e];
                const float sg = sigmoidf_acc(h1);
                const float dh1 = go[e] * (h2 - xi[e]) * sg * (1.f - sg), dh2 = go[e] * sg;
                d1[e] = dh1 * ks[0][e] * act_bwd(p.act, zs[0][e], as[0][e]);
                d2[e] = dh2 * ks[1][e] * act_bwd(p.act, zs[1][e], as[1][e]);
                dsk[e] = go[e] * (1.f - sg);
            }
            st4(dz + cis[0], make_float4(d1[0], d1[1], d1[2], d1[3]));
            st4(dz + cis[1], make_float4(d2[0], d2[1], d2[2], d2[3]));
            st4(dx_skip + oi, make_float4(dsk[0], dsk[1], dsk[2], dsk[3]));
        } else {
            float d[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) d[e] = go[e] * ks[0][e] * act_bwd(p.act, zs[0][e], as[0][e]);
            st4(dz + cis[0], make_float4(d[0], d[1], d[2], d[3]));
        }
    }
}

__global__ void __launch_bounds__(256) bn_bwd_apply_vec4_kernel(float* __restrict__ dz, const float* __restrict__ conv,
                                                                const float* __restrict__ mean, const float* __restrict__ invstd,
                                                                const float* __restrict__ gamma, int affine_gstride, const float* __restrict__ s1,
                                                                const float* __restrict__ s2, int NB, int G, int Cout, int L, int training,
                                                                const int* __restrict__ counts) {
    const int Ct = G * Cout, L4 = L >> 2;
    const unsigned total = (unsigned)NB * Ct * L4;
    const float inv_n_all = 1.f / (float)(NB * L);
    for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
        const unsigned row = idx / (unsigned)L4, l4 = idx - row * (unsigned)L4;
        const int ch = (int)(row % (unsigned)Ct);
        const size_t i = (size_t)row * L + 4 * l4;
        float inv_n = inv_n_all;
        if (counts) {
            const int rows = block_rows(counts, ch / Cout, NB);
            if ((int)(row / (unsigned)Ct) >= rows) { st4(dz + i, make_float4(0.f, 0.f, 0.f, 0.f)); continue; }
            inv_n = 1.f / (float)(rows * L);
        }
        const float is = invstd[ch], gm = gamma[(ch / Cout) * affine_gstride + ch % Cout] * is;
        float4 d = ld4(dz + i);
        if (training) {
            const float a = s1[ch] * inv_n, b = is * s2[ch] * inv_n, mu = mean[ch];
            const float4 x = ld4(conv + i);
            d.x = d.x - a - (x.x - mu) * b; d.y = d.y - a - (x.y - mu) * b; d.z = d.z - a - (x.z - mu) * b; d.w = d.w - a - (x.w - mu) * b;
        }
        st4(dz + i, make_float4(gm * d.x, gm * d.y, gm * d.z, gm * d.w));
    }
}

// backward through highway / dropout / activation: dz [NB, G*Cout, L] (grad wrt the batch-norm output) and,
// for highway blocks, the skip-path gradient dx = dout * (1 - sigmoid(h1)).
__global__ void block_bwd_prep_kernel(const BlockArgs p, const float* __restrict__ dout, float* __restrict__ dz, float* __restrict__ dx_skip) {
    const int Cf = p.highway ? p.Cout / 2 : p.Cout;
    const size_t total = (size_t)p.NB * p.G * Cf * p.L;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        int l, c, g; size_t nb;
        split_index(idx, total <= 0xffffffffull, p.L, Cf, p.G, l, c, g, nb);
        if (p.counts && (int)nb >= block_rows(p.counts, g, p.NB)) {      // vacant row: no gradient anywhere
            const size_t ci = (nb * p.G * p.Cout + g * p.Cout + c) * p.L + l;
            dz[ci] = 0.f;
            if (p.highway) { dz[ci + (size_t)Cf * p.L] = 0.f; dx_skip[idx] = 0.f; }
            continue;
        }
        float zs[2], as[2], ks[2];
        size_t cis[2];
        const int nch = p.highway ? 2 : 1;
        for (int j = 0; j < nch; ++j) {
            const int o = c + j * Cf, ch = g * p.Cout + o;
            cis[j] = (nb * p.G * p.Cout + ch) * p.L + l;
            zs[j] = (p.conv[cis[j]] - p.mean[ch]) * p.invstd[ch] * p.gamma[g * p.affine_gstride + o] + p.beta[g * p.affine_gstride + o];
            as[j] = act_fwd(p.act, zs[j]);
            ks[j] = p.keep ? (float)p.keep[cis[j]] * p.keep_scale : 1.f;
        }
        const float go = dout[idx];
        if (p.highway) {
            const float h1 = as[0] * ks[0], h2 = as[1] * ks[1];
            const float s = sigmoidf_acc(h1);
            const float dh1 = go * (h2 - p.xin[idx]) * s * (1.f - s), dh2 = go * s;
            dz[cis[0]] = dh1 * ks[0] * act_bwd(p.act, zs[0], as[0]);
            dz[cis[1]] = dh2 * ks[1] * act_bwd(p.act, zs[1], as[1]);
            dx_skip[idx] = go * (1.f - s);
        } else {
            dz[cis[0]] = go * ks[0] * act_bwd(p.act, zs[0], as[0]);
        }
    }
}

// per channel: s1 = sum dz, s2 = sum dz * xhat  -> dbeta += s1, dgamma += s2; keeps s1, s2 for the apply pass
__global__ void __launch_bounds__(256) bn_bwd_reduce_kernel(const float* __restrict__ dz, const float* __restrict__ conv,
                                                            const float* __restrict__ mean, const float* __restrict__ invstd,
                                                            float* __restrict__ s1o, float* __restrict__ s2o, float* __restrict__ dgamma,
                                                            float* __restrict__ dbeta, int affine_gstride, int NB, int G, int Cout, int L,
                                                            const int* __restrict__ counts) {
    __shared__ float red[64];
    const int ch = blockIdx.x, Ct = G * Cout;
    NB = block_rows(counts, ch / Cout, NB);      // the occupied rows of this channel's block (all of them without counts)
    const float mu = mean[ch], is = invstd[ch];
    float s1, s2;
    const bool vec = (L & 3) == 0 && (reinterpret_cast<uintptr_t>(dz) & 15) == 0 && (reinterpret_cast<uintptr_t>(conv) & 15) == 0;
    if (vec) {      // ONE pass over dz and conv (16-byte loads of both at the same position, two of them in flight per thread)
        float p1[4] = {0.f, 0.f, 0.f, 0.f}, p2[4] = {0.f, 0.f, 0.f, 0.f};
        const int L4 = L >> 2, total = NB * L4;
        for (int i0 = threadIdx.x; i0 < total; i0 += 2 * (int)blockDim.x) {
            float4 d4[2], c4[2]; bool ok[2];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int i = i0 + u * (int)blockDim.x;
                ok[u] = i < total;
                if (ok[u]) {
                    const int q = i / L4, l4 = i - q * L4;
                    const size_t off = ((size_t)q * Ct + ch) * L;
                    d4[u] = reinterpret_cast<const float4*>(dz + off)[l4];
                    c4[u] = reinterpret_cast<const float4*>(conv + off)[l4];
                }
            }
#pragma unroll
            for (int u = 0; u < 2; ++u)
                if (ok[u]) {
                    p1[0] += d4[u].x; p1[1] += d4[u].y; p1[2] += d4[u].z; p1[3] += d4[u].w;
                    p2[0] += d4[u].x * (c4[u].x - mu) * is; p2[1] += d4[u].y * (c4[u].y - mu) * is;
                    p2[2] += d4[u].z * (c4[u].z - mu) * is; p2[3] += d4[u].w * (c4[u].w - mu) * is;
                }
        }
        s1 = (p1[0] + p1[1]) + (p1[2] + p1[3]); s2 = (p2[0] + p2[1]) + (p2[2] + p2[3]);
    } else {
        s1 = channel_sum(dz, ch, NB, Ct, L, [](float d, int, int) { return d; });
        s2 = channel_sum(dz, ch, NB, Ct, L, [=](float d, int q, int l) { return d * (conv[((size_t)q * Ct + ch) * L + l] - mu) * is; });
    }
    s1 = block_sum(s1, red);
    s2 = block_sum(s2, red);
    if (threadIdx.x == 0) {
        s1o[ch] = s1; s2o[ch] = s2;
        const int g = ch / Cout, o = ch % Cout;
        if (dbeta) dbeta[g * affine_gstride + o] += s1;
        if (dgamma) dgamma[g * affine_gstride + o] += s2;
    }
}

// dconv = gamma * invstd * (dz - s1/n - xhat * s2/n)   (training);  gamma * invstd * dz (eval).  In place on dz.
__global__ void bn_bwd_apply_kernel(float* __restrict__ dz, const float* __restrict__ conv, const float* __restrict__ mean,
                                    const float* __restrict__ invstd, const float* __restrict__ gamma, int affine_gstride,
                                    const float* __restrict__ s1, const float* __restrict__ s2, int NB, int G, int Cout, int L, int training,
                                    const int* __restrict__ counts) {
    const int Ct = G * Cout;
    const size_t total = (size_t)NB * Ct * L;
    const float inv_n_all = 1.f / (float)(NB * L);
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int ch = total <= 0xffffffffull ? (int)(((unsigned)idx / (unsigned)L) % (unsigned)Ct) : (int)((idx / L) % Ct);
        float inv_n = inv_n_all;
        if (counts) {
            const int rows = block_rows(counts, ch / Cout, NB);
            if ((long long)(idx / ((size_t)L * Ct)) >= rows) { dz[idx] = 0.f; continue; }
            inv_n = 1.f / (float)(rows * L);
        }
        const float gm = gamma[(ch / Cout) * affine_gstride + ch % Cout] * invstd[ch];
        float d = dz[idx];
        if (training) d = d - s1[ch] * inv_n - (conv[idx] - mean[ch]) * invstd[ch] * s2[ch] * inv_n;
        dz[idx] = gm * d;
    }
}

// x [NB, G*C, L]: every vacant row (nb >= counts[g]) of channel block g set to 0.  The convolution-only stage's output and gradient.
__global__ void zero_vacant_kernel(float* __restrict__ x, const int* __restrict__ counts, int NB, int G, int C, int L) {
    const size_t total = (size_t)NB * G * C * L;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const size_t row = idx / L;
        const int g = (int)((row % ((size_t)G * C)) / C);
        if ((long long)(row / ((size_t)G * C)) >= block_rows(counts, g, NB)) x[idx] = 0.f;
    }
}

// out[b, l, :] = table[ids[b, l], :]
__global__ void embedding_fwd_kernel(float* __restrict__ out, int ldo, const float* __restrict__ table, const int* __restrict__ ids,
                                     size_t ntok, int E) {
    const size_t total = ntok * E;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const size_t t = idx / E;
        const int e = idx % E;
        out[t * ldo + e] = table[(size_t)ids[t] * E + e];
    }
}

// dtable[v, :] += sum over tokens with id v of dout[token, :]   (one CTA per vocabulary row: deterministic token order).
// The ids are staged through shared memory 1024 at a time; the positions of the matching tokens of a tile are compacted IN ORDER
// (4 consecutive tokens per thread, block-wide exclusive scan of the hit counts), so only the hits are visited afterwards.
__global__ void __launch_bounds__(256) embedding_bwd_kernel(float* __restrict__ dtable, const float* __restrict__ dout, int ldo,
                                                            const int* __restrict__ ids, int ntok, int E, int padding_idx) {
    __shared__ int s_hits[1024];
    __shared__ int s_wsum[8];
    const int v = blockIdx.x;
    if (v == padding_idx) return;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int EPT = 4;                                   // embedding columns per thread (E <= 1024)
    float acc[EPT];
#pragma unroll
    for (int j = 0; j < EPT; ++j) acc[j] = 0.f;
    for (int t0 = 0; t0 < ntok; t0 += 1024) {
        // this thread's 4 consecutive tokens of the tile
        int mine[4], cnt = 0;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int t = t0 + tid * 4 + u;
            mine[u] = (t < ntok && ids[t] == v) ? 1 : 0;
            cnt += mine[u];
        }
        int incl = cnt;                                       // inclusive scan inside the warp, then across the 8 warps
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int up = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += up;
        }
        __syncthreads();                                      // the previous tile's hit list is no longer read
        if (lane == 31) s_wsum[warp] = incl;
        __syncthreads();
        int base = 0, nh = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) { if (w < warp) base += s_wsum[w]; nh += s_wsum[w]; }
        int pos = base + incl - cnt;
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (mine[u]) s_hits[pos++] = tid * 4 + u;
        __syncthreads();
        for (int h = 0; h < nh; h += 4) {                    // 4 matching rows in flight, added in token order
            float val[4][EPT];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const bool on = h + u < nh;
                const float* row = dout + (size_t)(t0 + (on ? s_hits[h + u] : 0)) * ldo;
#pragma unroll
                for (int j = 0; j < EPT; ++j) {
                    const int e = tid + j * 256;
                    val[u][j] = (on && e < E) ? row[e] : 0.f;
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u)
#pragma unroll
                for (int j = 0; j < EPT; ++j) acc[j] += val[u][j];
        }
    }
#pragma unroll
    for (int j = 0; j < EPT; ++j) {
        const int e = tid + j * 256;
        if (e < E) dtable[(size_t)v * E + e] += acc[j];
    }
}

// ---- parameter generator: skinny products with one huge dimension R (the generated kernel) ----
constexpr int GEN_MAXG = 16, GEN_MAXBN = 16;
// out[g, r] = sum_j eb[g, j] Wk[r, j] + bk[r]
// The bottleneck eb[g, j] = e[g, :] . Wb[j, :] + bb[j] (G * bn values, gd terms each) is recomputed by every block in its prologue -- cheaper
// than a separate launch -- and block 0 stores it for the backward pass.
__global__ void generator_expand_kernel(float* __restrict__ out, float* __restrict__ eb, const float* __restrict__ Wk,
                                        const float* __restrict__ bk, int G, int bn, size_t R, const float* __restrict__ e,
                                        const float* __restrict__ Wb, const float* __restrict__ bb, int gd) {
    __shared__ float s_eb[GEN_MAXG * GEN_MAXBN];
    for (int i = threadIdx.x; i < G * bn; i += blockDim.x) {
        const int g = i / bn, j = i - g * bn;
        float a = bb ? bb[j] : 0.f;
        for (int d = 0; d < gd; ++d) a = fmaf(e[g * gd + d], Wb[j * gd + d], a);
        s_eb[i] = a;
        if (blockIdx.x == 0) eb[i] = a;
    }
    __syncthreads();
    const bool vec8 = (reinterpret_cast<uintptr_t>(Wk) & 15) == 0;
    for (size_t r = blockIdx.x * (size_t)blockDim.x + threadIdx.x; r < R; r += (size_t)gridDim.x * blockDim.x) {
        float w[GEN_MAXBN];
        if (bn == 8 && vec8) {           // one 32-byte row per thread: two 16-byte loads
            const float4 w0 = reinterpret_cast<const float4*>(Wk)[2 * r], w1 = reinterpret_cast<const float4*>(Wk)[2 * r + 1];
            w[0] = w0.x; w[1] = w0.y; w[2] = w0.z; w[3] = w0.w; w[4] = w1.x; w[5] = w1.y; w[6] = w1.z; w[7] = w1.w;
#pragma unroll
            for (int j = 8; j < GEN_MAXBN; ++j) w[j] = 0.f;
        } else {
#pragma unroll
            for (int j = 0; j < GEN_MAXBN; ++j) w[j] = j < bn ? Wk[r * bn + j] : 0.f;
        }
        const float b = bk ? bk[r] : 0.f;
        for (int g = 0; g < G; ++g) {
            float a = b;
#pragma unroll
            for (int j = 0; j < GEN_MAXBN; ++j) if (j < bn) a = fmaf(s_eb[g * bn + j], w[j], a);
            out[(size_t)g * R + r] = a;
        }
    }
}
// dWk[r, j] += sum_g dout[g, r] eb[g, j];  dbk[r] += sum_g dout[g, r]
__global__ void generator_dwk_kernel(float* __restrict__ dWk, float* __restrict__ dbk, const float* __restrict__ dout,
                                     const float* __restrict__ eb, int G, int bn, size_t R) {
    __shared__ float s_eb[GEN_MAXG * GEN_MAXBN];
    for (int i = threadIdx.x; i < G * bn; i += blockDim.x) s_eb[i] = eb[i];
    __syncthreads();
    for (size_t r = blockIdx.x * (size_t)blockDim.x + threadIdx.x; r < R; r += (size_t)gridDim.x * blockDim.x) {
        float acc[GEN_MAXBN];
#pragma unroll
        for (int j = 0; j < GEN_MAXBN; ++j) acc[j] = 0.f;
        float sb = 0.f;
        for (int g = 0; g < G; ++g) {
            const float d = dout[(size_t)g * R + r];
            sb += d;
#pragma unroll
            for (int j = 0; j < GEN_MAXBN; ++j) if (j < bn) acc[j] = fmaf(d, s_eb[g * bn + j], acc[j]);
        }
#pragma unroll
        for (int j = 0; j < GEN_MAXBN; ++j) if (j < bn) dWk[r * bn + j] += acc[j];
        if (dbk) dbk[r] += sb;
    }
}
// Fused backward of the expansion for bn == 8 and G <= 10 (every shipped configuration): ONE pass over dout and Wk, both read coalesced
// (thread = generated element r): dWk[r, :] += dout[:, r]^T eb, dbk[r] += sum_g dout[g, r], and per-block partial sums of
// deb[g, j] = sum_r dout[g, r] Wk[r, j] kept in 80 registers and reduced once per block (fixed order: deterministic).
constexpr int GEN_FG = 10;
__global__ void __launch_bounds__(256) generator_bwd_fused_kernel(float* __restrict__ dWk, float* __restrict__ dbk, float* __restrict__ partial,
                                                                  const float* __restrict__ dout, const float* __restrict__ Wk,
                                                                  const float* __restrict__ eb, int G, size_t R) {
    __shared__ float s_eb[GEN_FG * 8];
    __shared__ float s_red[8][GEN_FG * 8];
    for (int i = threadIdx.x; i < GEN_FG * 8; i += blockDim.x) s_eb[i] = i < G * 8 ? eb[i] : 0.f;
    __syncthreads();
    float acc[GEN_FG][8];
#pragma unroll
    for (int g = 0; g < GEN_FG; ++g)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[g][j] = 0.f;
    for (size_t r = blockIdx.x * (size_t)blockDim.x + threadIdx.x; r < R; r += (size_t)gridDim.x * blockDim.x) {
        float d[GEN_FG];
#pragma unroll
        for (int g = 0; g < GEN_FG; ++g) d[g] = g < G ? dout[(size_t)g * R + r] : 0.f;
        const float4 w0 = reinterpret_cast<const float4*>(Wk)[2 * r], w1 = reinterpret_cast<const float4*>(Wk)[2 * r + 1];
        const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
        float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, sb = 0.f;
#pragma unroll
        for (int g = 0; g < GEN_FG; ++g) {
            sb += d[g];
#pragma unroll
            for (int j = 0; j < 8; ++j) { a[j] = fmaf(d[g], s_eb[g * 8 + j], a[j]); acc[g][j] = fmaf(d[g], w[j], acc[g][j]); }
        }
        float4* o = reinterpret_cast<float4*>(dWk) + 2 * r;
        float4 o0 = o[0], o1 = o[1];
        o0.x += a[0]; o0.y += a[1]; o0.z += a[2]; o0.w += a[3]; o1.x += a[4]; o1.y += a[5]; o1.z += a[6]; o1.w += a[7];
        o[0] = o0; o[1] = o1;
        if (dbk) dbk[r] += sb;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int g = 0; g < GEN_FG; ++g)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float v = warp_sum(acc[g][j]);
            if (lane == 0) s_red[warp][g * 8 + j] = v;
        }
    __syncthreads();
    if (threadIdx.x < G * 8) {
        float t = 0.f;
#pragma unroll
        for (int w8 = 0; w8 < 8; ++w8) t += s_red[w8][threadIdx.x];
        partial[(size_t)blockIdx.x * G * 8 + threadIdx.x] = t;
    }
}
// partial[blk][g, j] = sum over this block's r-chunk of dout[g, r] Wk[r, j]   (thread = (g, j); fixed chunking: deterministic)
__global__ void generator_deb_partial_kernel(float* __restrict__ partial, const float* __restrict__ dout, const float* __restrict__ Wk,
                                             int G, int bn, size_t R, size_t chunk) {
    const int t = threadIdx.x;
    if (t >= G * bn) return;
    const int g = t / bn, j = t % bn;
    const size_t r0 = blockIdx.x * chunk, r1 = r0 + chunk < R ? r0 + chunk : R;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    size_t r = r0;
    for (; r + 3 < r1; r += 4) {
        a0 = fmaf(dout[(size_t)g * R + r], Wk[r * bn + j], a0);
        a1 = fmaf(dout[(size_t)g * R + r + 1], Wk[(r + 1) * bn + j], a1);
        a2 = fmaf(dout[(size_t)g * R + r + 2], Wk[(r + 2) * bn + j], a2);
        a3 = fmaf(dout[(size_t)g * R + r + 3], Wk[(r + 3) * bn + j], a3);
    }
    for (; r < r1; ++r) a0 = fmaf(dout[(size_t)g * R + r], Wk[r * bn + j], a0);
    partial[(size_t)blockIdx.x * G * bn + t] = (a0 + a1) + (a2 + a3);
}
// deb[t] = sum over the chunk partials, one CTA per output element (fixed tree: deterministic)
__global__ void __launch_bounds__(128) generator_deb_finish_kernel(float* __restrict__ deb, const float* __restrict__ partial, int nblk, int n) {
    __shared__ float red[64];
    const int t = blockIdx.x;
    float s = 0.f;
    for (int b = threadIdx.x; b < nblk; b += blockDim.x) s += partial[(size_t)b * n + t];
    s = block_sum(s, red);
    if (threadIdx.x == 0) deb[t] = s;
}

__global__ void colsum_rows_add_kernel(float* __restrict__ dst, const float* __restrict__ src, int rows, size_t cols) {
    for (size_t c = blockIdx.x * (size_t)blockDim.x + threadIdx.x; c < cols; c += (size_t)gridDim.x * blockDim.x) {
        float s = 0.f;
        for (int r = 0; r < rows; ++r) s += src[(size_t)r * cols + c];
        dst[c] += s;
    }
}

struct BlockDims {
    int NB, G, Cin, Cout, L, k, dil, pad, Cf;
    size_t conv_elems, col_elems, Ct;
};
inline BlockDims block_dims(const b200tts_convblock_shape& s) {
    BlockDims d;
    d.NB = s.NB; d.G = s.G; d.Cin = s.Cin; d.Cout = s.Cout; d.L = s.L; d.k = s.k; d.dil = s.dilation;
    d.pad = (s.k - 1) * s.dilation / 2;
    d.Cf = s.highway ? s.Cout / 2 : s.Cout;
    d.Ct = (size_t)s.G * s.Cout;
    d.conv_elems = (size_t)s.NB * d.Ct * s.L;
    d.col_elems = s.k > 1 ? (size_t)s.NB * s.G * s.Cin * s.k * s.L : 0;
    return d;
}
constexpr size_t kGemmScratch = (size_t)4 * 1024 * 1024;

// 4 positions per thread: needs L % 4 == 0, 16-byte aligned tensors and fewer than 2^32 float4 groups
bool vec4_ok(const b200tts_convblock_shape& s, const BlockDims& d, const float* conv, const float* out, const float* xin, const uint8_t* keep) {
    auto al = [](const void* p, uintptr_t m) { return (reinterpret_cast<uintptr_t>(p) & m) == 0; };
    return (s.L & 3) == 0 && al(conv, 15) && al(out, 15) && (!s.highway || al(xin, 15)) && (!keep || al(keep, 3)) &&
           d.conv_elems / 4 < 0xffffffffull;
}

int validate_block(const b200tts_convblock_shape& s) {
    B200_REQUIRE(s.NB > 0 && s.G > 0 && s.Cin > 0 && s.Cout > 0 && s.L > 0 && s.k > 0 && s.dilation > 0, "convblock: non-positive dimension");
    B200_REQUIRE(s.k % 2 == 1, "convblock: even kernel sizes are not supported (k=%d)", s.k);
    B200_REQUIRE(!s.highway || s.Cout == 2 * s.Cin, "convblock: highway needs Cout == 2*Cin (got %d, %d)", s.Cout, s.Cin);
    B200_REQUIRE(s.activation >= 0 && s.activation <= 2, "convblock: unknown activation %d", s.activation);
    B200_REQUIRE(s.dropout >= 0.f && s.dropout < 1.f, "convblock: dropout must be in [0,1)");
    B200_REQUIRE(s.stage >= 0 && s.stage <= 2, "convblock: unknown stage %d", s.stage);
    B200_REQUIRE(s.stage == 0 || !s.highway, "convblock: the highway gate needs the whole block (stage 0)");
    B200_REQUIRE(s.stage != 2 || (s.Cin == s.Cout && s.k == 1), "convblock: stage 2 (batch norm only) needs Cin == Cout and k == 1");
    return B200TTS_OK;
}

}  // namespace

static int convblock_forward_impl(const b200tts_convblock_shape& s, const float* x, const float* weight, const float* gamma,
                                  const float* beta, int affine_gstride, float* running_mean, float* running_var, const uint8_t* keep,
                                  float* out, float* saved, float* ws, cudaStream_t st, const int32_t* lengths = nullptr,
                                  const int32_t* counts = nullptr) {
    B200_TRY(validate_block(s));
    // padded batches: only the fused epilogue of an eval-mode whole block knows the lengths (training statistics would need them too)
    B200_REQUIRE(!lengths || (s.stage == 0 && !s.training), "convblock_forward_masked: lengths need an eval-mode whole block (stage 0)");
    const BlockDims d = block_dims(s);
    float* conv = s.stage == 1 ? out : saved;     // convolution only: the product IS the output
    float* mean = saved + align_up_sz(d.conv_elems, 64);
    float* invstd = mean + align_up_sz(d.Ct, 64);
    bool implicit = s.stage == 2;                 // batch norm only: there is no product, x plays the role of the convolution output
    if (s.stage == 2) conv = const_cast<float*>(x);
    if (!implicit && precision_mode() != 0 && s.k > 1)       // bf16 perf mode: implicit convolution on the wgmma GEMM (TMA row shifts per tap, no im2col)
        B200_TRY(gemm_tc_conv(weight, x, conv, s.NB, s.G, s.Cout, s.Cin, s.L, s.k, s.dilation, d.pad, 0, 0.f, st, &implicit));
    if (!implicit) {
        const float* col = x;
        if (s.k > 1) {
            im2col1d_kernel<<<grid_for(d.col_elems), 256, 0, st>>>(ws, x, (size_t)s.NB * s.G, s.Cin, s.L, s.k, s.dilation, d.pad);
            B200_LAUNCH_CHECK();
            col = ws;
        }
        GemmDesc g;
        g.A = weight; g.lda = s.Cin * s.k; g.transA = 0; g.a_batch_mod = s.G; g.strideA = (long long)s.Cout * s.Cin * s.k;
        g.B = col; g.ldb = s.L; g.transB = 0; g.strideB = (long long)s.Cin * s.k * s.L;
        g.C = conv; g.ldc = s.L; g.strideC = (long long)s.Cout * s.L;
        g.M = s.Cout; g.N = s.L; g.K = s.Cin * s.k; g.batch = s.NB * s.G;
        B200_TRY(gemm_run(g, st));
    }
    if (s.stage == 1) {
        if (counts) {
            zero_vacant_kernel<<<grid_for(d.conv_elems), 256, 0, st>>>(out, counts, s.NB, s.G, s.Cout, s.L);
            B200_LAUNCH_CHECK();
        }
        return B200TTS_OK;
    }
    if (s.training) {
        bn_stats_kernel<<<(int)d.Ct, 256, 0, st>>>(conv, mean, invstd, running_mean, running_var, s.NB, (int)d.Ct, s.L, s.eps, s.momentum,
                                                   counts, s.Cout);
    } else {
        B200_REQUIRE(running_mean && running_var, "convblock: eval mode needs running statistics");
        bn_eval_stats_kernel<<<cdiv(d.Ct, 256), 256, 0, st>>>(mean, invstd, running_mean, running_var, (int)d.Ct, s.eps);
    }
    B200_LAUNCH_CHECK();
    BlockArgs a{conv, mean, invstd, gamma, beta, affine_gstride, (s.training && s.dropout > 0.f) ? keep : nullptr,
                1.f / (1.f - s.dropout), x, s.NB, s.G, s.Cout, s.L, s.activation, s.highway, lengths, counts};
    if (vec4_ok(s, d, conv, out, x, a.keep))
        block_fwd_vec4_kernel<<<grid_for((size_t)s.NB * s.G * d.Cf * (s.L / 4)), 256, 0, st>>>(a, out);
    else
        block_fwd_kernel<<<grid_for((size_t)s.NB * s.G * d.Cf * s.L), 256, 0, st>>>(a, out);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

static int convblock_backward_impl(const b200tts_convblock_shape& s, const float* x, const float* weight, const float* gamma,
                                   const float* beta, int affine_gstride, const uint8_t* keep, const float* saved, const float* dout,
                                   float* dx, float* dweight, float* dgamma, float* dbeta, float* ws, cudaStream_t st,
                                   const int32_t* counts = nullptr) {
    B200_TRY(validate_block(s));
    const BlockDims d = block_dims(s);
    const float* conv = s.stage == 2 ? x : saved;
    const float* mean = saved + align_up_sz(d.conv_elems, 64);
    const float* invstd = mean + align_up_sz(d.Ct, 64);
    float* col = ws;
    float* dcol = col + align_up_sz(d.col_elems, 64);
    float* dz = dcol + align_up_sz(d.col_elems, 64);
    // the per-channel sums live in the workspace whatever the stage: placed after a stage 2 dz they would land past the caller's dx
    float* s1 = dz + align_up_sz(d.conv_elems, 64);
    float* s2 = s1 + align_up_sz(d.Ct, 64);
    float* scratch = s2 + align_up_sz(d.Ct, 64);
    if (s.stage == 2) {      // batch norm only: the gradient w.r.t. the normalised input IS dx
        B200_REQUIRE(dx, "convblock_backward: stage 2 needs dx");
        dz = dx;
    }

    BlockArgs a{conv, mean, invstd, gamma, beta, affine_gstride, (s.training && s.dropout > 0.f) ? keep : nullptr,
                1.f / (1.f - s.dropout), x, s.NB, s.G, s.Cout, s.L, s.activation, s.highway, nullptr, counts};
    if (s.stage == 1) {      // convolution only: dout is the gradient of the product
        B200_CUDA(cudaMemcpyAsync(dz, dout, d.conv_elems * sizeof(float), cudaMemcpyDeviceToDevice, st));
        if (counts) {
            zero_vacant_kernel<<<grid_for(d.conv_elems), 256, 0, st>>>(dz, counts, s.NB, s.G, s.Cout, s.L);
            B200_LAUNCH_CHECK();
        }
    } else {
    const bool v4 = vec4_ok(s, d, conv, dz, x, a.keep) && (reinterpret_cast<uintptr_t>(dout) & 15) == 0 && (!s.highway || (reinterpret_cast<uintptr_t>(dx) & 15) == 0);
    if (v4)
        block_bwd_prep_vec4_kernel<<<grid_for((size_t)s.NB * s.G * d.Cf * (s.L / 4)), 256, 0, st>>>(a, dout, dz, dx);
    else
        block_bwd_prep_kernel<<<grid_for((size_t)s.NB * s.G * d.Cf * s.L), 256, 0, st>>>(a, dout, dz, dx);
    B200_LAUNCH_CHECK();
    bn_bwd_reduce_kernel<<<(int)d.Ct, 256, 0, st>>>(dz, conv, mean, invstd, s1, s2, dgamma, dbeta, affine_gstride, s.NB, s.G, s.Cout, s.L,
                                               counts);
    B200_LAUNCH_CHECK();
    if (v4)
        bn_bwd_apply_vec4_kernel<<<grid_for(d.conv_elems / 4), 256, 0, st>>>(dz, conv, mean, invstd, gamma, affine_gstride, s1, s2, s.NB, s.G,
                                                                           s.Cout, s.L, s.training, counts);
    else
        bn_bwd_apply_kernel<<<grid_for(d.conv_elems), 256, 0, st>>>(dz, conv, mean, invstd, gamma, affine_gstride, s1, s2, s.NB, s.G, s.Cout,
                                                                    s.L, s.training, counts);
    B200_LAUNCH_CHECK();
    }
    if (s.stage == 2) return B200TTS_OK;
    const float* colr = x;
    bool have_col = (s.k == 1);
    auto ensure_col = [&]() -> int {         // im2col only for the paths that still need the materialised matrix
        if (!have_col) {
            im2col1d_kernel<<<grid_for(d.col_elems), 256, 0, st>>>(col, x, (size_t)s.NB * s.G, s.Cin, s.L, s.k, s.dilation, d.pad);
            B200_LAUNCH_CHECK();
            colr = col;
            have_col = true;
        }
        return B200TTS_OK;
    };
    const int R = s.Cin * s.k;
    if (dweight) {
        // dW[g] (+)= sum_rows dconv[row, g] . col[row, g]^T
        bool fused = false;
        if (precision_mode() != 0 && s.k > 1)   // bf16 perf mode: K over (sample row, position), the shifted-input operand packed straight from x
            B200_TRY(gemm_tc_conv_dw(dz, x, dweight, s.NB, s.G, s.Cout, s.Cin, s.L, s.k, s.dilation, d.pad, st, &fused));
        if (!fused && precision_mode() != 0 && s.NB > 1) {
            // ONE batched wgmma GEMM whose K runs over (sample row, position): K = NB * L (two-level K of the packer)
            B200_TRY(ensure_col());
            GemmDesc g;
            g.A = dz; g.lda = s.L; g.transA = 0; g.strideA = (long long)s.Cout * s.L; g.kosA = (long long)d.Ct * s.L;
            g.B = colr; g.ldb = s.L; g.transB = 1; g.strideB = (long long)R * s.L; g.kosB = (long long)s.G * R * s.L;
            g.C = dweight; g.ldc = R; g.strideC = (long long)s.Cout * R; g.beta = 1.f;
            g.M = s.Cout; g.N = R; g.K = s.NB * s.L; g.kin = s.L; g.batch = s.G;
            B200_TRY(gemm_tc_try(g, st, &fused));
        }
        if (!fused) B200_TRY(ensure_col());
        // otherwise one batched GEMM per sample row, accumulating
        for (int q = 0; q < s.NB && !fused; ++q) {
            GemmDesc g;
            g.A = dz + (size_t)q * d.Ct * s.L; g.lda = s.L; g.transA = 0; g.strideA = (long long)s.Cout * s.L;
            g.B = colr + (size_t)q * s.G * R * s.L; g.ldb = s.L; g.transB = 1; g.strideB = (long long)R * s.L;
            g.C = dweight; g.ldc = R; g.strideC = (long long)s.Cout * R; g.beta = 1.f;
            g.M = s.Cout; g.N = R; g.K = s.L; g.batch = s.G;
            B200_TRY(gemm_run(g, st));
        }
    }
    if (dx) {
        GemmDesc g;     // dcol[row, g] = W[g]^T . dconv[row, g]
        g.A = weight; g.lda = R; g.transA = 1; g.a_batch_mod = s.G; g.strideA = (long long)s.Cout * R;
        g.B = dz; g.ldb = s.L; g.transB = 0; g.strideB = (long long)s.Cout * s.L;
        g.M = R; g.N = s.L; g.K = s.Cout; g.batch = s.NB * s.G;
        if (s.k == 1) {
            g.C = dx; g.ldc = s.L; g.strideC = (long long)s.Cin * s.L; g.beta = s.highway ? 1.f : 0.f;
            B200_TRY(gemm_run(g, st));
        } else {
            bool implicit = false;
            if (precision_mode() != 0)      // input gradient as an implicit (transposed) convolution of d conv: no dcol, no col2im
                B200_TRY(gemm_tc_conv(weight, dz, dx, s.NB, s.G, s.Cout, s.Cin, s.L, s.k, s.dilation, d.pad, 1, s.highway ? 1.f : 0.f, st, &implicit));
            if (implicit) return B200TTS_OK;
            B200_TRY(ensure_col());
            g.C = dcol; g.ldc = s.L; g.strideC = (long long)R * s.L;
            B200_TRY(gemm_run(g, st));
            col2im1d_kernel<<<grid_for((size_t)s.NB * s.G * s.Cin * s.L), 256, 0, st>>>(dx, dcol, (size_t)s.NB * s.G, s.Cin, s.L, s.k,
                                                                                       s.dilation, d.pad, s.highway);
            B200_LAUNCH_CHECK();
        }
    }
    (void)scratch; (void)beta;
    return B200TTS_OK;
}

// ---------------------------------------------------------------------------------------------
// parameter generator: out[g, :] = (e[g] . Wb^T + bb) . Wk^T + bk        (modules/generated.py:38-39, 81-84)
// ---------------------------------------------------------------------------------------------
// Tail of the generator backward in ONE small launch: deb = fixed-order sum of the per-block partials, then
// dWb[j, d] += sum_g deb[g, j] e[g, d];  dbb[j] += sum_g deb[g, j];  de[g, d] += sum_j deb[g, j] Wb[j, d]
__global__ void __launch_bounds__(256) generator_tail_bwd_kernel(float* __restrict__ deb, const float* __restrict__ partial, int nblk,
                                                                 const float* __restrict__ e, const float* __restrict__ Wb,
                                                                 float* __restrict__ de, float* __restrict__ dWb, float* __restrict__ dbb,
                                                                 int G, int gd, int bn) {
    __shared__ float s_deb[GEN_MAXG * GEN_MAXBN];
    __shared__ float s_part[256];
    const int n = G * bn;
    // `parts` threads per output share the nblk partials (interleaved, four accumulators each), then a fixed-order combine: deterministic
    const int parts = n <= 256 ? 256 / n : 1;
    if (n <= 256) {
        const int t = threadIdx.x % n, part = threadIdx.x / n;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        if (part < parts) {
            int b = part;
            for (; b + 3 * parts < nblk; b += 4 * parts) {
                a0 += partial[(size_t)b * n + t]; a1 += partial[(size_t)(b + parts) * n + t];
                a2 += partial[(size_t)(b + 2 * parts) * n + t]; a3 += partial[(size_t)(b + 3 * parts) * n + t];
            }
            for (; b < nblk; b += parts) a0 += partial[(size_t)b * n + t];
            s_part[threadIdx.x] = (a0 + a1) + (a2 + a3);
        }
        __syncthreads();
        if (threadIdx.x < n) {
            float v = 0.f;
            for (int q = 0; q < parts; ++q) v += s_part[q * n + threadIdx.x];
            s_deb[threadIdx.x] = v; deb[threadIdx.x] = v;
        }
    } else {
        for (int t = threadIdx.x; t < n; t += blockDim.x) {
            float v = 0.f;
            for (int b = 0; b < nblk; ++b) v += partial[(size_t)b * n + t];
            s_deb[t] = v; deb[t] = v;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < bn * gd; i += blockDim.x) {
        const int j = i / gd, d = i - j * gd;
        float a = 0.f;
        for (int g = 0; g < G; ++g) a = fmaf(s_deb[g * bn + j], e[g * gd + d], a);
        dWb[i] += a;
    }
    for (int j = threadIdx.x; j < bn; j += blockDim.x) {
        float a = 0.f;
        for (int g = 0; g < G; ++g) a += s_deb[g * bn + j];
        dbb[j] += a;
    }
    for (int i = threadIdx.x; i < G * gd; i += blockDim.x) {
        const int g = i / gd, d = i - g * gd;
        float a = 0.f;
        for (int j = 0; j < bn; ++j) a = fmaf(s_deb[g * bn + j], Wb[j * gd + d], a);
        de[i] += a;
    }
}

}  // namespace b200tts
using namespace b200tts;

extern "C" {

size_t b200tts_convblock_saved_bytes(const b200tts_convblock_shape* s) {
    if (!s) return 0;
    const BlockDims d = block_dims(*s);
    return (align_up_sz(d.conv_elems, 64) + 2 * align_up_sz(d.Ct, 64)) * sizeof(float);
}
size_t b200tts_convblock_workspace_bytes(const b200tts_convblock_shape* s) {
    if (!s) return 0;
    const BlockDims d = block_dims(*s);
    // forward: im2col.  backward: im2col + dz/dconv + dcol + s1/s2 + split-K scratch
    return (align_up_sz(d.col_elems, 64) * 2 + align_up_sz(d.conv_elems, 64) + 2 * align_up_sz(d.Ct, 64) + kGemmScratch) * sizeof(float);
}

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

size_t b200tts_generator_workspace_bytes(int G, int bn) { return (align_up_sz((size_t)G * bn, 64) + kGemmScratch) * sizeof(float); }

int b200tts_generator_forward(int G, int gd, int bn, long long R, const float* e, const float* Wb, const float* bb, const float* Wk,
                              const float* bk, float* eb, float* out, void* stream) {
    B200_REQUIRE(e && Wb && bb && Wk && bk && eb && out, "generator_forward: null argument");
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    B200_REQUIRE(G > 0 && gd > 0 && bn > 0 && R > 0 && R < (1ll << 31), "generator: bad dimensions");
    if (G <= GEN_MAXG && bn <= GEN_MAXBN) {      // skinny product, bound by reading Wk / writing the generated kernel once (bottleneck folded in)
        generator_expand_kernel<<<grid_for((size_t)R), 256, 0, st>>>(out, eb, Wk, bk, G, bn, (size_t)R, e, Wb, bb, gd);
        B200_LAUNCH_CHECK();
        return B200TTS_OK;
    }
    GemmDesc a;
    a.A = e; a.lda = gd; a.B = Wb; a.ldb = gd; a.transB = 1; a.C = eb; a.ldc = bn; a.bias = bb; a.M = G; a.N = bn; a.K = gd;
    B200_TRY(gemm_f32(a, st));
    GemmDesc b;
    b.A = eb; b.lda = bn; b.B = Wk; b.ldb = bn; b.transB = 1; b.C = out; b.ldc = (int)R; b.bias = bk; b.M = G; b.N = (int)R; b.K = bn;
    return gemm_f32(b, st);
}

int b200tts_generator_backward(int G, int gd, int bn, long long R, const float* e, const float* Wb, const float* Wk, const float* eb,
                               const float* dout, float* de, float* dWb, float* dbb, float* dWk, float* dbk, void* workspace,
                               void* stream) {
    B200_REQUIRE(e && Wb && Wk && eb && dout && de && dWb && dbb && dWk && dbk && workspace, "generator_backward: null argument");
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    float* deb = (float*)workspace;
    float* scratch = deb + align_up_sz((size_t)G * bn, 64);
    const size_t chunk = 256;
    const int nblk = (int)((R + chunk - 1) / chunk);
    if (bn == 8 && G <= GEN_FG && (reinterpret_cast<uintptr_t>(Wk) & 15) == 0 && (reinterpret_cast<uintptr_t>(dWk) & 15) == 0 &&
        !getenv("B200TTS_GENERATOR_UNFUSED")) {
        // ONE coalesced pass over dout and Wk (fused dWk / dbk / per-block deb partials), then the fixed-order reduction of the partials
        const int fblk = (int)(((size_t)R + 255) / 256 < NUM_SMS * 2 ? ((size_t)R + 255) / 256 : NUM_SMS * 2);
        generator_bwd_fused_kernel<<<fblk, 256, 0, st>>>(dWk, dbk, scratch, dout, Wk, eb, G, (size_t)R);
        B200_LAUNCH_CHECK();
        generator_tail_bwd_kernel<<<1, 256, 0, st>>>(deb, scratch, fblk, e, Wb, de, dWb, dbb, G, gd, bn);     // finish + dWb + dbb + de
        B200_LAUNCH_CHECK();
        return B200TTS_OK;
    } else if (G <= GEN_MAXG && bn <= GEN_MAXBN && (size_t)nblk * G * bn <= kGemmScratch && G * bn <= 256) {
        // dWk [R, bn] += dout^T . eb and dbk += column sums of dout, in one pass over dout
        generator_dwk_kernel<<<grid_for((size_t)R), 256, 0, st>>>(dWk, dbk, dout, eb, G, bn, (size_t)R);
        B200_LAUNCH_CHECK();
        // deb [G, bn] = dout . Wk: per-chunk partial sums, then a fixed-order reduction
        generator_deb_partial_kernel<<<nblk, 256, 0, st>>>(scratch, dout, Wk, G, bn, (size_t)R, chunk);
        B200_LAUNCH_CHECK();
        generator_deb_finish_kernel<<<G * bn, 128, 0, st>>>(deb, scratch, nblk, G * bn);
        B200_LAUNCH_CHECK();
    } else {
        GemmDesc a;     // dWk [R, bn] += dout^T . eb
        a.A = dout; a.lda = (int)R; a.transA = 1; a.B = eb; a.ldb = bn; a.transB = 0; a.C = dWk; a.ldc = bn; a.beta = 1.f;
        a.M = (int)R; a.N = bn; a.K = G;
        B200_TRY(gemm_f32(a, st));
        colsum_rows_add_kernel<<<grid_for((size_t)R), 256, 0, st>>>(dbk, dout, G, (size_t)R);
        B200_LAUNCH_CHECK();
        GemmDesc b;     // deb [G, bn] = dout . Wk   (long K: split)
        b.A = dout; b.lda = (int)R; b.B = Wk; b.ldb = bn; b.transB = 0; b.C = deb; b.ldc = bn; b.M = G; b.N = bn; b.K = (int)R;
        B200_TRY(gemm_f32_auto(b, scratch, kGemmScratch, st));
    }
    GemmDesc c;     // dWb [bn, gd] += deb^T . e
    c.A = deb; c.lda = bn; c.transA = 1; c.B = e; c.ldb = gd; c.transB = 0; c.C = dWb; c.ldc = gd; c.beta = 1.f; c.M = bn; c.N = gd; c.K = G;
    B200_TRY(gemm_f32(c, st));
    colsum_rows_add_kernel<<<1, 256, 0, st>>>(dbb, deb, G, (size_t)bn);
    B200_LAUNCH_CHECK();
    GemmDesc dd;    // de [G, gd] += deb . Wb
    dd.A = deb; dd.lda = bn; dd.B = Wb; dd.ldb = gd; dd.transB = 0; dd.C = de; dd.ldc = gd; dd.beta = 1.f; dd.M = G; dd.N = gd; dd.K = bn;
    return gemm_f32(dd, st);
}

int b200tts_embedding_forward(float* out, int ldo, const float* table, const int32_t* ids, long long ntok, int E, void* stream) {
    B200_REQUIRE(out && table && ids && ntok >= 0 && E > 0 && ldo >= E, "embedding_forward: bad argument");
    B200_TRY(require_device());
    embedding_fwd_kernel<<<grid_for((size_t)ntok * E), 256, 0, (cudaStream_t)stream>>>(out, ldo, table, ids, (size_t)ntok, E);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

int b200tts_embedding_backward(float* dtable, int V, const float* dout, int ldo, const int32_t* ids, long long ntok, int E,
                               int padding_idx, void* stream) {
    B200_REQUIRE(dtable && dout && ids && V > 0 && E > 0 && ldo >= E, "embedding_backward: bad argument");
    B200_TRY(require_device());
    B200_REQUIRE(E <= 1024, "embedding_backward: embedding dimension %d > 1024 is not supported", E);
    embedding_bwd_kernel<<<V, 256, 0, (cudaStream_t)stream>>>(dtable, dout, ldo, ids, (int)ntok, E, padding_idx);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}

}  // extern "C"
