// WaveRNN training windows cut on the device: fatchord's collate_vocoder (modules/wavernn.py vocoder_batch) for a corpus already in
// device memory, one launch per batch.
//
//   * wavernn_cut_windows_kernel: row b of the batch reads its (utterance, mel offset o) from the table and copies the mel window
//     m[b] = mel[:, o : o + mel_win] and the seq_len + 1 labels from (o + pad) hop, written as x = label_2_float(labels[:seq_len]) and
//     y = labels[1:] (RAW: int64 labels; MOL: label_2_float(., 16)).  blockIdx.y is the row; the CTAs along x stride over the row's
//     feat mel_win + seq_len outputs.
//
// label_2_float is 2 x / (2^bits - 1) - 1 in fp32 with each operation IEEE-rounded (__fmul_rn / __fdiv_rn / __fsub_rn: no contraction and no
// approximate division whatever the compile flags), which is what the host expression computes, so x and y equal vocoder_batch's bit for bit.
// The kernel reads the table unchecked: the caller validates it on the host (VocoderCorpus.batch).
#include "decoder_internal.cuh"

namespace b200tts {

namespace {

constexpr int CUT_MAX_B = 64;
constexpr int CUT_MAX_HOPS = 16;
constexpr int CUT_THREADS = 256;
constexpr int CUT_MAX_CTAS_PER_ROW = 32;

__device__ __forceinline__ float label_to_float(unsigned v, float den) {
    return __fsub_rn(__fdiv_rn(__fmul_rn(2.f, (float)v), den), 1.f);
}

__global__ void __launch_bounds__(CUT_THREADS) wavernn_cut_windows_kernel(int mol, float x_den, int feat, int win, int seq_len, int pad, int hop,
                                                                          const float* __restrict__ mels, long long total_frames,
                                                                          const long long* __restrict__ frame_start,
                                                                          const unsigned short* __restrict__ labels,
                                                                          const long long* __restrict__ sample_start,
                                                                          const int* __restrict__ table, float* __restrict__ x,
                                                                          void* __restrict__ y, float* __restrict__ m) {
    const int b = blockIdx.y;
    const int u = table[2 * b], o = table[2 * b + 1];
    const int nm = feat * win, n = nm + seq_len;
    const float* mel = mels + frame_start[u] + o;
    const unsigned short* lab = labels + sample_start[u] + (long long)(o + pad) * hop;
    for (int e = blockIdx.x * CUT_THREADS + threadIdx.x; e < n; e += gridDim.x * CUT_THREADS) {
        if (e < nm) {
            const int c = e / win, j = e - c * win;
            m[(size_t)b * nm + e] = mel[(size_t)c * total_frames + j];
        } else {
            const int t = e - nm;
            const size_t i = (size_t)b * seq_len + t;
            x[i] = label_to_float(lab[t], x_den);
            const unsigned next = lab[t + 1];
            if (mol)
                static_cast<float*>(y)[i] = label_to_float(next, 65535.f);
            else
                static_cast<long long*>(y)[i] = (long long)next;
        }
    }
}

}  // namespace

}  // namespace b200tts
using namespace b200tts;

extern "C" int b200tts_wavernn_cut_windows(int mode, int bits, int B, int feat, int seq_len, int pad, int hop, const float* mels,
                                           long long total_frames, const int64_t* frame_start, const uint16_t* labels,
                                           const int64_t* sample_start, const int32_t* table, float* x, void* y, float* m, void* stream) {
    B200_REQUIRE(mels && frame_start && labels && sample_start && table && x && y && m, "wavernn_cut_windows: null argument");
    B200_REQUIRE(mode == B200TTS_WAVERNN_RAW || mode == B200TTS_WAVERNN_MOL, "wavernn_cut_windows: unknown mode %d", mode);
    B200_REQUIRE(bits >= 1 && bits <= 16, "wavernn_cut_windows: bits %d outside [1, 16]", bits);
    B200_REQUIRE(B >= 1 && B <= CUT_MAX_B, "wavernn_cut_windows: batch %d outside [1, %d]", B, CUT_MAX_B);
    B200_REQUIRE(hop >= 1 && seq_len >= hop && seq_len % hop == 0 && seq_len / hop <= CUT_MAX_HOPS,
                 "wavernn_cut_windows: seq_len %d must be a positive multiple of the hop %d, at most %d hops", seq_len, hop, CUT_MAX_HOPS);
    B200_REQUIRE(pad >= 0 && pad <= 64, "wavernn_cut_windows: pad %d outside [0, 64]", pad);
    B200_REQUIRE(feat >= 1 && feat <= 1024, "wavernn_cut_windows: %d mel channels outside [1, 1024]", feat);
    B200_REQUIRE(total_frames >= 1, "wavernn_cut_windows: %lld packed frames", total_frames);
    B200_TRY(require_device());
    cudaStream_t st = (cudaStream_t)stream;
    const int mol = mode == B200TTS_WAVERNN_MOL;
    const float x_den = (float)((1 << (mol ? 16 : bits)) - 1);
    const int win = seq_len / hop + 2 * pad;
    const int per_row = feat * win + seq_len;
    int ctas = cdiv(per_row, CUT_THREADS);
    if (ctas > CUT_MAX_CTAS_PER_ROW) ctas = CUT_MAX_CTAS_PER_ROW;
    KernelTimer kt("wavernn_cut_windows", st);
    wavernn_cut_windows_kernel<<<dim3(ctas, B), CUT_THREADS, 0, st>>>(mol, x_den, feat, win, seq_len, pad, hop, mels, total_frames,
                                                                     reinterpret_cast<const long long*>(frame_start), labels,
                                                                     reinterpret_cast<const long long*>(sample_start), table, x, y, m);
    B200_LAUNCH_CHECK();
    return B200TTS_OK;
}
