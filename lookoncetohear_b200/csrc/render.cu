// GPU binaural renderer (SURVEY.md section 8 f-3): the data-side arithmetic that feeds the two networks, so that
// synthetic evaluation inputs can be produced at the rate the engine consumes them.
//   * per event and ear: causal FIR with the head-related / room impulse response, truncated to the source length --
//     SOFASimulator._convolve, reference src/datasets/multi_ch_simulator.py:56-58
//     (`convolve(src, rir[0])[:len(src)]`, `convolve(src, rir[1])[:len(src)]`);
//   * mixture assembly -- reference src/datasets/MixLibriSpeechNoisyEnrollNorm.py:179-202: noise scaled by
//     `noise_scale`, `norm_factor = |sum(events) + noise|.max()`; if it exceeds 1 every event and the noise are
//     divided by it; `mixture = sum(events) + noise`.
// Direct-form convolution in fp32 on the CUDA cores (HRIRs are a few hundred taps, BRIRs a few thousand: 2 n_src N L
// MACs per mixture is microseconds of GPU time); one CTA = 1024 output samples of one (mixture, event, ear).
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>

#include "../../include/lookonce_b200.h"
#include "host_errors.h"
#include "common.cuh"

namespace l2h {

constexpr int FIR_TILE = 1024, FIR_CHUNK = 256;

__global__ void __launch_bounds__(256)
fir_kernel(const float* __restrict__ src, const float* __restrict__ rir, float* __restrict__ out, int n_src, int n, int rir_len) {
    __shared__ float xs[FIR_TILE + FIR_CHUNK];       // source samples n0 - (k0 + CHUNK - 1) .. n0 + TILE - 1 - k0
    __shared__ float hs[FIR_CHUNK];
    const int tid = threadIdx.x;
    const int n0 = blockIdx.x * FIR_TILE, se = blockIdx.y, b = blockIdx.z;
    const int s = se >> 1;
    const float* x = src + ((int64_t)b * n_src + s) * n;
    const float* h = rir + ((int64_t)b * n_src * 2 + se) * rir_len;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int k0 = 0; k0 < rir_len; k0 += FIR_CHUNK) {
        __syncthreads();
        const int base = n0 - k0 - (FIR_CHUNK - 1);            // xs[i] = x[base + i]
        for (int i = tid; i < FIR_TILE + FIR_CHUNK - 1; i += 256) {
            const int idx = base + i;
            xs[i] = (idx >= 0 && idx < n) ? x[idx] : 0.f;
        }
        for (int i = tid; i < FIR_CHUNK; i += 256) hs[i] = (k0 + i < rir_len) ? h[k0 + i] : 0.f;
        __syncthreads();
        // outputs o = n0 + 4*tid + j;  y[o] += sum_kk h[k0+kk] * x[o - k0 - kk];  x[o - k0 - kk] = xs[4*tid + j + CHUNK-1 - kk]
        const int p = 4 * tid + FIR_CHUNK - 1;
        float w0 = xs[p], w1 = xs[p + 1], w2 = xs[p + 2], w3 = xs[p + 3];
#pragma unroll 8
        for (int kk = 0; kk < FIR_CHUNK; ++kk) {
            const float hv = hs[kk];
            acc[0] = fmaf(hv, w0, acc[0]); acc[1] = fmaf(hv, w1, acc[1]);
            acc[2] = fmaf(hv, w2, acc[2]); acc[3] = fmaf(hv, w3, acc[3]);
            w3 = w2; w2 = w1; w1 = w0;
            w0 = (kk + 1 < FIR_CHUNK) ? xs[p - kk - 1] : 0.f;
        }
    }
    float* y = out + ((int64_t)b * n_src * 2 + se) * n;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int o = n0 + 4 * tid + j;
        if (o < n) y[o] = acc[j];
    }
}

// peak of |sum(events) + scale * noise| per mixture -> norm[b] (float bits, non-negative: integer max works)
__global__ void __launch_bounds__(256)
mix_peak_kernel(const float* __restrict__ ev, const float* __restrict__ noise, const float* __restrict__ nscale, int n_src, int n,
                unsigned int* __restrict__ peak) {
    __shared__ float red[8];
    const int b = blockIdx.y, tid = threadIdx.x;
    const float sc = nscale ? nscale[b] : 1.f;
    float mx = 0.f;
    for (int64_t i = (int64_t)blockIdx.x * 256 + tid; i < (int64_t)2 * n; i += (int64_t)gridDim.x * 256) {
        float v = noise ? sc * noise[(int64_t)b * 2 * n + i] : 0.f;
        for (int s = 0; s < n_src; ++s) v += ev[((int64_t)b * n_src + s) * 2 * n + i];
        mx = fmaxf(mx, fabsf(v));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((tid & 31) == 0) red[tid >> 5] = mx;
    __syncthreads();
    if (tid == 0) {
        for (int k = 1; k < 8; ++k) mx = fmaxf(mx, red[k]);
        atomicMax(peak + b, __float_as_uint(mx));
    }
}

// divide by the peak when it exceeds 1 (events in place, scaled noise into the mixture), mixture = sum + noise
__global__ void __launch_bounds__(256)
mix_norm_kernel(float* __restrict__ ev, const float* __restrict__ noise, const float* __restrict__ nscale, int n_src, int n,
                const unsigned int* __restrict__ peak, float* __restrict__ mixture, float* __restrict__ norm_out) {
    const int b = blockIdx.y, tid = threadIdx.x;
    const float pk = __uint_as_float(peak[b]);
    const float nf = pk > 1.f ? pk : 1.f;
    const float sc = (nscale ? nscale[b] : 1.f) / nf;
    if (blockIdx.x == 0 && tid == 0 && norm_out) norm_out[b] = nf;
    for (int64_t i = (int64_t)blockIdx.x * 256 + tid; i < (int64_t)2 * n; i += (int64_t)gridDim.x * 256) {
        float v = noise ? sc * noise[(int64_t)b * 2 * n + i] : 0.f;
        for (int s = 0; s < n_src; ++s) {
            float* e = ev + ((int64_t)b * n_src + s) * 2 * n + i;
            const float x = *e / nf;
            *e = x;
            v += x;
        }
        mixture[(int64_t)b * 2 * n + i] = v;
    }
}
}  // namespace l2h

extern "C" int l2h_render_binaural(const float* src_dev, const float* rir_dev, const float* noise_dev, const float* noise_scale_dev,
                                   int32_t batch, int32_t n_src, int32_t n_samples, int32_t rir_len, float* events_dev,
                                   float* mixture_dev, float* norm_dev, void* scratch_dev, void* stream) {
    using namespace l2h;
    if (!src_dev || !rir_dev || !events_dev || !mixture_dev || !scratch_dev || batch <= 0 || n_src <= 0 || n_samples <= 0 || rir_len <= 0)
        return fail(1, "l2h_render_binaural: bad argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    unsigned int* peak = static_cast<unsigned int*>(scratch_dev);          // batch words
    cudaError_t e = cudaMemsetAsync(peak, 0, sizeof(unsigned int) * batch, st);
    if (e == cudaSuccess) {
        fir_kernel<<<dim3((n_samples + FIR_TILE - 1) / FIR_TILE, 2 * n_src, batch), 256, 0, st>>>(src_dev, rir_dev, events_dev, n_src, n_samples, rir_len);
        e = cudaGetLastError();
    }
    const int gx = (int)((2ll * n_samples + 255) / 256 < NUM_SMS ? (2ll * n_samples + 255) / 256 : NUM_SMS);
    if (e == cudaSuccess) {
        mix_peak_kernel<<<dim3(gx, batch), 256, 0, st>>>(events_dev, noise_dev, noise_scale_dev, n_src, n_samples, peak);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        mix_norm_kernel<<<dim3(gx, batch), 256, 0, st>>>(events_dev, noise_dev, noise_scale_dev, n_src, n_samples, peak, mixture_dev, norm_dev);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) return fail(3, std::string("l2h_render_binaural: ") + cudaGetErrorString(e));
    return 0;
}
