// Band-limited resampling on the device: torchaudio.functional.resample(x, orig, new) at its defaults (Hann-windowed
// sinc, lowpass_filter_width 6, rolloff 0.99), the only form the reference uses -- impulse responses from the rate of
// their SOFA / BRIR file to the dataset rate (src/datasets/multi_ch_simulator.py:49) and the dataset's resample_rate
// step (MixLibriSpeechNoisyEnrollNorm.py:69-75).
//
// Rates reduced by their gcd to o (input samples) and q (output samples) per common period; cutoff base = min(o, q) *
// 0.99 cycles per period.  Output m sits at time m / q, input n at n / o:
//     y[m] = sum_n x[n] * (base / o) * sinc(u) * cos^2(pi u / 12),   u = base * (m / q - n / o),   |u| < 6,
// i.e. the taps n = floor(m o / q) - w .. floor(m o / q) + w with w = ceil(6 o / base).  The taps are computed on the
// device from (phase, tap, rates) -- no filter table -- with u in fp64 (its fraction decides the weight) and the
// sinc / window in fp32; accumulation in fp32.
//
// One CTA = up to RS_TILE consecutive outputs of one row (one thread per output).  It stages the input window of its
// outputs in shared memory once (RS_TILE * o / q + 2 w + 2 samples), so each tap is a shared-memory read.  Rows carry
// their own `orig`: a launch takes, as its kernel parameter, a table of up to RS_MAX_RATES distinct rates and up to
// RS_MAX_RUNS runs of consecutive rows with the same rate (no per-row table in device memory); a CTA finds its row's
// run by binary search.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <numeric>
#include <string>

#include "../../include/lookonce_b200.h"
#include "host_errors.h"

namespace l2h {

constexpr int RS_TILE = 256;              // outputs (threads) per CTA
constexpr int RS_MAX_RATES = 16;          // distinct `orig` per launch
constexpr int RS_MAX_RUNS = 768;          // runs of equal `orig` per launch (the parameter block stays under 4 KB)
constexpr int RS_MAX_ROWS = 65535;        // rows per launch (grid.y)
constexpr int RS_SMEM_BYTES = 48 * 1024;  // staged input window per CTA
constexpr int RS_WIDTH = 6;               // zero crossings of the sinc on each side (lowpass_filter_width)
constexpr double RS_ROLLOFF = 0.99;

struct RsRate {
    int32_t o, q;   // reduced rates; o == q (== 1): the row is copied
    int32_t w;      // taps on each side of floor(m o / q)
    int32_t n_out;  // ceil(q n_in / o)
    float scale;    // base / o
    double du;      // base / o: step of u from one tap to the next
    double du_r;    // base / (o q): u per unit of the remainder (m o) mod q
};
struct RsLaunch {
    int32_t n_run;
    uint32_t run[RS_MAX_RUNS];  // (first row, relative to the launch) << 8 | index into rate[]
    RsRate rate[RS_MAX_RATES];
};

__global__ void __launch_bounds__(RS_TILE)
resample_kernel(const float* __restrict__ x, int64_t x_stride, int n_in, float* __restrict__ y, int64_t y_stride, int cap,
                const __grid_constant__ RsLaunch L) {
    extern __shared__ float xs[];
    const int row = blockIdx.y, tid = threadIdx.x;
    int lo_run = 0, hi_run = L.n_run - 1;                       // the last run that starts at or before `row`
    while (lo_run < hi_run) {
        const int mid = (lo_run + hi_run + 1) >> 1;
        if ((int)(L.run[mid] >> 8) <= row) lo_run = mid; else hi_run = mid - 1;
    }
    const RsRate& g = L.rate[L.run[lo_run] & 0xffu];
    const float* xr = x + (int64_t)row * x_stride;
    float* yr = y + (int64_t)row * y_stride;
    const int m0 = blockIdx.x * blockDim.x, m = m0 + tid;
    if (g.o == g.q) {                                           // equal rates: the input, bit for bit, then zeros
        if (m < cap) yr[m] = m < n_in ? xr[m] : 0.f;
        return;
    }
    const int m_last = min(m0 + (int)blockDim.x, g.n_out) - 1;
    int64_t lo = 0;
    if (m0 <= m_last) {                                         // stage x[lo .. hi], zero outside the row
        lo = (int64_t)m0 * g.o / g.q - g.w;
        const int cnt = (int)((int64_t)m_last * g.o / g.q + g.w + 1 - lo);
        for (int i = tid; i < cnt; i += blockDim.x) {
            const int64_t n = lo + i;
            xs[i] = (n >= 0 && n < n_in) ? xr[n] : 0.f;
        }
    }
    __syncthreads();
    if (m >= cap) return;
    float acc = 0.f;
    if (m < g.n_out) {
        const int64_t mo = (int64_t)m * g.o, c = mo / g.q;
        const double u0 = (double)(mo - c * g.q) * g.du_r + g.w * g.du;    // u of tap n = c - w
        const float* xp = xs + (c - g.w - lo);
        for (int t = 0; t <= 2 * g.w; ++t) {
            const float u = (float)fma(-(double)t, g.du, u0);
            if (fabsf(u) < (float)RS_WIDTH) {
                const float sinc = u == 0.f ? 1.f : sinpif(u) / (3.14159265358979f * u);
                const float win = 0.5f + 0.5f * cospif(u * (1.f / RS_WIDTH));     // cos^2(pi u / 12)
                acc = fmaf(g.scale * sinc * win, xp[t], acc);
            }
        }
    }
    yr[m] = acc;
}
}  // namespace l2h

extern "C" int l2h_resample(const float* x_dev, int64_t x_row_stride, int32_t n_in, int32_t n_rows, const int32_t* orig_freq,
                            int32_t new_freq, float* y_dev, int64_t y_row_stride, int32_t y_capacity, void* stream) {
    using namespace l2h;
    if (!x_dev || !y_dev || !orig_freq || n_rows <= 0 || n_in < 0 || x_row_stride < n_in || y_capacity < 0 ||
        y_row_stride < y_capacity)
        return fail(1, "l2h_resample: bad argument");
    if (new_freq <= 0) return fail(1, "l2h_resample: new_freq " + std::to_string(new_freq) + " is not positive");
    // every row is checked before anything is launched
    for (int32_t r = 0; r < n_rows; ++r) {
        const int32_t orig = orig_freq[r];
        if (orig <= 0) return fail(1, "l2h_resample: row " + std::to_string(r) + ": orig_freq " + std::to_string(orig) + " is not positive");
        if (r > 0 && orig == orig_freq[r - 1]) continue;
        const int64_t n_out = ((int64_t)new_freq * n_in + orig - 1) / orig;
        if (n_out > y_capacity)
            return fail(1, "l2h_resample: row " + std::to_string(r) + " (" + std::to_string(orig) + " -> " + std::to_string(new_freq) +
                               " Hz) has " + std::to_string(n_out) + " output samples, capacity " + std::to_string(y_capacity));
        const int32_t gd = std::gcd(orig, new_freq), o = orig / gd, q = new_freq / gd;
        const int64_t w = (int64_t)std::ceil(RS_WIDTH * (double)o / (std::min(o, q) * RS_ROLLOFF));
        if ((((int64_t)(RS_TILE - 1) * o) / q + 2 * w + 2) * (int64_t)sizeof(float) > RS_SMEM_BYTES)
            return fail(2, "l2h_resample: reduced rate ratio " + std::to_string(o) + "/" + std::to_string(q) + " (" + std::to_string(orig) +
                               " -> " + std::to_string(new_freq) + " Hz) is too large: the input window of a tile exceeds shared memory");
    }
    if (y_capacity == 0) return 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int threads = std::min(RS_TILE, (y_capacity + 31) / 32 * 32);
    static_assert(sizeof(RsLaunch) + 64 <= 4096, "kernel parameters");
    RsLaunch L;
    int32_t rate_hz[RS_MAX_RATES];                              // orig of L.rate[i]
    int n_rates = 0, smem = 0;
    int32_t row0 = 0;
    L.n_run = 0;
    auto launch = [&](int32_t row_end) {
        resample_kernel<<<dim3((y_capacity + threads - 1) / threads, row_end - row0), threads, smem, st>>>(
            x_dev + row0 * x_row_stride, x_row_stride, n_in, y_dev + row0 * y_row_stride, y_row_stride, y_capacity, L);
        return cudaGetLastError();
    };
    cudaError_t e = cudaSuccess;
    for (int32_t r = 0; r < n_rows && e == cudaSuccess; ++r) {
        const int32_t orig = orig_freq[r];
        const bool same = L.n_run > 0 && orig == orig_freq[r - 1];
        int idx = 0;
        while (idx < n_rates && rate_hz[idx] != orig) ++idx;
        if (L.n_run > 0 && (r - row0 == RS_MAX_ROWS || (!same && (L.n_run == RS_MAX_RUNS || idx == RS_MAX_RATES)))) {
            e = launch(r);
            L.n_run = n_rates = smem = idx = 0;
            row0 = r;
        } else if (same) {
            continue;
        }
        L.run[L.n_run++] = (uint32_t)(r - row0) << 8 | (uint32_t)idx;
        if (idx < n_rates) continue;
        const int32_t gd = std::gcd(orig, new_freq);
        RsRate& g = L.rate[n_rates];
        rate_hz[n_rates++] = orig;
        g.o = orig / gd;
        g.q = new_freq / gd;
        const double base = std::min(g.o, g.q) * RS_ROLLOFF;
        g.w = (int32_t)std::ceil(RS_WIDTH * (double)g.o / base);
        g.n_out = (int32_t)(((int64_t)new_freq * n_in + orig - 1) / orig);
        g.scale = (float)(base / g.o);
        g.du = base / g.o;
        g.du_r = base / ((double)g.o * g.q);
        if (g.o != g.q) smem = std::max(smem, (int)((((int64_t)(threads - 1) * g.o) / g.q + 2 * g.w + 2) * sizeof(float)));
    }
    if (e == cudaSuccess) e = launch(n_rows);
    if (e != cudaSuccess) return fail(3, std::string("l2h_resample: ") + cudaGetErrorString(e));
    return 0;
}
