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
//
// The file also holds the per-slot stages of the serving front end, which share one scaffold: on the device slot_row
// and row_ch find a call row's state and operands, row_hops and row_pushed its hop or sample count, int_word, clamp_word
// and add_word read and count state words, and hop_gain turns a hop's dB gains into sample gains; on the host slot_call,
// disjoint, overlap, hop_lens and staging check a call before it is launched, and launched after.  The stages are the
// streaming resamplers (pushes of whole periods, resample_stream_kernel; pushes of any length,
// resample_packets_kernel), the hop FIFO that turns 16 kHz pieces into separator chunks (hop_fifo_kernel), the
// enrollment capture (enroll_capture_kernel), the target mixer that sums a listener's separated voices and its ambient
// mixture into one row (target_mix_kernel, target_mix_set_kernel), the look-ahead limiter that keeps each listener's
// output under a ceiling with one gain for all channels (limiter_kernel), the leveler that brings each voice to one
// loudness with one gain for all channels (leveler_kernel), and the multiband compressor that fits each listener's output
// to their hearing, per band and per ear, with its compression linked across the channels (band_compressor_kernel), and
// the jitter buffer that puts a device's packets back in sequence order and conceals lost ones (jitter_buffer_kernel, and
// jitter_buffer_kernel_t<true>, which also releases missing packets on deadlines from the server's clock).
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <initializer_list>
#include <numeric>
#include <string>
#include <utility>
#include <vector>

#include "../../include/lookonce_b200.h"
#include "host_errors.h"
#include "enroll_capture.cuh"
#include "sep_layout.h"

namespace l2h {

constexpr int RS_TILE = 256;              // outputs (threads) per CTA
constexpr int RS_MAX_RATES = 16;          // distinct `orig` per launch
constexpr int RS_MAX_RUNS = 768;          // runs of equal `orig` per launch (the parameter block stays under 4 KB)
constexpr int RS_MAX_ROWS = 65535;        // rows per launch (grid.y)
constexpr int RS_SMEM_BYTES = 48 * 1024;  // staged input window per CTA
constexpr int RS_WIDTH = 6;               // zero crossings of the sinc on each side (lowpass_filter_width)
constexpr double RS_ROLLOFF = 0.99;
static_assert(CHUNK_HOP == HOP && CHUNK_CARRY == LOOKAHEAD, "the FIFO and the capture cut the separator's chunks");

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

// One output sample: the 2w + 1 taps xp[0 .. 2w] (input samples c - w .. c + w, c = floor(m o / q)) weighted for the
// phase r = (m o) mod q.  Tap t = 0 always has u >= w du >= 6, so xp[0] never enters the sum.  Both kernels call this,
// so a streamed sample is the whole-signal sample bit for bit.
__device__ __forceinline__ float rs_output(const float* xp, int64_t r, const RsRate& g) {
    const double u0 = (double)r * g.du_r + g.w * g.du;                // u of tap n = c - w
    float acc = 0.f;
    for (int t = 0; t <= 2 * g.w; ++t) {
        const float u = (float)fma(-(double)t, g.du, u0);
        if (fabsf(u) < (float)RS_WIDTH) {
            const float sinc = u == 0.f ? 1.f : sinpif(u) / (3.14159265358979f * u);
            const float win = 0.5f + 0.5f * cospif(u * (1.f / RS_WIDTH));     // cos^2(pi u / 12)
            acc = fmaf(g.scale * sinc * win, xp[t], acc);
        }
    }
    return acc;
}

// the filter of orig -> new_freq Hz for rows of n_in samples (n_out 0 when n_in is not known)
static RsRate rs_rate(int32_t orig, int32_t new_freq, int32_t n_in) {
    RsRate g;
    const int32_t gd = std::gcd(orig, new_freq);
    g.o = orig / gd;
    g.q = new_freq / gd;
    const double base = std::min(g.o, g.q) * RS_ROLLOFF;
    g.w = (int32_t)std::min(std::ceil(RS_WIDTH * (double)g.o / base), (double)INT32_MAX);   // refused by the size checks
    g.n_out = (int32_t)(((int64_t)new_freq * n_in + orig - 1) / orig);
    g.scale = (float)(base / g.o);
    g.du = base / g.o;
    g.du_r = base / ((double)g.o * g.q);
    return g;
}

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
        acc = rs_output(xs + (c - g.w - lo), mo - c * g.q, g);
    }
    yr[m] = acc;
}

// ---- the per-slot scaffold -------------------------------------------------------------------------------------------
// A per-slot stage keeps a state [n_slots][C][row_floats], all zeros for a fresh slot, and runs one CTA per (call row,
// channel), or per call row where its channels share a gain.  The slot, hop and count lists are read on the device: a
// row whose slot lies outside the state, whose hop count lies outside [1, T] or whose push lies outside [0, max_in]
// stores nothing.
struct SlotRow {
    int row, ch;
    bool live;   // the row's slot lies inside the state
    float* st;   // its state row of channel ch (when live)
};

L2H_DEVINL SlotRow slot_row(int C, const int32_t* slots, int n_slots, float* state, int64_t row_floats) {
    const int row = blockIdx.x / C, ch = blockIdx.x - row * C, slot = slots[row];
    return {row, ch, !(slot < 0 || slot >= n_slots), state + ((int64_t)slot * C + ch) * row_floats};
}

// row `row`, channel `ch` of a strided [n][C][*] tensor
template <class T>
L2H_DEVINL T* row_ch(T* p, int64_t row_stride, int64_t ch_stride, int row, int ch) {
    return p + (int64_t)row * row_stride + (int64_t)ch * ch_stride;
}

// the hops row `row` takes, hops[row] (T without a hop list): 0 for a count outside [1, T], a row that stores nothing
L2H_DEVINL int row_hops(const int32_t* hops, int row, int T) {
    const int h = hops ? hops[row] : T;
    return h >= 1 && h <= T ? h : 0;
}

// the samples row `row` pushes, counts[row] * unit: 0 for a push outside [0, max_in], a push of nothing
L2H_DEVINL int row_pushed(const int32_t* counts, int row, int unit, int max_in) {
    const int64_t pushed = (int64_t)counts[row] * unit;
    return pushed >= 0 && pushed <= max_in ? (int)pushed : 0;
}

// a count word of a state row, stored as a float, clamped into [0, hi]
L2H_DEVINL int clamp_word(float v, int hi) { return v >= (float)hi ? hi : (v > 0.f ? (int)v : 0); }

// an int32 word of a state row, clamped into [0, hi]
L2H_DEVINL int int_word(float w, int hi) { return min(max(__float_as_int(w), 0), hi); }

// the int32 counter word w (a negative one counts as 0) plus add >= 0, saturating at INT32_MAX
L2H_DEVINL float add_word(float w, int add) {
    const int before = max(__float_as_int(w), 0);
    return __int_as_float(add > INT32_MAX - before ? INT32_MAX : before + add);
}

// The leveler's and the compressor's gains are in dB, interpolated across each hop.  A sample of magnitude HG_BIG (2^32)
// or more is not measured: its squares could overflow.
constexpr float HG_BIG = 4294967296.f;
constexpr float HG_LOG2_10_20 = 0.16609640474436813f;   // log2(10) / 20: dB to an octave of amplitude

// the linear gain of the calling thread's sample k = threadIdx.x + 1 of a hop (one thread per sample), interpolated in dB
// from g0 at the hop's start to g1 at its end; a gain of 0 dB is exactly 1
L2H_DEVINL float hop_gain(float g0, float g1) {
    const float gk = fmaf(g1 - g0, (float)(threadIdx.x + 1) * (1.f / CHUNK_HOP), g0);
    return gk == 0.f ? 1.f : exp2f(gk * HG_LOG2_10_20);
}

// Sample jd + D of the delayed output z' below: zero before z's start (!started), else rs_output at input c = floor(jd o /
// q), which sits at win[origin + c].
L2H_DEVINL float rs_delayed(const float* win, int origin, int64_t jd, bool started, const RsRate& g) {
    if (!started) return 0.f;
    const int64_t a = jd * g.o;
    const int64_t c = a >= 0 ? a / g.q : -((-a + g.q - 1) / g.q);       // floor(a / q)
    return rs_output(win + (origin + c - g.w), a - c * g.q, g);
}

// ---- streaming: per-slot state, pushes of `block` input samples ------------------------------------------------------
// A stream's output is the whole-signal output z of everything it was pushed, delayed by D = floor(w q / o) samples
// (z'[j] = z[j - D], zero before z's start): after k pushes exactly the k * out_block - D samples of z whose taps have all
// arrived are final.  A slot's state row per channel is [H + keep] floats: the last H = ceil(D o / q) + w input samples,
// which the next push's outputs read, then the last `keep` outputs.  The oldest history word sits under tap 0 of the
// push's first output only, which always weighs zero (rs_output), so it holds the number of outputs the stream has made,
// capped at D, instead: a zeroed row is a fresh stream and knows which of its first outputs precede z's start.
struct RsStream {
    RsRate g;
    int32_t block, out_block;  // input samples per push (a multiple of o) and the outputs each push yields
    int32_t delay, hist, keep; // D, H and the output samples repeated from the previous call
};

// One CTA = one (call row, channel): stage the slot's history and the row's h pushes, compute the h * out_block outputs
// with their absolute phase ((j - D) o mod q: pushes are whole periods), write keep + outputs, then store the new history
// and keep tail.  A slot is listed once per call, so no other CTA touches its rows.
__global__ void __launch_bounds__(RS_TILE)
resample_stream_kernel(const float* __restrict__ x, int64_t x_row, int64_t x_ch, float* __restrict__ y, int64_t y_row,
                       int64_t y_ch, int C, int T, const int32_t* __restrict__ slots, const int32_t* __restrict__ hops,
                       float* __restrict__ state, int n_slots, const __grid_constant__ RsStream s) {
    extern __shared__ float sm[];
    const int tid = threadIdx.x, H = s.hist, keep = s.keep, D = s.delay;
    const SlotRow r = slot_row(C, slots, n_slots, state, H + keep);
    const int h = row_hops(hops, r.row, T);
    if (h == 0 || !r.live) return;                                      // a row that stores nothing
    const int n_win = H + h * s.block, n_new = h * s.out_block;
    float* st = r.st;
    const float* xr = row_ch(x, x_row, x_ch, r.row, r.ch);
    float* yr = row_ch(y, y_row, y_ch, r.row, r.ch);
    float* win = sm;                                 // [H + h * block]: the history, then the row's new samples
    float* out = sm + H + T * s.block;               // [keep + h * out_block]: the keep tail, then the new outputs
    const int before = clamp_word(st[0], D);
    for (int i = tid; i < n_win; i += blockDim.x) win[i] = i == 0 ? 0.f : (i < H ? st[i] : xr[i - H]);
    for (int i = tid; i < keep; i += blockDim.x) out[i] = st[H + i];
    __syncthreads();
    // win[H] is x[0] of the push: output j centres on x[floor((j - D) o / q)]
    for (int j = tid; j < n_new; j += blockDim.x) out[keep + j] = rs_delayed(win, H, j - D, before + j >= D, s.g);
    __syncthreads();
    for (int i = tid; i < keep + n_new; i += blockDim.x) yr[i] = out[i];
    for (int i = tid; i < H + keep; i += blockDim.x)
        st[i] = i == 0 ? (float)min(D, before + n_new) : (i < H ? win[n_win - H + i] : out[n_new + i - H]);
}

static std::string rs_rates(int32_t orig, int32_t new_freq) { return std::to_string(orig) + " -> " + std::to_string(new_freq) + " Hz"; }

// the shared-memory bytes of a per-slot call that stages `floats` per row, into *smem unless it is null (a layout
// query): 0, or 2 when they exceed shared memory, with the message "who: what: <floats> staged <unit> exceed ...""
static int staging(const std::string& who, int64_t floats, const std::string& what, const char* unit, int* smem) {
    if (floats * (int64_t)sizeof(float) > RS_SMEM_BYTES)
        return fail(2, who + ": " + what + ": " + std::to_string(floats) + " staged " + unit + " exceed shared memory (" +
                           std::to_string(RS_SMEM_BYTES / sizeof(float)) + ")");
    if (smem) *smem = (int)(floats * sizeof(float));
    return 0;
}

// Lets `kernel` take RS_SMEM_BYTES of dynamic shared memory on the current device.  A kernel with static shared memory
// of its own cannot launch by default when the two together pass 48 KB, which a staging just under RS_SMEM_BYTES does.
template <class Kernel>
static cudaError_t full_staging(Kernel kernel) {
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, RS_SMEM_BYTES);
}

// the filter of a stream of orig -> new_freq Hz and its delay D = floor(w q / o): 0, or 1 with its message
static int rs_streaming(const std::string& who, int32_t orig, int32_t new_freq, RsRate* g, int64_t* delay) {
    if (orig <= 0 || new_freq <= 0) return fail(1, who + ": rates must be positive, got " + rs_rates(orig, new_freq));
    if (orig == new_freq) return fail(1, who + ": " + rs_rates(orig, new_freq) + " needs no resampling");
    *g = rs_rate(orig, new_freq, 0);
    *delay = (int64_t)g->w * g->q / g->o;
    return 0;
}

// the stream of orig -> new_freq Hz in pushes of `block` samples with `keep` repeated outputs, for calls of up to `blocks`
// pushes per row, and the bytes of a row's window: 0, or an error code (1 invalid, 2 the window exceeds shared memory)
// with its message
static int rs_stream(const std::string& who, int32_t orig, int32_t new_freq, int32_t block, int32_t keep, int32_t blocks,
                     RsStream* s, int* smem) {
    int64_t delay;
    if (int rc = rs_streaming(who, orig, new_freq, &s->g, &delay)) return rc;
    const RsRate& g = s->g;
    const std::string rates = rs_rates(orig, new_freq);
    if (block <= 0 || block % g.o != 0)
        return fail(1, who + ": block " + std::to_string(block) + " is not a positive multiple of " + std::to_string(g.o) +
                           ", the input samples of one period of " + rates);
    if (keep < 0) return fail(1, who + ": keep " + std::to_string(keep) + " is negative");
    const int64_t out_block = (int64_t)block / g.o * g.q;
    const int64_t hist = (delay * g.o + g.q - 1) / g.q + g.w;
    const int64_t floats = hist + (int64_t)blocks * block + keep + (int64_t)blocks * out_block;
    const std::string what = rates + " in blocks of " + std::to_string(block) + " with keep " + std::to_string(keep) +
                             " and " + std::to_string(blocks) + " blocks per row is too large";
    if (int rc = staging(who, floats, what, "samples per row", smem)) return rc;
    s->block = block;
    s->out_block = (int32_t)out_block;
    s->delay = (int32_t)delay;
    s->hist = (int32_t)hist;
    s->keep = keep;
    return 0;
}

// ---- packets: pushes of any number of samples ------------------------------------------------------------------------
// A stream pushed N samples in all has returned floor(N q / o) of them, each the sample of z' above (the same D).  Output j
// reads taps up to floor((j - D) o / q) + w, and D o / q >= w - (o - 1) / q, so every tap of j <= floor(N q / o) - 1 has
// arrived.  Relative to the last period boundary at or before the stream's input count N0 (phase p = N0 mod o), the push
// makes the outputs floor(p q / o) .. floor((p + n) q / o) - 1, so the phase is all the clock a stream needs.  A state row
// per channel is [RP_HEAD + H]: the outputs made (capped at D) and the phase, exact in floats, then the last H = ceil((D +
// 1) o / q) + w + 1 input samples, enough for the taps of a push's first output at any phase.
constexpr int RP_HEAD = 2;

struct RsPackets {
    RsRate g;
    int32_t delay, hist;       // D, H
    int32_t max_in, unit;      // row i pushes counts[i] * unit samples, counted as 0 outside [0, max_in]
};

// One CTA = one (call row, channel): stage the slot's history and the row's new samples, compute the new outputs with
// their phase relative to the period boundary, write them, then store the new history, phase and count.
__global__ void __launch_bounds__(RS_TILE)
resample_packets_kernel(const float* __restrict__ x, int64_t x_row, int64_t x_ch, float* __restrict__ y, int64_t y_row,
                        int64_t y_ch, int C, const int32_t* __restrict__ counts, int32_t* __restrict__ out_counts,
                        const int32_t* __restrict__ slots, float* __restrict__ state, int n_slots,
                        const __grid_constant__ RsPackets s) {
    extern __shared__ float win[];                   // [H + n]: the history, then the row's new samples
    const int tid = threadIdx.x, H = s.hist, D = s.delay;
    const SlotRow r = slot_row(C, slots, n_slots, state, RP_HEAD + H);
    const int n = row_pushed(counts, r.row, s.unit, s.max_in);
    if (!r.live || n == 0) {                                            // a row that stores nothing
        if (r.ch == 0 && tid == 0) out_counts[r.row] = 0;
        return;
    }
    const RsRate& g = s.g;
    float* st = r.st;
    const int before = clamp_word(st[0], D), p = clamp_word(st[1], g.o - 1);
    const int64_t j0 = (int64_t)p * g.q / g.o;                         // the push's outputs j0 .. j0 + n_new - 1
    const int n_new = (int)((int64_t)(p + n) * g.q / g.o - j0);
    if (r.ch == 0 && tid == 0) out_counts[r.row] = n_new;
    const float* xr = row_ch(x, x_row, x_ch, r.row, r.ch);
    float* yr = row_ch(y, y_row, y_ch, r.row, r.ch);
    for (int i = tid; i < H + n; i += blockDim.x) win[i] = i < H ? st[RP_HEAD + i] : xr[i - H];
    __syncthreads();
    // win[H - p] is the input at the period boundary: output j (relative to it) centres on its input c = floor((j - D) o / q)
    for (int k = tid; k < n_new; k += blockDim.x) yr[k] = rs_delayed(win, H - p, j0 + k - D, before + k >= D, g);
    for (int i = tid; i < H; i += blockDim.x) st[RP_HEAD + i] = win[n + i];
    if (tid == 0) {
        st[0] = (float)min(D, before + n_new);
        st[1] = (float)((p + n) % g.o);
    }
}

// the packet stream of orig -> new_freq Hz for pushes of up to max_in samples, and the bytes of a row's window: 0, or an
// error code (1 invalid, 2 the window exceeds shared memory) with its message
static int rs_packets(const std::string& who, int32_t orig, int32_t new_freq, int32_t max_in, RsPackets* s,
                      int32_t* max_out, int* smem) {
    int64_t delay;
    if (int rc = rs_streaming(who, orig, new_freq, &s->g, &delay)) return rc;
    if (max_in <= 0) return fail(1, who + ": max_in " + std::to_string(max_in) + " is not positive");
    const RsRate& g = s->g;
    const int64_t hist = ((delay + 1) * g.o + g.q - 1) / g.q + g.w + 1;
    const int64_t out = ((int64_t)max_in * g.q + g.o - 1) / g.o;
    if (int rc = staging(who, hist + max_in, rs_rates(orig, new_freq) + " in pushes of up to " + std::to_string(max_in) +
                                                 " samples is too large", "samples per row (history and push)", smem))
        return rc;
    s->delay = (int32_t)delay;
    s->hist = (int32_t)hist;
    s->max_in = max_in;
    *max_out = (int32_t)out;
    return 0;
}

// ---- the hop FIFO: 16 kHz pieces of any length -> separator chunks and hop counts ------------------------------------
// A slot's row per channel is [FF_HEAD + 64 + capacity]: the read position, the samples held and the samples dropped (int32
// words), then a ring of 64 + capacity samples.  The 64 (CHUNK_CARRY) samples before the read position are the carry, the
// held ones follow it.  All zeros is an empty FIFO whose carry is 64 zeros.
constexpr int FF_HEAD = 3;

__global__ void __launch_bounds__(RS_TILE)
hop_fifo_kernel(const float* __restrict__ x, int64_t x_row, int64_t x_ch, int max_in, const int32_t* __restrict__ counts,
                int unit, float* __restrict__ chunk, int64_t c_row, int64_t c_ch, int32_t* __restrict__ hops, int C, int T,
                const int32_t* __restrict__ slots, float* __restrict__ state, int n_slots, int capacity) {
    const int tid = threadIdx.x, R = CHUNK_CARRY + capacity;
    const SlotRow r = slot_row(C, slots, n_slots, state, FF_HEAD + R);
    if (!r.live) {                                                      // a row that stores nothing
        if (r.ch == 0 && tid == 0) hops[r.row] = 0;
        return;
    }
    const int n = row_pushed(counts, r.row, unit, max_in);
    float* st = r.st;
    float* ring = st + FF_HEAD;
    const int pos = int_word(st[0], R - 1), held = int_word(st[1], capacity);
    const int kept = min(n, capacity - held), h = min(T, (held + kept) / CHUNK_HOP);
    const float* xr = row_ch(x, x_row, x_ch, r.row, r.ch);
    // ring indices in int64: pos + held + i reaches 2 capacity + 62, which passes INT32_MAX from capacity ~2^30 on
    for (int i = tid; i < kept; i += blockDim.x) ring[((int64_t)pos + held + i) % R] = xr[i];
    __syncthreads();                                                    // the appended samples, visible to the block
    float* cr = row_ch(chunk, c_row, c_ch, r.row, r.ch);
    for (int i = tid; i < h * CHUNK_HOP + CHUNK_CARRY; i += blockDim.x) cr[i] = ring[((int64_t)pos + R - CHUNK_CARRY + i) % R];
    if (tid == 0) {
        if (r.ch == 0) hops[r.row] = h;
        st[0] = __int_as_float((int)(((int64_t)pos + h * CHUNK_HOP) % R));
        st[1] = __int_as_float(held + kept - h * CHUNK_HOP);
        st[2] = add_word(st[2], n - kept);
    }
}

// ---- the enrollment capture: the hops' new samples into a per-slot ring (layout: enroll_capture.cuh) -----------------
// Row i appends samples CHUNK_CARRY .. CHUNK_CARRY + 128 h - 1 of its chunk (the hops' new samples, no look-ahead repeat)
// to slot slots[i], h = hops[i]; a slot outside [0, n_slots) or h outside [1, T] stores nothing.  grid n * C, a CTA per
// (row, channel).
__global__ void __launch_bounds__(RS_TILE)
enroll_capture_kernel(const float* __restrict__ chunk, int64_t c_row, int64_t c_ch, int C, int T,
                      const int32_t* __restrict__ slots, const int32_t* __restrict__ hops, float* __restrict__ state,
                      int n_slots, int capacity) {
    const int tid = threadIdx.x;
    const SlotRow sr = slot_row(C, slots, n_slots, state, EC_HEAD + capacity);
    const int h = row_hops(hops, sr.row, T);
    if (h == 0 || !sr.live) return;
    float* st = sr.st;
    const CaptureRow r = capture_row(st, capacity);
    float* ring = st + EC_HEAD;
    const int n = h * CHUNK_HOP, skip = n > capacity ? n - capacity : 0;   // only the last `capacity` samples survive
    const float* src = row_ch(chunk, c_row, c_ch, sr.row, sr.ch) + CHUNK_CARRY;
    for (int i = skip + tid; i < n; i += blockDim.x) ring[(int)(((int64_t)r.wpos + i) % capacity)] = src[i];
    __syncthreads();                                                    // every thread has read the head
    if (tid == 0) {
        st[0] = __int_as_float((int)(((int64_t)r.wpos + n) % capacity));
        st[1] = __int_as_float((int)min((int64_t)r.captured + n, (int64_t)capacity));
    }
}

// ---- the target mixer: a listener's target rows, gain-ramped, and its ambient mixture summed into one row -------------
// The state is [n_records + n_slots][C][TM_FLOATS]: one ramp per (separator record, channel), then one per (listener slot,
// channel) for the ambient term.  A ramp (g0, g1, F, p) goes from g0 to g1 over F samples, p of them mixed already: the
// sample at position q of the ramp is mixed at ramp_level(q + 1), so the gain of a sample depends only on (g0, g1, F) and
// q, never on how the ramp was cut into calls.  Word 2 holds F + 1 (0: never set, settled at the row's rest gain, 1 for a
// record and 0 for a slot), so all zeros is a fresh row.
constexpr int TM_FLOATS = 4;     // g0, g1, then int32 words F + 1 and p
constexpr int TM_THREADS = 128;
constexpr int TM_TERMS = 64;     // target rows staged per pass

struct Ramp {
    float g0, g1;
    int F, p;    // p in [0, F]
};

L2H_DEVINL Ramp ramp_of(const float* w, float rest) {
    const int f1 = __float_as_int(w[2]);
    if (f1 <= 0) return {rest, rest, 0, 0};
    const int F = f1 - 1;
    return {w[0], w[1], F, int_word(w[3], F)};
}

// the gain after q samples of the ramp: g1 from q = F on, a raised cosine from g0 before
L2H_DEVINL float ramp_level(const Ramp& r, int64_t q) {
    if (q >= r.F) return r.g1;
    return r.g0 + (r.g1 - r.g0) * (1.f - cospif((float)q / (float)r.F)) * 0.5f;
}

// a ramp that mixes 0 into every one of the next n samples (a raised cosine is monotone, so its ends decide)
L2H_DEVINL bool ramp_mute(const Ramp& r, int n) {
    return ramp_level(r, (int64_t)r.p + 1) == 0.f && ramp_level(r, (int64_t)r.p + n) == 0.f;
}

// the word p of a ramp after n more samples (only a running ramp changes)
L2H_DEVINL void ramp_advance(float* w, const Ramp& r, int n) {
    if (r.p < r.F) w[3] = __int_as_float((int)min((int64_t)r.F, (int64_t)r.p + n));
}

// V consecutive floats (V = 1 or 4; 4 only where every operand is 16-byte aligned)
template <int V> struct Vec { float v[V]; };
template <int V> L2H_DEVINL Vec<V> vload(const float* p) {
    Vec<V> a;
    if constexpr (V == 4) {
        const float4 f = *reinterpret_cast<const float4*>(p);
        a.v[0] = f.x; a.v[1] = f.y; a.v[2] = f.z; a.v[3] = f.w;
    } else {
        a.v[0] = *p;
    }
    return a;
}
template <int V> L2H_DEVINL void vstore(float* p, const Vec<V>& a) {
    if constexpr (V == 4) *reinterpret_cast<float4*>(p) = make_float4(a.v[0], a.v[1], a.v[2], a.v[3]);
    else *p = a.v[0];
}

// acc += gain * x over V samples at ramp position q0, each sample's gain from the ramp.  A sample whose gain is 0 is left
// as it is, so whether a term enters a sample depends only on that sample's gain, never on how the hops were cut.
template <int V> L2H_DEVINL void mix_term(Vec<V>& acc, const Vec<V>& x, const Ramp& r, int64_t q0) {
    const bool flat = (int64_t)r.p + 1 >= r.F;
#pragma unroll
    for (int k = 0; k < V; ++k) {
        const float g = flat ? r.g1 : ramp_level(r, q0 + k + 1);
        if (g != 0.f) acc.v[k] = fmaf(g, x.v[k], acc.v[k]);
    }
}

// max over the block of v (TM_THREADS threads)
L2H_DEVINL int block_max(int v, int* red) {
    for (int d = 16; d > 0; d >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, d));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    v = red[0];
    for (int w = 1; w < TM_THREADS / 32; ++w) v = max(v, red[w]);
    __syncthreads();
    return v;
}

// One CTA = one (listener row, channel).  Row i owns target rows start .. end - 1, start = the running maximum of the
// offsets clamped to [0, R] (the separator's clamp, targets_kernels.cuh), and writes out[i][c][0 .. 128 h) with h = hops[i]
// (T without hops): the sum in row order of its live target rows scaled by their records' ramps, then the ambient term
// (chunk row i scaled by its slot's ramp).  Each sample's sum starts at -0 and takes, with fmaf, every term whose gain at
// that sample is nonzero: fmaf(g, x, -0) is g x exactly, so the first such term starts the sum with nothing added to a
// zero, and a sample with none is -0.  A term whose gain is 0 over all 128 h samples is not read.  Target rows are staged
// TM_TERMS at a time; a later pass continues the sum from `out`, which the same thread wrote.  Each staged term's ramp word is read once, by the thread that stages it, which also advances it.
template <int V>
__global__ void __launch_bounds__(TM_THREADS)
target_mix_kernel(const float* __restrict__ y, int64_t y_row, int64_t y_ch, const float* __restrict__ chunk, int64_t c_row,
                  int64_t c_ch, float* __restrict__ out, int64_t o_row, int64_t o_ch, int C, int R, int T,
                  const int32_t* __restrict__ records, const int32_t* __restrict__ offsets,
                  const int32_t* __restrict__ hops, const int32_t* __restrict__ slots, float* __restrict__ state,
                  int n_records, int n_slots) {
    __shared__ Ramp ramp[TM_TERMS];
    __shared__ int term_row[TM_TERMS];   // the staged target rows, -1 for a row that mixes nothing
    __shared__ int red[TM_THREADS / 32];
    const int tid = threadIdx.x;
    const SlotRow sr = slot_row(C, slots, n_slots, state + (int64_t)n_records * C * TM_FLOATS, TM_FLOATS);
    const int h = row_hops(hops, sr.row, T);
    if (h == 0 || !sr.live) return;                                     // a row that stores nothing
    const int n = h * CHUNK_HOP, i = sr.row, ch = sr.ch;
    int lo = 0, hi = 0;                                                 // max of the clamped offsets 0 .. i and 0 .. i + 1
    for (int j = tid; j <= i + 1; j += TM_THREADS) {
        const int v = min(max(offsets[j], 0), R);
        hi = max(hi, v);
        if (j <= i) lo = max(lo, v);
    }
    const int start = block_max(lo, red), end = block_max(hi, red);
    const Ramp amb = ramp_of(sr.st, 0.f);
    const bool amb_live = chunk != nullptr && !ramp_mute(amb, n);
    const float* cr = chunk ? row_ch(chunk, c_row, c_ch, i, ch) : nullptr;
    float* orow = row_ch(out, o_row, o_ch, i, ch);
    bool started = false;                                               // out holds a partial sum (uniform)
    for (int r0 = start;; r0 += TM_TERMS) {
        const int cnt = max(0, min(TM_TERMS, end - r0));
        const bool last = r0 + TM_TERMS >= end;
        if (tid < cnt) {
            const int rec = records[r0 + tid];
            int row = -1;
            if (rec >= 0 && rec < n_records) {
                float* w = state + ((int64_t)rec * C + ch) * TM_FLOATS;
                const Ramp g = ramp_of(w, 1.f);
                ramp[tid] = g;
                if (!ramp_mute(g, n)) row = r0 + tid;
                ramp_advance(w, g, n);
            }
            term_row[tid] = row;
        }
        __syncthreads();
        bool any = false;
        for (int t = 0; t < cnt; ++t) any = any || term_row[t] >= 0;
        if (any || (last && (amb_live || !started))) {
            for (int s = tid * V; s < n; s += TM_THREADS * V) {
                Vec<V> acc;
                if (started) acc = vload<V>(orow + s);
                else
                    for (int k = 0; k < V; ++k) acc.v[k] = -0.f;             // the identity of the sum
                for (int t = 0; t < cnt; ++t) {
                    const int row = term_row[t];
                    if (row >= 0)
                        mix_term<V>(acc, vload<V>(row_ch(y, y_row, y_ch, row, ch) + s), ramp[t], (int64_t)ramp[t].p + s);
                }
                if (last && amb_live) mix_term<V>(acc, vload<V>(cr + s), amb, (int64_t)amb.p + s);
                vstore<V>(orow + s, acc);
            }
            started = true;
        }
        if (last) break;
        __syncthreads();                                                // the staged terms are read before the next pass
    }
    if (tid == 0) ramp_advance(sr.st, amb, n);                         // every thread read the ambient ramp above
}

// Entry e of a gain set (j = e * C + ch): the ramp of state row rows[e] becomes (start, gains[e], fades[e], 0), start =
// starts[e], or without starts the gain of the last sample mixed.  A row outside the state, or a fade outside [0, 2^31 - 2],
// stores nothing.
__global__ void __launch_bounds__(RS_TILE)
target_mix_set_kernel(float* __restrict__ state, int n_records, int n_rows, int C, const int32_t* __restrict__ rows, int n,
                      const float* __restrict__ gains, const float* __restrict__ starts, const int32_t* __restrict__ fades) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n * C) return;
    const int e = j / C, ch = j - e * C, row = rows[e], F = fades[e];
    if (row < 0 || row >= n_rows || F < 0 || F == INT32_MAX) return;
    float* w = state + ((int64_t)row * C + ch) * TM_FLOATS;
    const Ramp g = ramp_of(w, row < n_records ? 1.f : 0.f);
    w[0] = starts ? starts[e] : ramp_level(g, g.p);
    w[1] = gains[e];
    w[2] = __int_as_float(F + 1);
    w[3] = __int_as_float(0);
}

// ---- the limiter: a look-ahead peak limiter per slot, one gain for all channels ---------------------------------------
// Gains live in an integer log domain, LM_Q quanta per octave of amplitude, so the release recurrence is exact integer
// arithmetic: computed as a parallel max-scan it is still the same bits under any cut into calls.  Per input sample k:
//   q[k] = 0 if p <= ceiling, else ceil(LM_Q log2(p / ceiling)) + 1      p = max over channels of |x[c][k]|
//          (LM_MUTE for a non-finite sample); the + 1 covers the rounding of the fp32 gain and product
//   s[k] = max q[k - La .. k]                                             hold
//   r[k] = max(s[k], r[k - 1] - step)                                     release, `step` quanta per sample
//   a[k] = sum r[k - La .. k]                                             smoothing box of La + 1
//   y[c][k] = 2^(-a[k] / (LM_Q (La + 1))) x[c][k - La]                    0 where x is not finite, or a mutes
// A peak at P keeps r >= q[P] over [P, P + La], so the box at P + La, which scales x[P], is at least q[P]: |y| <= ceiling.
// A slot's state row per channel is [LM_HEAD + 3 La]: the head words (channel 0's only: r of the last sample, the slot's
// ceiling (0: the call's), the samples written with a > 0, saturating, and the dB of reduction at the last sample), the
// channel's last La input samples, then (channel 0's only) the last La q and the last La r.  All zeros is a fresh slot.
constexpr int LM_HEAD = 4;
constexpr int LM_Q = 1 << 16;
constexpr int LM_MUTE_OCT = 150;                        // a reduction of 150 octaves is a gain of exactly 0
constexpr int LM_MUTE = LM_MUTE_OCT * LM_Q;            // the q of a non-finite sample, and every q's and r's cap

// the maximum of v over the block's threads before this one (INT64_MIN for thread 0); every thread of the block calls it
L2H_DEVINL int64_t block_exclusive_max(int64_t v, int64_t* warp_max) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int64_t inc = v;
    for (int d = 1; d < 32; d <<= 1) {
        const int64_t o = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc = max(inc, o);
    }
    int64_t ex = __shfl_up_sync(0xffffffffu, inc, 1);
    if (lane == 0) ex = INT64_MIN;
    if (lane == 31) warp_max[w] = inc;
    __syncthreads();
    for (int i = 0; i < w; ++i) ex = max(ex, warp_max[i]);
    return ex;
}

// One CTA = one call row over all C channels (the gain is linked).  The slot's C channel rows are consecutive, so the
// scaffold's slot_row finds them as one row of C row_floats.  Row i pushes n = counts[i] * unit samples (0 outside
// [0, max_in]: the row stores nothing) and writes y[i][c][0 .. n).
__global__ void __launch_bounds__(RS_TILE)
limiter_kernel(const float* __restrict__ x, int64_t x_row, int64_t x_ch, int max_in, const int32_t* __restrict__ counts,
               int unit, float* __restrict__ y, int64_t y_row, int64_t y_ch, int C, const int32_t* __restrict__ slots,
               float* __restrict__ state, int n_slots, float ceiling, int La, int step) {
    extern __shared__ float sm[];
    __shared__ int64_t warp_max[RS_TILE / 32];
    __shared__ int limited;
    const int tid = threadIdx.x;
    const int64_t rf = LM_HEAD + 3 * (int64_t)La;
    const SlotRow sr = slot_row(1, slots, n_slots, state, C * rf);
    const int n = row_pushed(counts, sr.row, unit, max_in);
    if (!sr.live || n == 0) return;                                     // a row that stores nothing
    float* st = sr.st;                                                  // channel c's row at st + c rf
    const int W = La + n;
    float* xs = sm;                                                     // [C][W]: each channel's delay line, then x
    int* qs = reinterpret_cast<int*>(sm + (int64_t)C * W);              // [W]: the last La q, then the new ones
    int* rs = qs + W;                                                   // [W]: the last La r, then s, then r
    const float cw = st[1];
    const float lim = cw >= FLT_MIN && cw <= FLT_MAX ? cw : ceiling;     // the slot's ceiling, else the call's
    const int64_t r_in = int_word(st[0], LM_MUTE);
    for (int c = 0; c < C; ++c) {
        const float* d = st + c * rf + LM_HEAD;
        const float* xr = row_ch(x, x_row, x_ch, sr.row, c);
        for (int i = tid; i < W; i += blockDim.x) xs[(int64_t)c * W + i] = i < La ? d[i] : xr[i - La];
    }
    for (int i = tid; i < La; i += blockDim.x) {
        qs[i] = int_word(st[LM_HEAD + La + i], LM_MUTE);
        rs[i] = int_word(st[LM_HEAD + 2 * La + i], LM_MUTE);
    }
    if (tid == 0) limited = 0;
    __syncthreads();
    for (int k = tid; k < n; k += blockDim.x) {
        float p = 0.f;
        bool finite = true;
        for (int c = 0; c < C; ++c) {
            const float v = xs[(int64_t)c * W + La + k];
            finite = finite && isfinite(v);
            p = fmaxf(p, fabsf(v));
        }
        int q = 0;
        if (!finite) q = LM_MUTE;
        else if (p > lim) q = (int)fmin((double)LM_MUTE, ceil(LM_Q * log2((double)p / (double)lim)) + 1.0);
        qs[La + k] = q;
    }
    __syncthreads();
    // hold and release over contiguous pieces of the push, one per thread: r[k] = max(r_in - (k + 1) step,
    // max_{j <= k} (s[j] + j step) - k step), the running max carried across the pieces by a block scan
    const int per = (n + blockDim.x - 1) / blockDim.x, k0 = min(n, tid * per), k1 = min(n, k0 + per);
    int64_t run = INT64_MIN;
    for (int k = k0; k < k1; ++k) {
        int s = 0;
        for (int j = k; j <= k + La; ++j) s = max(s, qs[j]);             // q[k - La .. k]
        rs[La + k] = s;
        run = max(run, s + (int64_t)k * step);
    }
    run = block_exclusive_max(run, warp_max);
    for (int k = k0; k < k1; ++k) {
        run = max(run, rs[La + k] + (int64_t)k * step);
        rs[La + k] = (int)max(r_in - (int64_t)(k + 1) * step, run - (int64_t)k * step);
    }
    __syncthreads();
    const double inv = 1.0 / ((double)LM_Q * (La + 1));
    int mine = 0;
    for (int k = tid; k < n; k += blockDim.x) {
        int64_t a = 0;
        for (int j = k; j <= k + La; ++j) a += rs[j];                    // r[k - La .. k], exact in any order
        // the gain 2^-e as 2^-f 2^-i (i = floor(e)): the power of two scales exactly, so a gain below the normal range
        // keeps its precision
        const double e = (double)a * inv;
        const int ei = (int)e;
        const float gf = a == 0 ? 1.f : (a >= (int64_t)LM_MUTE * (La + 1) ? 0.f : exp2f(-(float)(e - ei)));
        mine += a > 0;
        for (int c = 0; c < C; ++c) {
            const float v = xs[(int64_t)c * W + k];                     // x[c][k - La]
            row_ch(y, y_row, y_ch, sr.row, c)[k] = isfinite(v) ? (ei ? ldexpf(gf * v, -ei) : gf * v) : 0.f;
        }
        if (k == n - 1) st[3] = (float)(e * 6.020599913279624);        // 20 log10(2) dB per octave
    }
    if (mine) atomicAdd(&limited, mine);
    for (int c = 0; c < C; ++c)
        for (int i = tid; i < La; i += blockDim.x) st[c * rf + LM_HEAD + i] = xs[(int64_t)c * W + n + i];
    for (int i = tid; i < La; i += blockDim.x) {
        st[LM_HEAD + La + i] = __int_as_float(qs[n + i]);
        st[LM_HEAD + 2 * La + i] = __int_as_float(rs[n + i]);
    }
    __syncthreads();                                                    // every thread counted
    if (tid == 0) {
        st[0] = __int_as_float(rs[La + n - 1]);
        st[2] = add_word(st[2], limited);
    }
}

// ---- the leveler: a gated, K-weighted loudness leveler per row, one gain for all channels ------------------------------
// A row (a separator record, or a listener slot on the mixer's sum) is leveled hop by hop on the 16 kHz grid.  Each
// channel's samples pass the two BS.1770 pre-filters (a high shelf, then a high-pass, in transposed direct form II); the
// hop's power P is the mean square of the weighted samples summed over the channels, its loudness -0.691 + 10 log10 P
// LUFS.  A hop at or above `gate`, and, once the row has an estimate, at or above the estimate's loudness + `relative`,
// updates the estimate E += w (P - E), w = max(alpha, 1 / (n + 1)) over the n gated hops before it.  The gain (dB) stays
// where it is until the row has `settle` gated hops, takes d = clamp(target - L(E), min_gain, max_gain) in the hop that
// reaches them, and then moves toward d by at most `rise` dB up and `fall` dB down per hop.  Sample k = 1 .. 128 of the hop
// is scaled in every channel by the gain interpolated in dB from the hop's start to its end; a gain of 0 dB is exactly 1.
// A hop with a sample that is not finite, or whose magnitude reaches 2^32 (where the weighted squares could overflow), is
// not measured: filters, estimate, count and gain keep their values, so the state stays finite.  A hop's result depends
// only on the state at its start and its samples, so cutting the hops into other calls changes no bit.
// A row's state per channel is [LV_HEAD + 4]: the head words (channel 0's only: E, n as an int32 word, the gain in dB),
// then the channel's shelf and high-pass states.  All zeros is a fresh row.
constexpr int LV_HEAD = 3;
constexpr int LV_FLOATS = LV_HEAD + 4;
constexpr int LV_THREADS = TM_THREADS;                  // one thread per sample of a hop; block_max's block
static_assert(LV_THREADS == CHUNK_HOP, "the leveler runs one thread per sample of a hop");

struct LvParams {
    float sb0, sb1, sb2, sa1, sa2;   // the shelf
    float ha1, ha2;                  // the high-pass, whose numerator is 1, -2, 1
    float target, gate, relative, alpha, min_gain, max_gain, rise, fall;
    int settle;
};

L2H_DEVINL float lv_lufs(float power) { return -0.691f + 10.f * log10f(power); }

// One CTA = one call row over all C channels (the gain is linked).  Listener i owns rows start .. end - 1 (the separator's
// clamp: the first j with offsets[j] > r ends the listeners at or before row r), or row i alone without offsets; its rows
// level their first 128 h samples, h = hops[i] (T without hops).  Row r keeps its state in row records[r].  y and out may
// be the same tensor: each hop's samples are read before they are written.
__global__ void __launch_bounds__(LV_THREADS)
leveler_kernel(const float* y, int64_t y_row, int64_t y_ch, float* out, int64_t o_row, int64_t o_ch, int n, int C, int T,
               const int32_t* __restrict__ records, const int32_t* __restrict__ offsets, const int32_t* __restrict__ hops,
               float* __restrict__ state, int n_rows, const __grid_constant__ LvParams p) {
    __shared__ int red[LV_THREADS / 32];
    __shared__ float part[LV_THREADS];
    __shared__ float g_from, g_to;                                      // the hop's gain in dB at its start and its end
    const int tid = threadIdx.x;
    const SlotRow sr = slot_row(1, records, n_rows, state, (int64_t)C * LV_FLOATS);
    const int r = sr.row;
    int i = r;
    if (offsets) {
        int first = n + 1;
        for (int j = tid; j <= n; j += LV_THREADS)
            if (offsets[j] > r) { first = j; break; }
        i = -block_max(-first, red) - 1;
    }
    if (i < 0 || i >= n) return;                                        // a row of no listener
    const int h = row_hops(hops, i, T);
    if (h == 0 || !sr.live) return;                                     // a row that stores nothing
    float* st = sr.st;                                                  // channel c's row at st + c LV_FLOATS
    float E = st[0], g = st[2];
    int cnt = int_word(st[1], INT32_MAX);
    for (int t = 0; t < h; ++t) {
        const int64_t s = (int64_t)t * CHUNK_HOP + tid;
        bool bad = false;
        for (int c = 0; c < C; ++c) bad = bad || !(fabsf(row_ch(y, y_row, y_ch, r, c)[s]) < HG_BIG);
        const bool measured = !__syncthreads_or(bad);
        if (measured) {
            float acc = 0.f;
            for (int c = tid; c < C; c += LV_THREADS) {
                float* f = st + (int64_t)c * LV_FLOATS + LV_HEAD;
                float s1 = f[0], s2 = f[1], h1 = f[2], h2 = f[3];
                const float* xr = row_ch(y, y_row, y_ch, r, c) + (int64_t)t * CHUNK_HOP;
#pragma unroll 16
                for (int k = 0; k < CHUNK_HOP; ++k) {
                    const float x = xr[k];
                    const float u = fmaf(p.sb0, x, s1);
                    s1 = fmaf(p.sb1, x, fmaf(-p.sa1, u, s2));
                    s2 = fmaf(p.sb2, x, -p.sa2 * u);
                    const float w = u + h1;
                    h1 = fmaf(-2.f, u, fmaf(-p.ha1, w, h2));
                    h2 = fmaf(-p.ha2, w, u);
                    acc = fmaf(w, w, acc);
                }
                f[0] = s1; f[1] = s2; f[2] = h1; f[3] = h2;
            }
            part[tid] = acc;
            __syncthreads();
        }
        if (tid == 0) {
            const float g0 = g;
            if (measured) {
                float P = 0.f;
                for (int c = 0; c < min(C, LV_THREADS); ++c) P += part[c];   // channel order: the same bits every call
                P *= 1.f / CHUNK_HOP;
                const float L = lv_lufs(P);
                const int before = cnt;
                if (L >= p.gate && (cnt == 0 || L >= lv_lufs(E) + p.relative)) {
                    E = fmaf(fmaxf(p.alpha, 1.f / (float)(cnt + 1ll)), P - E, E);   // no overflow at INT32_MAX
                    cnt += cnt < INT32_MAX;
                }
                if (cnt >= p.settle) {
                    const float d = fminf(fmaxf(p.target - lv_lufs(E), p.min_gain), p.max_gain);
                    g = before < p.settle ? d : g + fminf(fmaxf(d - g, -p.fall), p.rise);
                }
            }
            g_from = g0;
            g_to = g;
        }
        __syncthreads();
        const float lin = hop_gain(g_from, g_to);
        for (int c = 0; c < C; ++c) row_ch(out, o_row, o_ch, r, c)[s] = row_ch(y, y_row, y_ch, r, c)[s] * lin;
    }
    if (tid == 0) {
        st[0] = E;
        st[1] = __int_as_float(cnt);
        st[2] = g;
    }
}

// ---- the band compressor: per-band gain and compression per slot, the compression linked across channels --------------
// A slot (a listener, on the mixer's 16 kHz sum) is split hop by hop into K bands by linear-phase FIRs of L taps (the
// bank of l2h_band_compressor_design, [K][L], summing to a delay of D = (L - 1) / 2 samples).  Per hop: the band's linked
// level P_b is its mean square over the hop's samples and the channels; the detector S_b moves toward it by `attack` when
// P_b > S_b, else by `release`; the compression R_b = slope_b max(0, 10 log10 S_b - knee_b) dB is the same for every
// channel, and channel c's band b takes g = clamp(gain_cb - R_b, -40, 40) dB at the hop's end.  Sample k = 1 .. 128 of
// the hop is the sum in band order of each band's sample times 10^(g_k / 20), g_k interpolated in dB from the gain at the
// previous hop's end (a g_k of 0 dB is exactly 1).  When every gain of the slot is 0 dB at the hop's start and end, the
// output is the staged input delayed by D, bit for bit.  A sample that is not finite, or whose magnitude reaches 2^32,
// is staged as 0, and its hop is not measured (the detector keeps its values), so the state stays finite.  A hop's result
// depends only on the state at its start and its samples, so cutting hops into other calls changes no bit.
// A slot's state per channel is [5 K + L - 1]: the channel's K profile gains (dB) and its K current gains (dB, at the last
// sample written); then, channel 0's only, S_b, knee_b (dBFS) and slope_b = 1 - 1 / ratio; then the channel's last L - 1
// staged samples.  All zeros is a fresh slot: flat 0 dB and no compression.
constexpr int BC_THREADS = CHUNK_HOP;                   // one thread per sample of a hop
constexpr int BC_MAX_BANDS = 16;
constexpr int BC_MIN_TAPS = 33, BC_MAX_TAPS = 255;
constexpr float BC_RANGE = 40.f;                        // the gains' clamp, dB
static_assert(BC_MAX_BANDS <= BC_THREADS, "one thread per band updates the detectors");

// The steps both banks share, one thread per sample of the hop.  measure: sq[b] is the thread's sample of band b squared
// and summed over the channels in channel order; the block sums it over the samples (a warp shuffle, then the warps in
// order) into P_b and moves the detector S_b toward it.  The caller syncs before and after.
template <int KP>
L2H_DEVINL void bc_measure(const float (&sq)[KP], float (*part)[KP], float* S, int K, int C, float attack, float release) {
    const int tid = threadIdx.x;
#pragma unroll
    for (int b = 0; b < KP; ++b) {
        float v = sq[b];
        for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
        if ((tid & 31) == 0) part[tid >> 5][b] = v;
    }
    __syncthreads();
    if (tid < K) {
        float P = part[0][tid];
        for (int w = 1; w < BC_THREADS / 32; ++w) P += part[w][tid];
        P *= 1.f / (float)(CHUNK_HOP * C);
        const float old = S[tid];
        S[tid] = fmaf(P > old ? attack : release, P - old, old);
    }
}

// gain: element i = c K + b of the gains (dB) at the hop's end, from the detectors S and the slot's state rows st (rf
// words per channel)
L2H_DEVINL float bc_gain(const float* st, int64_t rf, const float* S, int K, int i) {
    const int c = i / K, b = i - c * K;
    const float R = st[4 * K + b] * fmaxf(0.f, 10.f * log10f(S[b]) - st[3 * K + b]);
    return fminf(fmaxf(st[c * rf + b] - R, -BC_RANGE), BC_RANGE);
}

template <int KP>
__global__ void __launch_bounds__(BC_THREADS)
band_compressor_kernel(const float* y, int64_t y_row, int64_t y_ch, float* out, int64_t o_row, int64_t o_ch, int C, int T,
                       const int32_t* __restrict__ slots, const int32_t* __restrict__ hops, const float* __restrict__ bank,
                       int K, int L, float* __restrict__ state, int n_slots, float attack, float release) {
    extern __shared__ float4 sm4[];
    __shared__ float part[BC_THREADS / 32][KP];
    __shared__ float S[KP];
    const int tid = threadIdx.x, H = L - 1, W = H + CHUNK_HOP, D = H / 2, CK = C * K;
    const int64_t rf = 5 * K + H;
    const SlotRow sr = slot_row(1, slots, n_slots, state, C * rf);
    const int h = row_hops(hops, sr.row, T);
    if (h == 0 || !sr.live) return;                                     // a row that stores nothing
    float* st = sr.st;                                                  // channel c's row at st + c rf
    float* taps = reinterpret_cast<float*>(sm4);                        // [L][KP]: tap j of band b, zero past K
    float* win = taps + L * KP;                                         // [C][W]: the last H staged samples, then the hop
    float* band = win + C * W;                                          // [C][K][128]: the hop's band signals
    float* g0 = band + CK * CHUNK_HOP;                                  // [C][K]: the gains (dB) at the hop's start
    float* g1 = g0 + CK;                                                // [C][K]: and at its end
    for (int i = tid; i < L * KP; i += BC_THREADS) {
        const int j = i / KP, b = i - j * KP;
        taps[i] = b < K ? bank[b * L + j] : 0.f;
    }
    for (int c = 0; c < C; ++c)
        for (int i = tid; i < H; i += BC_THREADS) win[c * W + i] = st[c * rf + 5 * K + i];
    for (int i = tid; i < CK; i += BC_THREADS) {
        const int c = i / K;
        g0[i] = st[c * rf + K + (i - c * K)];
    }
    if (tid < K) S[tid] = st[2 * K + tid];
    for (int t = 0; t < h; ++t) {
        const int64_t s = (int64_t)t * CHUNK_HOP + tid;
        bool bad = false;
        for (int c = 0; c < C; ++c) {
            const float v = row_ch(y, y_row, y_ch, sr.row, c)[s];
            const bool ok = fabsf(v) < HG_BIG;
            bad = bad || !ok;
            win[c * W + H + tid] = ok ? v : 0.f;
        }
        const bool measured = !__syncthreads_or(bad);                   // and the staged hop is visible to the block
        float sq[KP];
#pragma unroll
        for (int b = 0; b < KP; ++b) sq[b] = 0.f;
        for (int c = 0; c < C; ++c) {
            float acc[KP];
#pragma unroll
            for (int b = 0; b < KP; ++b) acc[b] = 0.f;
            const float* xk = win + c * W + H + tid;                   // xk[-j] is the sample j before this one
#pragma unroll 4
            for (int j = 0; j < L; ++j) {
                const float x = xk[-j];
                const float4* tp = reinterpret_cast<const float4*>(taps + j * KP);
#pragma unroll
                for (int q = 0; q < KP / 4; ++q) {
                    const float4 w = tp[q];
                    acc[4 * q] = fmaf(w.x, x, acc[4 * q]);
                    acc[4 * q + 1] = fmaf(w.y, x, acc[4 * q + 1]);
                    acc[4 * q + 2] = fmaf(w.z, x, acc[4 * q + 2]);
                    acc[4 * q + 3] = fmaf(w.w, x, acc[4 * q + 3]);
                }
            }
#pragma unroll
            for (int b = 0; b < KP; ++b) {
                if (b < K) band[(c * K + b) * CHUNK_HOP + tid] = acc[b];
                sq[b] = fmaf(acc[b], acc[b], sq[b]);
            }
        }
        if (measured) bc_measure<KP>(sq, part, S, K, C, attack, release);   // the same order of sums every call
        __syncthreads();                                                // the detectors, and every band sample
        bool live = false;
        for (int i = tid; i < CK; i += BC_THREADS) {
            g1[i] = bc_gain(st, rf, S, K, i);
            live = live || g0[i] != 0.f || g1[i] != 0.f;
        }
        live = __syncthreads_or(live);                                  // and every gain is visible to the block
        for (int c = 0; c < C; ++c) {
            float o = win[c * W + H + tid - D];                         // the staged input delayed by D
            if (live) {
                o = 0.f;
                for (int b = 0; b < K; ++b)
                    o = fmaf(hop_gain(g0[c * K + b], g1[c * K + b]), band[(c * K + b) * CHUNK_HOP + tid], o);
            }
            row_ch(out, o_row, o_ch, sr.row, c)[s] = o;
        }
        for (int c = 0; c < C; ++c) {                                   // the last H staged samples become the history
            const float a = tid < H ? win[c * W + CHUNK_HOP + tid] : 0.f;
            const float b = tid + BC_THREADS < H ? win[c * W + CHUNK_HOP + BC_THREADS + tid] : 0.f;
            __syncthreads();                                            // every thread has read the channel's window
            if (tid < H) win[c * W + tid] = a;
            if (tid + BC_THREADS < H) win[c * W + BC_THREADS + tid] = b;
        }
        for (int i = tid; i < CK; i += BC_THREADS) g0[i] = g1[i];
    }
    __syncthreads();                                                    // the history and the gains
    for (int c = 0; c < C; ++c)
        for (int i = tid; i < H; i += BC_THREADS) st[c * rf + 5 * K + i] = win[c * W + i];
    for (int i = tid; i < CK; i += BC_THREADS) {
        const int c = i / K;
        st[c * rf + K + (i - c * K)] = g0[i];
    }
    if (tid < K) st[2 * K + tid] = S[tid];
}

// ---- the Linkwitz-Riley band compressor: the same per-hop steps on an IIR crossover bank with a short delay ------------
// The bank (l2h_band_compressor_lr_design) cuts the band at the K - 1 edges with Linkwitz-Riley crossovers of order
// N = 4 or 8: at edge e, LP_e and HP_e are a Butterworth filter of order N / 2 applied twice and AP_e is the allpass on
// the same poles, so LP_e + HP_e = AP_e.  Band b is HP_1 .. HP_b, then LP_{b+1} (every band but the last), then
// AP_{b+2} .. AP_{K-1}, so the bands sum to the allpass cascade AP_1 .. AP_{K-1}: flat in magnitude, with a delay that
// falls with frequency.  Each band is a cascade of S = N / 2 (K - 1) biquads, [K][S][5] (b0, b1, b2, a1, a2), the
// shorter cascades ending in identity sections; they run in transposed direct form II with fp32 states, one thread per
// (channel, band), sample by sample through the whole cascade.  The stage, measure, gain and apply steps are the FIR
// kernel's, the measure and the gain through the same helpers (bc_measure, bc_gain).  There is no bypass: at 0 dB
// every band is scaled by exactly 1, and the output is the bands' sum in band order, started from -0, so that K = 1
// (no sections) returns its staged input bit for bit.
// A slot's state per channel is [5 K + 2 K S]: the FIR bank's 5 K head words, then the two states of each band's
// sections, [K][S][2].  All zeros is a fresh slot.

// one band of one channel through the hop's 128 samples: x the staged hop, cf [S][5] its sections in shared memory,
// z [S][2] their states (read and written back), yb the band's 128 samples.  S is a compile-time count, so the cascade
// unrolls without a branch and the sections of neighbouring samples overlap.  The states stay in registers, and the
// coefficients too while S <= LR_REG_SECTIONS.
constexpr int LR_REG_SECTIONS = 16;
template <int S>
L2H_DEVINL void lr_band(const float* x, const float* cf, float* z, float* yb) {
    constexpr int SR = S > 0 ? S : 1;
    constexpr bool REGS = S <= LR_REG_SECTIONS;
    float z1[SR], z2[SR], c[REGS ? SR : 1][5];
#pragma unroll
    for (int q = 0; q < S; ++q) {
        z1[q] = z[2 * q];
        z2[q] = z[2 * q + 1];
        if (REGS)
            for (int j = 0; j < 5; ++j) c[REGS ? q : 0][j] = cf[5 * q + j];
    }
#pragma unroll 4
    for (int k = 0; k < CHUNK_HOP; ++k) {
        float v = x[k];
#pragma unroll
        for (int q = 0; q < S; ++q) {
            const float* cq = REGS ? c[REGS ? q : 0] : cf + 5 * q;
            const float u = fmaf(cq[0], v, z1[q]);
            z1[q] = fmaf(cq[1], v, fmaf(-cq[3], u, z2[q]));
            z2[q] = fmaf(cq[2], v, -cq[4] * u);
            v = u;
        }
        yb[k] = v;
    }
#pragma unroll
    for (int q = 0; q < S; ++q) {
        z[2 * q] = z1[q];
        z[2 * q + 1] = z2[q];
    }
}

// One CTA = one call row over all C channels, as band_compressor_kernel.  One instantiation per band count K and order
// N: KP = bc_padded(K) accumulators per thread, and each band's NS = N / 2 (K - 1) sections known at compile time.
template <int K, int N>
__global__ void __launch_bounds__(BC_THREADS)
band_compressor_lr_kernel(const float* y, int64_t y_row, int64_t y_ch, float* out, int64_t o_row, int64_t o_ch, int C,
                          int T, const int32_t* __restrict__ slots, const int32_t* __restrict__ hops,
                          const float* __restrict__ sos, float* __restrict__ state, int n_slots, float attack,
                          float release) {
    constexpr int KP = (K + 3) / 4 * 4, NS = N / 2 * (K - 1);
    extern __shared__ float4 sm4[];
    __shared__ float part[BC_THREADS / 32][KP];
    __shared__ float S[KP];
    const int tid = threadIdx.x, CK = C * K;
    const int64_t rf = 5 * K + 2 * K * NS;
    const SlotRow sr = slot_row(1, slots, n_slots, state, C * rf);
    const int h = row_hops(hops, sr.row, T);
    if (h == 0 || !sr.live) return;                                     // a row that stores nothing
    float* st = sr.st;                                                  // channel c's row at st + c rf
    float* coef = reinterpret_cast<float*>(sm4);                        // [K][NS][5]: the bank
    float* win = coef + K * NS * 5;                                     // [C][128]: the staged hop
    float* band = win + C * CHUNK_HOP;                                  // [C][K][128]: the hop's band signals
    float* g0 = band + CK * CHUNK_HOP;                                  // [C][K]: the gains (dB) at the hop's start
    float* g1 = g0 + CK;                                                // [C][K]: and at its end
    for (int i = tid; i < K * NS * 5; i += BC_THREADS) coef[i] = sos[i];
    for (int i = tid; i < CK; i += BC_THREADS) {
        const int c = i / K;
        g0[i] = st[c * rf + K + (i - c * K)];
    }
    if (tid < K) S[tid] = st[2 * K + tid];
    for (int t = 0; t < h; ++t) {
        const int64_t s = (int64_t)t * CHUNK_HOP + tid;
        bool bad = false;
        for (int c = 0; c < C; ++c) {
            const float v = row_ch(y, y_row, y_ch, sr.row, c)[s];
            const bool ok = fabsf(v) < HG_BIG;
            bad = bad || !ok;
            win[c * CHUNK_HOP + tid] = ok ? v : 0.f;
        }
        const bool measured = !__syncthreads_or(bad);                   // and the staged hop is visible to the block
        for (int i = tid; i < CK; i += BC_THREADS) {
            const int c = i / K, b = i - c * K;
            lr_band<NS>(win + c * CHUNK_HOP, coef + b * NS * 5, st + c * rf + 5 * K + 2 * b * NS, band + i * CHUNK_HOP);
        }
        __syncthreads();                                                // every band sample
        float sq[KP];
#pragma unroll
        for (int b = 0; b < KP; ++b) sq[b] = 0.f;
        for (int c = 0; c < C; ++c) {
#pragma unroll
            for (int b = 0; b < KP; ++b) {
                const float v = b < K ? band[(c * K + b) * CHUNK_HOP + tid] : 0.f;
                sq[b] = fmaf(v, v, sq[b]);
            }
        }
        if (measured) bc_measure<KP>(sq, part, S, K, C, attack, release);
        __syncthreads();                                                // the detectors
        for (int i = tid; i < CK; i += BC_THREADS) g1[i] = bc_gain(st, rf, S, K, i);
        __syncthreads();                                                // every gain
        for (int c = 0; c < C; ++c) {
            float o = -0.f;                                             // so that o + -0 is o, -0 included
            for (int b = 0; b < K; ++b)
                o = fmaf(hop_gain(g0[c * K + b], g1[c * K + b]), band[(c * K + b) * CHUNK_HOP + tid], o);
            row_ch(out, o_row, o_ch, sr.row, c)[s] = o;
        }
        __syncthreads();                                                // every thread has read the gains and the bands
        for (int i = tid; i < CK; i += BC_THREADS) g0[i] = g1[i];
    }
    __syncthreads();                                                    // the gains
    for (int i = tid; i < CK; i += BC_THREADS) {
        const int c = i / K;
        st[c * rf + K + (i - c * K)] = g0[i];
    }
    if (tid < K) st[2 * K + tid] = S[tid];
}

// ---- the host side of the per-slot calls ------------------------------------------------------------------------------
// The checks every per-slot call makes first, in this order: its pointers, its sizes (`sizes` names them), n <= n_slots,
// and a grid of n * channels CTAs.  0, or 1 with its message.
static int slot_call(const std::string& who, std::initializer_list<const void*> ptrs, const char* sizes,
                     std::initializer_list<int32_t> values, int32_t n, int32_t channels, int32_t n_slots) {
    for (const void* p : ptrs) if (!p) return fail(1, who + ": null pointer");
    for (int32_t v : values) if (v <= 0) return fail(1, who + ": " + sizes + " must be positive");
    if (n > n_slots) return fail(1, who + ": a call needs n <= n_slots");
    if ((int64_t)n * channels > INT32_MAX) return fail(1, who + ": n * channels is too large");
    return 0;
}

// a strided [n][channels][len] operand of a per-slot call
struct Rows { const char* name; int64_t row, ch, len; };

// 0 when no two rows or channels of any operand overlap, else 1 with its message
static int disjoint(const std::string& who, int32_t channels, std::initializer_list<Rows> ops) {
    bool ok = true;
    std::string what;
    for (const Rows& r : ops) {
        ok = ok && r.ch >= r.len && r.row / channels >= r.ch;
        what += (what.empty() ? "" : " and ") + std::string(r.name) + " (" + std::to_string(r.len) + " samples)";
    }
    return ok ? 0 : fail(1, who + ": bad stride: rows and channels of " + what + " must not overlap");
}

// the samples of `frames` hops (len) and of a separator chunk of them (c_len: the carry, then the hops): 0, or 1 when
// they do not fit an int32
static int hop_lens(const std::string& who, int32_t frames, int64_t* len, int64_t* c_len) {
    *len = (int64_t)frames * CHUNK_HOP;
    *c_len = *len + CHUNK_CARRY;
    return *c_len > INT32_MAX ? fail(1, who + ": frames is too large") : 0;
}

// whether n_out rows of `out` at po share a byte with n_in rows of `in` at pi (none when pi is null); out may be `in`
// itself (the same pointer and strides) where `in_place`
static bool overlap(const void* po, int64_t n_out, const Rows& out, const void* pi, int64_t n_in, const Rows& in,
                    int32_t channels, bool in_place) {
    if (!pi || (in_place && po == pi && out.row == in.row && out.ch == in.ch)) return false;
    const auto end = [channels](const void* p, int64_t rows, const Rows& r) {    // the end of the bytes the rows span
        return reinterpret_cast<uintptr_t>(p) +
               (uintptr_t)(((rows - 1) * r.row + (int64_t)(channels - 1) * r.ch + r.len) * (int64_t)sizeof(float));
    };
    return reinterpret_cast<uintptr_t>(po) < end(pi, n_in, in) && reinterpret_cast<uintptr_t>(pi) < end(po, n_out, out);
}

// the error of the launch just made: 0, or 3 with its message
static int launched(const std::string& who) {
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail(3, who + ": " + cudaGetErrorString(e));
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
            return fail(1, "l2h_resample: row " + std::to_string(r) + " (" + rs_rates(orig, new_freq) + ") has " + std::to_string(n_out) + " output samples, capacity " + std::to_string(y_capacity));
        const RsRate g = rs_rate(orig, new_freq, 0);
        if ((((int64_t)(RS_TILE - 1) * g.o) / g.q + 2 * (int64_t)g.w + 2) * (int64_t)sizeof(float) > RS_SMEM_BYTES)
            return fail(2, "l2h_resample: reduced rate ratio " + std::to_string(g.o) + "/" + std::to_string(g.q) + " (" +
                               rs_rates(orig, new_freq) + ") is too large: the input window of a tile exceeds shared memory");
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
        const RsRate& g = L.rate[n_rates] = rs_rate(orig, new_freq, n_in);
        rate_hz[n_rates++] = orig;
        if (g.o != g.q) smem = std::max(smem, (int)((((int64_t)(threads - 1) * g.o) / g.q + 2 * g.w + 2) * sizeof(float)));
    }
    if (e == cudaSuccess) e = launch(n_rows);
    if (e != cudaSuccess) return fail(3, std::string("l2h_resample: ") + cudaGetErrorString(e));
    return 0;
}

extern "C" int l2h_resample_stream_layout(int32_t orig_freq, int32_t new_freq, int32_t block, int32_t keep, int32_t* hist,
                                          int32_t* delay, int32_t* out_block) {
    using namespace l2h;
    if (!hist || !delay || !out_block) return fail(1, "l2h_resample_stream_layout: null pointer");
    RsStream s;
    if (int rc = rs_stream("l2h_resample_stream_layout", orig_freq, new_freq, block, keep, 1, &s, nullptr)) return rc;
    *hist = s.hist;
    *delay = s.delay;
    *out_block = s.out_block;
    return 0;
}

extern "C" int l2h_resample_stream(const float* x_dev, int64_t x_row_stride, int64_t x_ch_stride, float* y_dev,
                                   int64_t y_row_stride, int64_t y_ch_stride, int32_t n, int32_t channels, int32_t blocks,
                                   const int32_t* slots_dev, const int32_t* hops_dev, float* state_dev, int32_t n_slots,
                                   int32_t orig_freq, int32_t new_freq, int32_t block, int32_t keep, void* stream) {
    using namespace l2h;
    const std::string who = "l2h_resample_stream";
    if (int rc = slot_call(who, {x_dev, y_dev, slots_dev, state_dev}, "n, channels, blocks and n_slots",
                           {n, channels, blocks, n_slots}, n, channels, n_slots))
        return rc;
    RsStream s;
    int smem;
    if (int rc = rs_stream(who, orig_freq, new_freq, block, keep, blocks, &s, &smem)) return rc;
    const int64_t x_len = (int64_t)blocks * block, y_len = keep + (int64_t)blocks * s.out_block;
    if (int rc = disjoint(who, channels, {{"x", x_row_stride, x_ch_stride, x_len}, {"y", y_row_stride, y_ch_stride, y_len}}))
        return rc;
    resample_stream_kernel<<<(unsigned)(n * channels), RS_TILE, smem, static_cast<cudaStream_t>(stream)>>>(
        x_dev, x_row_stride, x_ch_stride, y_dev, y_row_stride, y_ch_stride, channels, blocks, slots_dev, hops_dev, state_dev,
        n_slots, s);
    return launched(who);
}

extern "C" int l2h_resample_packets_layout(int32_t orig_freq, int32_t new_freq, int32_t max_in, int32_t* row_floats,
                                           int32_t* delay, int32_t* max_out) {
    using namespace l2h;
    if (!row_floats || !delay || !max_out) return fail(1, "l2h_resample_packets_layout: null pointer");
    RsPackets s;
    int32_t out;
    if (int rc = rs_packets("l2h_resample_packets_layout", orig_freq, new_freq, max_in, &s, &out, nullptr)) return rc;
    *row_floats = RP_HEAD + s.hist;
    *delay = s.delay;
    *max_out = out;
    return 0;
}

extern "C" int l2h_resample_packets(const float* x_dev, int64_t x_row_stride, int64_t x_ch_stride, float* y_dev,
                                    int64_t y_row_stride, int64_t y_ch_stride, int32_t n, int32_t channels, int32_t max_in,
                                    const int32_t* counts_dev, int32_t unit, int32_t* out_counts_dev,
                                    const int32_t* slots_dev, float* state_dev, int32_t n_slots, int32_t orig_freq,
                                    int32_t new_freq, void* stream) {
    using namespace l2h;
    const std::string who = "l2h_resample_packets";
    if (int rc = slot_call(who, {x_dev, y_dev, counts_dev, out_counts_dev, slots_dev, state_dev},
                           "n, channels, unit and n_slots", {n, channels, unit, n_slots}, n, channels, n_slots))
        return rc;
    RsPackets s;
    int32_t max_out;
    int smem;
    if (int rc = rs_packets(who, orig_freq, new_freq, max_in, &s, &max_out, &smem)) return rc;
    s.unit = unit;
    if (int rc = disjoint(who, channels, {{"x", x_row_stride, x_ch_stride, max_in}, {"y", y_row_stride, y_ch_stride, max_out}}))
        return rc;
    resample_packets_kernel<<<(unsigned)(n * channels), RS_TILE, smem, static_cast<cudaStream_t>(stream)>>>(
        x_dev, x_row_stride, x_ch_stride, y_dev, y_row_stride, y_ch_stride, channels, counts_dev, out_counts_dev, slots_dev,
        state_dev, n_slots, s);
    return launched(who);
}

extern "C" int l2h_hop_fifo_layout(int32_t capacity, int32_t* row_floats) {
    using namespace l2h;
    if (!row_floats) return fail(1, "l2h_hop_fifo_layout: null pointer");
    if (capacity < CHUNK_HOP || capacity > INT32_MAX - FF_HEAD - CHUNK_CARRY)
        return fail(1, "l2h_hop_fifo_layout: capacity " + std::to_string(capacity) + " cannot hold one hop of " +
                           std::to_string(CHUNK_HOP) + " samples");
    *row_floats = FF_HEAD + CHUNK_CARRY + capacity;
    return 0;
}

extern "C" int l2h_hop_fifo(const float* x_dev, int64_t x_row_stride, int64_t x_ch_stride, int32_t max_in,
                            const int32_t* counts_dev, int32_t unit, float* chunk_dev, int64_t chunk_row_stride,
                            int64_t chunk_ch_stride, int32_t* hops_dev, int32_t n, int32_t channels, int32_t frames,
                            const int32_t* slots_dev, float* state_dev, int32_t n_slots, int32_t capacity, void* stream) {
    using namespace l2h;
    const std::string who = "l2h_hop_fifo";
    if (int rc = slot_call(who, {x_dev, counts_dev, chunk_dev, hops_dev, slots_dev, state_dev},
                           "n, channels, max_in, unit, frames and n_slots", {n, channels, max_in, unit, frames, n_slots}, n,
                           channels, n_slots))
        return rc;
    int32_t row_floats;
    int64_t len, c_len;
    if (int rc = l2h_hop_fifo_layout(capacity, &row_floats)) return rc;
    if (int rc = hop_lens(who, frames, &len, &c_len)) return rc;
    if (int rc = disjoint(who, channels, {{"x", x_row_stride, x_ch_stride, max_in},
                                          {"chunk", chunk_row_stride, chunk_ch_stride, c_len}}))
        return rc;
    hop_fifo_kernel<<<(unsigned)(n * channels), RS_TILE, 0, static_cast<cudaStream_t>(stream)>>>(
        x_dev, x_row_stride, x_ch_stride, max_in, counts_dev, unit, chunk_dev, chunk_row_stride, chunk_ch_stride, hops_dev,
        channels, frames, slots_dev, state_dev, n_slots, capacity);
    return launched(who);
}

extern "C" int l2h_enroll_capture_layout(int32_t capacity, int32_t* row_floats) {
    using namespace l2h;
    if (!row_floats) return fail(1, "l2h_enroll_capture_layout: null pointer");
    if (capacity < EC_MIN_CAPACITY || capacity > INT32_MAX - EC_HEAD)
        return fail(1, "l2h_enroll_capture_layout: capacity " + std::to_string(capacity) + " cannot hold the " +
                           std::to_string(EC_MIN_CAPACITY) + " samples of the shortest enrollment");
    *row_floats = EC_HEAD + capacity;
    return 0;
}

extern "C" int l2h_enroll_capture(const float* chunk_dev, int64_t chunk_row_stride, int64_t chunk_ch_stride, int32_t n,
                                  int32_t channels, int32_t frames, const int32_t* slots_dev, const int32_t* hops_dev,
                                  float* state_dev, int32_t n_slots, int32_t capacity, void* stream) {
    using namespace l2h;
    const std::string who = "l2h_enroll_capture";
    if (int rc = slot_call(who, {chunk_dev, slots_dev, hops_dev, state_dev}, "n, channels, frames and n_slots",
                           {n, channels, frames, n_slots}, n, channels, n_slots))
        return rc;
    int32_t row_floats;
    int64_t len, c_len;
    if (int rc = l2h_enroll_capture_layout(capacity, &row_floats)) return rc;
    if (int rc = hop_lens(who, frames, &len, &c_len)) return rc;
    if (int rc = disjoint(who, channels, {{"chunk", chunk_row_stride, chunk_ch_stride, c_len}})) return rc;
    enroll_capture_kernel<<<(unsigned)(n * channels), RS_TILE, 0, static_cast<cudaStream_t>(stream)>>>(
        chunk_dev, chunk_row_stride, chunk_ch_stride, channels, frames, slots_dev, hops_dev, state_dev, n_slots, capacity);
    return launched(who);
}

extern "C" int l2h_target_mix_layout(int32_t* row_floats) {
    using namespace l2h;
    if (!row_floats) return fail(1, "l2h_target_mix_layout: null pointer");
    *row_floats = TM_FLOATS;
    return 0;
}

extern "C" int l2h_target_mix(const float* y_dev, int64_t y_row_stride, int64_t y_ch_stride, const float* chunk_dev,
                              int64_t chunk_row_stride, int64_t chunk_ch_stride, float* out_dev, int64_t out_row_stride,
                              int64_t out_ch_stride, int32_t n, int32_t R, int32_t channels, int32_t frames,
                              const int32_t* records_dev, const int32_t* offsets_dev, const int32_t* hops_dev,
                              const int32_t* slots_dev, float* state_dev, int32_t n_records, int32_t n_slots, void* stream) {
    using namespace l2h;
    const std::string who = "l2h_target_mix";
    if (int rc = slot_call(who, {y_dev, out_dev, records_dev, offsets_dev, slots_dev, state_dev},
                           "n, R, channels, frames, n_records and n_slots", {n, R, channels, frames, n_records, n_slots}, n,
                           channels, n_slots))
        return rc;
    if (n > R) return fail(1, who + ": a call needs n <= R (every listener row owns its target rows)");
    int64_t len, c_len;
    if (int rc = hop_lens(who, frames, &len, &c_len)) return rc;
    const Rows y{"y", y_row_stride, y_ch_stride, len}, out{"out", out_row_stride, out_ch_stride, len},
        ck{"chunk", chunk_row_stride, chunk_ch_stride, c_len};
    if (int rc = chunk_dev ? disjoint(who, channels, {y, ck, out}) : disjoint(who, channels, {y, out})) return rc;
    if (overlap(out_dev, n, out, y_dev, R, y, channels, false) ||
        overlap(out_dev, n, out, chunk_dev, n, ck, channels, false))
        return fail(1, who + ": out must not overlap y or the chunk");
    bool vec = true;                                    // float4 loads and stores where every operand allows them
    for (const Rows& r : {y, out, ck}) vec = vec && r.row % 4 == 0 && r.ch % 4 == 0;
    for (const void* p : {(const void*)y_dev, (const void*)out_dev, (const void*)chunk_dev})
        vec = vec && reinterpret_cast<uintptr_t>(p) % 16 == 0;
    const auto kernel = vec ? target_mix_kernel<4> : target_mix_kernel<1>;
    kernel<<<(unsigned)(n * channels), TM_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
        y_dev, y_row_stride, y_ch_stride, chunk_dev, chunk_row_stride, chunk_ch_stride, out_dev, out_row_stride,
        out_ch_stride, channels, R, frames, records_dev, offsets_dev, hops_dev, slots_dev, state_dev, n_records, n_slots);
    return launched(who);
}

extern "C" int l2h_target_mix_set(float* state_dev, int32_t n_records, int32_t n_slots, int32_t channels,
                                  const int32_t* rows_dev, int32_t n, const float* gains_dev, const float* starts_dev,
                                  const int32_t* fades_dev, void* stream) {
    using namespace l2h;
    const std::string who = "l2h_target_mix_set";
    for (const void* p : {(const void*)state_dev, (const void*)rows_dev, (const void*)gains_dev, (const void*)fades_dev})
        if (!p) return fail(1, who + ": null pointer");
    if (n_records <= 0 || n_slots <= 0 || channels <= 0 || n <= 0)
        return fail(1, who + ": n_records, n_slots, channels and n must be positive");
    if ((int64_t)n_records + n_slots > INT32_MAX || (int64_t)n * channels > INT32_MAX)
        return fail(1, who + ": n_records + n_slots or n * channels is too large");
    const int jobs = n * channels;
    target_mix_set_kernel<<<(unsigned)((jobs + RS_TILE - 1) / RS_TILE), RS_TILE, 0, static_cast<cudaStream_t>(stream)>>>(
        state_dev, n_records, n_records + n_slots, channels, rows_dev, n, gains_dev, starts_dev, fades_dev);
    return launched(who);
}

namespace l2h {
// the staged floats of a limiter row of `max_in` samples: 0, or an error code (1 invalid, 2 the staging exceeds shared
// memory) with its message
static int lm_staging(const std::string& who, int32_t channels, int32_t lookahead, int32_t max_in, int* smem) {
    if (channels <= 0) return fail(1, who + ": channels must be positive");
    if (lookahead < 0) return fail(1, who + ": lookahead " + std::to_string(lookahead) + " is negative");
    return staging(who, ((int64_t)channels + 2) * ((int64_t)lookahead + max_in),
                   std::to_string(channels) + " channels with a look-ahead of " + std::to_string(lookahead) +
                       " samples and pushes of up to " + std::to_string(max_in) + " samples are too large",
                   "words per row", smem);
}
}  // namespace l2h

extern "C" int l2h_limiter_layout(int32_t channels, int32_t lookahead, int32_t* row_floats) {
    using namespace l2h;
    if (!row_floats) return fail(1, "l2h_limiter_layout: null pointer");
    if (int rc = lm_staging("l2h_limiter_layout", channels, lookahead, 1, nullptr)) return rc;
    *row_floats = LM_HEAD + 3 * lookahead;
    return 0;
}

extern "C" int l2h_limiter(const float* x_dev, int64_t x_row_stride, int64_t x_ch_stride, int32_t max_in,
                           const int32_t* counts_dev, int32_t unit, float* y_dev, int64_t y_row_stride, int64_t y_ch_stride,
                           int32_t n, int32_t channels, const int32_t* slots_dev, float* state_dev, int32_t n_slots,
                           float ceiling, int32_t lookahead, int32_t release_step, void* stream) {
    using namespace l2h;
    const std::string who = "l2h_limiter";
    if (int rc = slot_call(who, {x_dev, counts_dev, y_dev, slots_dev, state_dev}, "n, channels, max_in, unit and n_slots",
                           {n, channels, max_in, unit, n_slots}, n, channels, n_slots))
        return rc;
    if (!(ceiling >= FLT_MIN && ceiling <= FLT_MAX))
        return fail(1, who + ": ceiling " + std::to_string(ceiling) + " is not a positive normal float");
    if (release_step <= 0 || release_step > LM_MUTE)
        return fail(1, who + ": release_step " + std::to_string(release_step) + " lies outside [1, " +
                           std::to_string(LM_MUTE) + "]");
    int smem;
    if (int rc = lm_staging(who, channels, lookahead, max_in, &smem)) return rc;
    const Rows x{"x", x_row_stride, x_ch_stride, max_in}, y{"y", y_row_stride, y_ch_stride, max_in};
    if (int rc = disjoint(who, channels, {x, y})) return rc;
    if (overlap(y_dev, n, y, x_dev, n, x, channels, false)) return fail(1, who + ": y must not overlap x");
    if (smem > RS_SMEM_BYTES - 1024)                                    // then the static words need the opt-in
        if (cudaError_t e = full_staging(limiter_kernel)) return fail(3, who + ": " + cudaGetErrorString(e));
    limiter_kernel<<<(unsigned)n, RS_TILE, smem, static_cast<cudaStream_t>(stream)>>>(
        x_dev, x_row_stride, x_ch_stride, max_in, counts_dev, unit, y_dev, y_row_stride, y_ch_stride, channels, slots_dev,
        state_dev, n_slots, ceiling, lookahead, release_step);
    return launched(who);
}

namespace l2h {
// The BS.1770 pre-filters at `rate` Hz from their analog prototypes, as libebur128 derives them (at 48 kHz they are the
// recommendation's table): a high shelf, then a high-pass whose numerator is 1, -2, 1.
static void lv_filters(double rate, LvParams* p) {
    double K = std::tan(M_PI * 1681.974450955533 / rate);
    const double Q = 0.7071752369554196, Vh = std::pow(10.0, 3.999843853973347 / 20.0);
    const double Vb = std::pow(Vh, 0.4996667741545416), a0 = 1.0 + K / Q + K * K;
    p->sb0 = (float)((Vh + Vb * K / Q + K * K) / a0);
    p->sb1 = (float)(2.0 * (K * K - Vh) / a0);
    p->sb2 = (float)((Vh - Vb * K / Q + K * K) / a0);
    p->sa1 = (float)(2.0 * (K * K - 1.0) / a0);
    p->sa2 = (float)((1.0 - K / Q + K * K) / a0);
    K = std::tan(M_PI * 38.13547087602444 / rate);
    const double Qh = 0.5003270373238773, ah = 1.0 + K / Qh + K * K;
    p->ha1 = (float)(2.0 * (K * K - 1.0) / ah);
    p->ha2 = (float)((1.0 - K / Qh + K * K) / ah);
}
}  // namespace l2h

extern "C" int l2h_leveler_layout(int32_t channels, int32_t* row_floats) {
    using namespace l2h;
    if (!row_floats) return fail(1, "l2h_leveler_layout: null pointer");
    if (channels <= 0) return fail(1, "l2h_leveler_layout: channels must be positive");
    *row_floats = LV_FLOATS;
    return 0;
}

extern "C" int l2h_leveler(const float* y_dev, int64_t y_row_stride, int64_t y_ch_stride, float* out_dev,
                           int64_t out_row_stride, int64_t out_ch_stride, int32_t n, int32_t R, int32_t channels,
                           int32_t frames, const int32_t* records_dev, const int32_t* offsets_dev, const int32_t* hops_dev,
                           float* state_dev, int32_t n_rows, float target, float gate, float relative, float alpha,
                           int32_t settle_hops, float min_gain, float max_gain, float rise_step, float fall_step,
                           void* stream) {
    using namespace l2h;
    const std::string who = "l2h_leveler";
    if (int rc = slot_call(who, {y_dev, out_dev, records_dev, state_dev}, "n, R, channels, frames and n_rows",
                           {n, R, channels, frames, n_rows}, n, channels, n_rows))
        return rc;
    if (n > R) return fail(1, who + ": a call needs n <= R (every listener row owns its rows)");
    int64_t len, c_len;
    if (int rc = hop_lens(who, frames, &len, &c_len)) return rc;
    for (float v : {target, gate, relative, min_gain, max_gain})
        if (!std::isfinite(v)) return fail(1, who + ": target, gate, relative, min_gain and max_gain must be finite");
    if (relative > 0.f) return fail(1, who + ": relative " + std::to_string(relative) + " dB is above 0");
    if (!(alpha > 0.f && alpha <= 1.f)) return fail(1, who + ": alpha " + std::to_string(alpha) + " lies outside (0, 1]");
    if (!(min_gain <= max_gain && min_gain >= -40.f && max_gain <= 40.f))
        return fail(1, who + ": the gain range [" + std::to_string(min_gain) + ", " + std::to_string(max_gain) +
                           "] dB is empty or leaves [-40, 40]");
    if (!(rise_step >= 0.f && fall_step >= 0.f && std::isfinite(rise_step) && std::isfinite(fall_step)))
        return fail(1, who + ": rise_step and fall_step must be finite and not negative");
    if (settle_hops < 1) return fail(1, who + ": settle_hops " + std::to_string(settle_hops) + " is below 1");
    const Rows y{"y", y_row_stride, y_ch_stride, len}, out{"out", out_row_stride, out_ch_stride, len};
    if (int rc = disjoint(who, channels, {y, out})) return rc;
    if (overlap(out_dev, R, out, y_dev, R, y, channels, true))
        return fail(1, who + ": out must be y itself (same pointer and strides) or not overlap it");
    LvParams p;
    lv_filters(16000.0, &p);
    p.target = target;
    p.gate = gate;
    p.relative = relative;
    p.alpha = alpha;
    p.min_gain = min_gain;
    p.max_gain = max_gain;
    p.rise = rise_step;
    p.fall = fall_step;
    p.settle = settle_hops;
    leveler_kernel<<<(unsigned)R, LV_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
        y_dev, y_row_stride, y_ch_stride, out_dev, out_row_stride, out_ch_stride, n, channels, frames, records_dev,
        offsets_dev, hops_dev, state_dev, n_rows, p);
    return launched(who);
}

namespace l2h {
// the bank's shape and a call's staging (taps, windows, band signals and gains): 0, or an error code (1 invalid, 2 the
// staging exceeds shared memory) with its message
static int bc_staging(const std::string& who, int32_t channels, int32_t bands, int32_t taps, int* kp, int* smem) {
    if (channels <= 0) return fail(1, who + ": channels must be positive");
    if (bands < 1 || bands > BC_MAX_BANDS)
        return fail(1, who + ": bands " + std::to_string(bands) + " lies outside [1, " + std::to_string(BC_MAX_BANDS) + "]");
    if (taps < BC_MIN_TAPS || taps > BC_MAX_TAPS || taps % 2 == 0)
        return fail(1, who + ": taps " + std::to_string(taps) + " is not odd in [" + std::to_string(BC_MIN_TAPS) + ", " +
                           std::to_string(BC_MAX_TAPS) + "]");
    *kp = (bands + 3) / 4 * 4;                          // the kernel reads each tap row as float4
    const int64_t floats = (int64_t)taps * *kp + (int64_t)channels * (taps - 1 + CHUNK_HOP) +
                           (int64_t)channels * bands * (CHUNK_HOP + 2);
    return staging(who, floats, std::to_string(channels) + " channels of " + std::to_string(bands) + " bands of " +
                                    std::to_string(taps) + " taps are too large", "words per row", smem);
}
}  // namespace l2h

extern "C" int l2h_band_compressor_design(int32_t bands, const float* edges_hz, int32_t taps, float* out) {
    using namespace l2h;
    const std::string who = "l2h_band_compressor_design";
    if (!out || (bands > 1 && !edges_hz)) return fail(1, who + ": null pointer");
    int kp;
    if (int rc = bc_staging(who, 1, bands, taps, &kp, nullptr)) return rc;   // one channel always fits
    for (int j = 0; j + 1 < bands; ++j) {
        const float e = edges_hz[j];
        if (!(e > 0.f && e < 8000.f) || (j > 0 && !(e > edges_hz[j - 1])))
            return fail(1, who + ": the edges must rise strictly inside (0, 8000) Hz, got edge " + std::to_string(j) + " = " +
                               std::to_string(e));
    }
    // LP_j: scipy.signal.firwin(taps, edge_j, fs=16000), a Hamming-windowed sinc scaled to a DC gain of 1; band 0 is LP_1,
    // band j LP_{j+1} - LP_j, the last band the delay D minus LP_{K-1}, all in float64
    const int L = taps, D = (L - 1) / 2;
    std::vector<double> prev(L, 0.0), lp(L);
    for (int b = 0; b < bands; ++b) {
        if (b + 1 < bands) {
            const double cut = edges_hz[b] / 8000.0;
            double sum = 0.0;
            for (int i = 0; i < L; ++i) {
                const double m = i - D, u = M_PI * cut * m;
                const double win = 0.54 - 0.46 * std::cos(2.0 * M_PI * i / (L - 1));
                lp[i] = cut * (m == 0 ? 1.0 : std::sin(u) / u) * win;
                sum += lp[i];
            }
            for (double& v : lp) v /= sum;
        } else {
            for (int i = 0; i < L; ++i) lp[i] = i == D ? 1.0 : 0.0;
        }
        for (int i = 0; i < L; ++i) out[(int64_t)b * L + i] = (float)(lp[i] - prev[i]);
        prev.swap(lp);
    }
    return 0;
}

extern "C" int l2h_band_compressor_layout(int32_t channels, int32_t bands, int32_t taps, int32_t* row_floats) {
    using namespace l2h;
    if (!row_floats) return fail(1, "l2h_band_compressor_layout: null pointer");
    int kp;
    if (int rc = bc_staging("l2h_band_compressor_layout", channels, bands, taps, &kp, nullptr)) return rc;
    *row_floats = 5 * bands + taps - 1;
    return 0;
}

extern "C" int l2h_band_compressor(const float* y_dev, int64_t y_row_stride, int64_t y_ch_stride, float* out_dev,
                                   int64_t out_row_stride, int64_t out_ch_stride, int32_t n, int32_t channels, int32_t frames,
                                   const int32_t* slots_dev, const int32_t* hops_dev, const float* taps_dev, int32_t bands,
                                   int32_t taps, float* state_dev, int32_t n_slots, float attack, float release,
                                   void* stream) {
    using namespace l2h;
    const std::string who = "l2h_band_compressor";
    if (int rc = slot_call(who, {y_dev, out_dev, slots_dev, taps_dev, state_dev}, "n, channels, frames and n_slots",
                           {n, channels, frames, n_slots}, n, channels, n_slots))
        return rc;
    int64_t len, c_len;
    if (int rc = hop_lens(who, frames, &len, &c_len)) return rc;
    if (!(attack > 0.f && attack <= 1.f) || !(release > 0.f && release <= 1.f))
        return fail(1, who + ": attack " + std::to_string(attack) + " and release " + std::to_string(release) +
                           " must lie in (0, 1]");
    int kp, smem;
    if (int rc = bc_staging(who, channels, bands, taps, &kp, &smem)) return rc;
    const Rows y{"y", y_row_stride, y_ch_stride, len}, out{"out", out_row_stride, out_ch_stride, len};
    if (int rc = disjoint(who, channels, {y, out})) return rc;
    if (overlap(out_dev, n, out, y_dev, n, y, channels, true))
        return fail(1, who + ": out must be y itself (same pointer and strides) or not overlap it");
    const auto kernel = kp == 4 ? band_compressor_kernel<4> : kp == 8 ? band_compressor_kernel<8>
                      : kp == 12 ? band_compressor_kernel<12> : band_compressor_kernel<16>;
    if (smem > RS_SMEM_BYTES - 1024)                                    // then the static words need the opt-in
        if (cudaError_t e = full_staging(kernel)) return fail(3, who + ": " + cudaGetErrorString(e));
    kernel<<<(unsigned)n, BC_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
        y_dev, y_row_stride, y_ch_stride, out_dev, out_row_stride, out_ch_stride, channels, frames, slots_dev, hops_dev,
        taps_dev, bands, taps, state_dev, n_slots, attack, release);
    return launched(who);
}

namespace l2h {
// the Linkwitz-Riley bank's shape and a call's staging (the sections, the staged hop, band signals and gains): 0, or
// an error code (1 invalid, 2 the staging exceeds shared memory) with its message; *ns the sections per band
static int lr_staging(const std::string& who, int32_t channels, int32_t bands, int32_t order, int* ns, int* smem) {
    if (channels <= 0) return fail(1, who + ": channels must be positive");
    if (bands < 1 || bands > BC_MAX_BANDS)
        return fail(1, who + ": bands " + std::to_string(bands) + " lies outside [1, " + std::to_string(BC_MAX_BANDS) + "]");
    if (order != 4 && order != 8) return fail(1, who + ": order " + std::to_string(order) + " is not 4 or 8");
    *ns = order / 2 * (bands - 1);
    const int64_t floats = (int64_t)bands * *ns * 5 + (int64_t)channels * CHUNK_HOP +
                           (int64_t)channels * bands * (CHUNK_HOP + 2);
    return staging(who, floats, std::to_string(channels) + " channels of " + std::to_string(bands) + " bands of order " +
                                    std::to_string(order) + " are too large", "words per row", smem);
}

// the biquads (b0, b1, b2, a1, a2) of a Butterworth filter of order n (even) cut at f Hz, by the bilinear transform
// prewarped at f, as scipy.signal.butter(n, f, fs=16000) designs it; `kind` 'l' low-pass, 'h' high-pass, 'a' the allpass
// on the same poles.  Section k holds the poles at angles pi (2 k + 1) / (2 n) from the negative real axis.
static std::vector<double> lr_butter(int n, double f, char kind) {
    std::vector<double> out;
    const double K = std::tan(M_PI * f / 16000.0), K2 = K * K;
    for (int k = 0; k < n / 2; ++k) {
        const double d = 2.0 * std::sin(M_PI * (2 * k + 1) / (2.0 * n));   // 1 / Q
        const double norm = 1.0 / (1.0 + d * K + K2);
        const double a1 = 2.0 * (K2 - 1.0) * norm, a2 = (1.0 - d * K + K2) * norm;
        if (kind == 'l') out.insert(out.end(), {K2 * norm, 2.0 * K2 * norm, K2 * norm, a1, a2});
        else if (kind == 'h') out.insert(out.end(), {norm, -2.0 * norm, norm, a1, a2});
        else out.insert(out.end(), {a2, a1, 1.0, a1, a2});
    }
    return out;
}

using LrKernel = decltype(&band_compressor_lr_kernel<1, 4>);

template <int N, int... K>
static LrKernel lr_kernel_of(int bands, std::integer_sequence<int, K...>) {
    static const LrKernel table[] = {band_compressor_lr_kernel<K + 1, N>...};
    return table[bands - 1];
}

// the instantiation for `bands` in [1, BC_MAX_BANDS] and `order` 4 or 8
static LrKernel lr_kernel(int bands, int order) {
    const auto K = std::make_integer_sequence<int, BC_MAX_BANDS>{};
    return order == 4 ? lr_kernel_of<4>(bands, K) : lr_kernel_of<8>(bands, K);
}
}  // namespace l2h

extern "C" int l2h_band_compressor_lr_design(int32_t bands, const float* edges_hz, int32_t order, float* out) {
    using namespace l2h;
    const std::string who = "l2h_band_compressor_lr_design";
    if (!out || (bands > 1 && !edges_hz)) return fail(1, who + ": null pointer");
    int ns;
    if (int rc = lr_staging(who, 1, bands, order, &ns, nullptr)) return rc;
    for (int j = 0; j + 1 < bands; ++j) {
        const float e = edges_hz[j];
        if (!(e > 0.f && e < 8000.f) || (j > 0 && !(e > edges_hz[j - 1])))
            return fail(1, who + ": the edges must rise strictly inside (0, 8000) Hz, got edge " + std::to_string(j) + " = " +
                               std::to_string(e));
    }
    // band b: HP of edges 0 .. b - 1, the LP of edge b (not the last band), the AP of edges b + 1 .. K - 2, each LR
    // filter the Butterworth sections twice; then identity sections up to ns, all in float64
    const int n = order / 2;
    for (int b = 0; b < bands; ++b) {
        std::vector<double> sec;
        const auto add = [&](const std::vector<double>& v, int times) {
            for (int r = 0; r < times; ++r) sec.insert(sec.end(), v.begin(), v.end());
        };
        for (int e = 0; e < b; ++e) add(lr_butter(n, edges_hz[e], 'h'), 2);
        if (b + 1 < bands) add(lr_butter(n, edges_hz[b], 'l'), 2);
        for (int e = b + 1; e + 1 < bands; ++e) add(lr_butter(n, edges_hz[e], 'a'), 1);
        while ((int)sec.size() < 5 * ns) sec.insert(sec.end(), {1.0, 0.0, 0.0, 0.0, 0.0});
        for (int i = 0; i < 5 * ns; ++i) out[(int64_t)b * 5 * ns + i] = (float)sec[i];
    }
    return 0;
}

extern "C" int l2h_band_compressor_lr_layout(int32_t channels, int32_t bands, int32_t order, int32_t* row_floats) {
    using namespace l2h;
    if (!row_floats) return fail(1, "l2h_band_compressor_lr_layout: null pointer");
    int ns;
    if (int rc = lr_staging("l2h_band_compressor_lr_layout", channels, bands, order, &ns, nullptr)) return rc;
    *row_floats = 5 * bands + 2 * bands * ns;
    return 0;
}

extern "C" int l2h_band_compressor_lr(const float* y_dev, int64_t y_row_stride, int64_t y_ch_stride, float* out_dev,
                                      int64_t out_row_stride, int64_t out_ch_stride, int32_t n, int32_t channels,
                                      int32_t frames, const int32_t* slots_dev, const int32_t* hops_dev,
                                      const float* sos_dev, int32_t bands, int32_t order, float* state_dev,
                                      int32_t n_slots, float attack, float release, void* stream) {
    using namespace l2h;
    const std::string who = "l2h_band_compressor_lr";
    if (int rc = slot_call(who, {y_dev, out_dev, slots_dev, sos_dev, state_dev}, "n, channels, frames and n_slots",
                           {n, channels, frames, n_slots}, n, channels, n_slots))
        return rc;
    int64_t len, c_len;
    if (int rc = hop_lens(who, frames, &len, &c_len)) return rc;
    if (!(attack > 0.f && attack <= 1.f) || !(release > 0.f && release <= 1.f))
        return fail(1, who + ": attack " + std::to_string(attack) + " and release " + std::to_string(release) +
                           " must lie in (0, 1]");
    int ns, smem;
    if (int rc = lr_staging(who, channels, bands, order, &ns, &smem)) return rc;
    const Rows y{"y", y_row_stride, y_ch_stride, len}, out{"out", out_row_stride, out_ch_stride, len};
    if (int rc = disjoint(who, channels, {y, out})) return rc;
    if (overlap(out_dev, n, out, y_dev, n, y, channels, true))
        return fail(1, who + ": out must be y itself (same pointer and strides) or not overlap it");
    const auto kernel = lr_kernel(bands, order);
    if (smem > RS_SMEM_BYTES - 1024)                                    // then the static words need the opt-in
        if (cudaError_t e = full_staging(kernel)) return fail(3, who + ": " + cudaGetErrorString(e));
    kernel<<<(unsigned)n, BC_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
        y_dev, y_row_stride, y_ch_stride, out_dev, out_row_stride, out_ch_stride, channels, frames, slots_dev, hops_dev,
        sos_dev, state_dev, n_slots, attack, release);
    return launched(who);
}

// ---- the jitter buffer: packets back in sequence order, losses concealed ----------------------------------------------
// Packets of P samples carry RTP's 16-bit sequence numbers, compared in serial-number arithmetic (RFC 1982).  A slot keeps
// `next`, the sequence number of the next packet to decide, a window of the W numbers next .. next + W - 1 (the packets
// stored there wait for their turn), and a backlog of up to W decided packets its calls have not written yet, so a packet
// is placed, released or declared lost from the arrivals alone: cutting them into other calls, or another max_out,
// changes no decision.  Thread 0 runs each row's arrivals in order on ring tags staged in shared memory; all threads then
// copy the stored packets into the ring and write the decided ones, concealing a lost one by repeating the last pitch
// period (found by a normalised autocorrelation over the lags in parallel, each lag's sums in one fixed order) with a gain
// that holds for 10 ms and falls to 0 by 60 ms, and fading the first real packet after a run or a restart in from the
// continuing concealment along a raised cosine.
//
// A slot's row per channel is [JB_HEAD + R + R P + H + tau_max] floats, R = 2 W: the head words and the R ring tags
// (channel 0's only), the ring of R packets, the last H = Wc + tau_max written samples, and the period being repeated.
// A tag is 0 (empty), s + 1 for a stored packet s (| JB_RECOVER for a released one that fades in), or JB_LOST (a
// released loss); a backlog entry with any other tag is concealed.  The backlog occupies ring positions head .. head + pend - 1, the window the W after it.
namespace l2h {
constexpr int JB_HEAD = 16;
constexpr int JB_LOST = -1;
constexpr int JB_RECOVER = 1 << 17;
constexpr int JB_SEQ = 1 << 16;
constexpr int JB_MAX_WINDOW = 4096;
// head words (int32 in the floats' bits): started, next, head, pend, run (concealed samples into the run, capped at its
// silent point), tau (0: no run), then the counters lost, late, duplicate, dropped, restarts, and held and pitch; the
// timed form adds the anchor (the highest packet placed and the clock of its call) and the counter expired
enum { JB_STARTED, JB_NEXT, JB_POS, JB_PEND, JB_RUN, JB_TAU, JB_C_LOST, JB_C_LATE, JB_C_DUP, JB_C_DROPPED, JB_C_RESTARTS,
       JB_HELD, JB_PITCH, JB_ANCHOR_SEQ, JB_ANCHOR_T, JB_C_EXPIRED };

struct JbParams {
    int32_t P, W, R, D, M, max_out;   // packet, window, ring (2 W), depth, arrivals per row, packets written per row
    int32_t tmin, tmax, wc, hist;     // lags, correlation window, history H = wc + tmax
    int32_t lr, ga, gb;               // crossfade samples; a run's gain is 1 before sample ga, 0 from sample gb
    int64_t rf;                       // floats per channel row
};

// the timed form's clock: the server's clock (µs, int32 that wraps) read when the kernel runs, the deadline (µs), the
// packet period (µs, mod 2^32) and the stall S (packets past the anchor after which deadline releases stop)
struct JbClock {
    const int32_t* now;
    int32_t deadline;
    uint32_t period;
    int32_t stall;
};

// The adaptive form: the timed form whose deadline is drawn per slot from a histogram of the lateness of its packets.
// Channel 0's row ends in a block of JB_STATS words (int32): JB_BINS bins summing to about JB_UNIT, the packets
// measured (saturating), and the deadline of the slot's last call.
constexpr int JB_BINS = 64;
constexpr int JB_STATS = JB_BINS + 2;
constexpr int JB_UNIT = 1 << 24;
constexpr int JB_BIN_MAX = 1 << 30;    // a bin read from the state is clamped to [0, JB_BIN_MAX]
enum { JB_UNTIMED, JB_TIMED, JB_ADAPTIVE };

// the adaptive form's parameters: the arrival times [n][M] (µs, or null: every packet arrives at now), the bounds of the
// deadline, the bin width w = max(1, ceil(hi / 64)), r = round(late_rate 2^16), the warm-up ceil(1 / late_rate)
// (packets measured before the quantile is used) and the memory N = max(1, round(5e6 / period)) in packets
struct JbAdapt {
    const int32_t* arrivals;
    int32_t lo, hi, w, r, warm, mem;
};

// a difference of 16-bit sequence numbers in serial arithmetic: v mod 2^16 taken in [-2^15, 2^15)
L2H_DEVINL int jb_ser(int v) {
    v &= JB_SEQ - 1;
    return v >= JB_SEQ / 2 ? v - JB_SEQ : v;
}

// a sample as it enters: 0 when it is not finite or its magnitude is 2^32 or more
L2H_DEVINL float jb_clean(float v) { return fabsf(v) < HG_BIG ? v : 0.f; }

// the gain of concealed sample k of a run
L2H_DEVINL float jb_gain(int k, const JbParams& p) {
    return k < p.ga ? 1.f : (k >= p.gb ? 0.f : (float)(p.gb - k) / (float)(p.gb - p.ga));
}

// The lag of the period that ends at the history win[c][base + H] (every thread calls it): the first maximiser over
// tmin .. tmax of sum_k s[k] s[k - t] / sqrt(max(sum_k s[k - t]^2, FLT_MIN)) over the last wc samples of the channel
// sum s, tmax when no numerator is positive.
L2H_DEVINL int jb_pitch(const float* win, int64_t WL, int base, int C, float* sum, float* sc, int* lt, int* tau,
                        const JbParams& p) {
    const int tid = threadIdx.x, H = p.hist;
    for (int i = tid; i < H; i += blockDim.x) {
        float a = win[base + i];
        for (int c = 1; c < C; ++c) a += win[c * WL + base + i];
        sum[i] = a;
    }
    __syncthreads();
    float best = -1.f;
    int bt = p.tmax;
    const float* a = sum + H - p.wc;
    for (int t = p.tmin + tid; t <= p.tmax; t += blockDim.x) {
        const float* b = a - t;
        float num = 0.f, en = 0.f;
        for (int k = 0; k < p.wc; ++k) {
            num = fmaf(a[k], b[k], num);
            en = fmaf(b[k], b[k], en);
        }
        if (num > 0.f) {
            const float score = num / sqrtf(fmaxf(en, FLT_MIN));
            if (score > best) best = score, bt = t;
        }
    }
    sc[tid] = best;
    lt[tid] = bt;
    __syncthreads();
    if (tid == 0) {
        float b0 = -1.f;
        int t0 = p.tmax;
        for (int i = 0; i < (int)blockDim.x; ++i)
            if (sc[i] > b0 || (sc[i] == b0 && lt[i] < t0)) b0 = sc[i], t0 = lt[i];
        *tau = t0;
    }
    __syncthreads();
    return *tau;
}

// the histogram bin of a lateness of l µs: floor(l / w) clamped to [0, JB_BINS - 1]
L2H_DEVINL int jb_bin(int l, int w) { return l < 0 ? 0 : min(l / w, JB_BINS - 1); }

// The adaptive form's statistics, run by warp 0 of a row whose slot has started (every lane calls it): the `nm`
// lateness bins mb[] of this call, in arrival order, enter the slot's block sb (lane l owns bins 2 l and 2 l + 1); then
// the deadline is found by a suffix scan over the bins.  Returns the deadline (on every lane) and writes the block.
L2H_DEVINL int jb_stats(float* sb, const int* mb, int nm, const JbAdapt& ad) {
    const int lane = threadIdx.x;
    int h0 = min(max(__float_as_int(sb[2 * lane]), 0), JB_BIN_MAX);
    int h1 = min(max(__float_as_int(sb[2 * lane + 1]), 0), JB_BIN_MAX);
    int k = max(__float_as_int(sb[JB_BINS]), 0);
    for (int j = 0; j < nm; ++j) {                                      // packet k is weighted 1 / min(k + 1, N)
        const int m = min(k, ad.mem - 1) + 1, b = mb[j];
        h0 -= h0 / m;
        h1 -= h1 / m;
        if (b == 2 * lane) h0 += JB_UNIT / m;
        if (b == 2 * lane + 1) h1 += JB_UNIT / m;
        k += k < INT32_MAX;
    }
    const int64_t pair = (int64_t)h0 + h1;
    int64_t suf = pair;                                                 // bins 2 lane .. 63
    for (int o = 1; o < 32; o <<= 1) {
        const int64_t v = __shfl_down_sync(~0u, suf, o);
        if (lane + o < 32) suf += v;
    }
    const int64_t total = __shfl_sync(~0u, suf, 0), lim = (int64_t)ad.r * total;
    const int64_t t1 = suf - pair, t0 = t1 + h1;                        // the tails beyond bins 2 lane + 1 and 2 lane
    const unsigned q0 = __ballot_sync(~0u, (t0 << 16) <= lim), q1 = __ballot_sync(~0u, (t1 << 16) <= lim);
    // the smallest bin whose tail holds at most the fraction: q1 always holds on lane 31 (its tail is 0)
    const int b = min(q0 ? 2 * (__ffs(q0) - 1) : JB_BINS, 2 * (__ffs(q1) - 1) + 1);
    const int dl = k < ad.warm ? ad.hi : (int)min(max((int64_t)(b + 1) * ad.w, (int64_t)ad.lo), (int64_t)ad.hi);
    sb[2 * lane] = __int_as_float(h0);
    sb[2 * lane + 1] = __int_as_float(h1);
    if (lane == 0) {
        sb[JB_BINS] = __int_as_float(k);
        sb[JB_BINS + 1] = __int_as_float(dl);
    }
    return dl;
}

// One CTA = one call row over all C channels (one decision per slot).  Row i pushes packets j < counts[i] of x row i
// with sequence numbers seqs[i][j] and writes y[i][c][0 .. out_counts[i] P).  Timed: the arrivals also keep the anchor,
// an arrival at or past next restarts a stalled slot, and after them a missing next is also released as a loss once its
// deadline on the clock has passed (`ck`; unused untimed).  Adaptive: as timed, with each packet's own arrival time, the
// lateness of the measured arrivals kept in the slot's statistics block by warp 0 between thread 0's arrivals and its
// release at now, and the deadline the block gives (`ad`; unused otherwise).
template <int Mode>
L2H_DEVINL void jb_row(const float* __restrict__ x, int64_t x_row, int64_t x_ch, const int32_t* __restrict__ seqs,
                       const int32_t* __restrict__ counts, float* __restrict__ y, int64_t y_row, int64_t y_ch,
                       int32_t* __restrict__ out_counts, int C, const int32_t* __restrict__ slots, float* __restrict__ state,
                       int n_slots, const JbParams& p, const JbClock& ck, const JbAdapt& ad) {
    constexpr bool Timed = Mode != JB_UNTIMED, Adaptive = Mode == JB_ADAPTIVE;
    extern __shared__ float sm[];
    __shared__ float sc[RS_TILE];
    __shared__ int lt[RS_TILE];
    __shared__ int n_out_s, tau_s;
    const int tid = threadIdx.x, P = p.P, R = p.R, W = p.W, H = p.hist;
    const int64_t rf = p.rf, WL = H + (int64_t)p.max_out * P;
    const SlotRow sr = slot_row(1, slots, n_slots, state, C * rf);
    const int cnt = counts[sr.row];
    if (!sr.live || cnt < 0 || cnt > p.M) {                             // a row that stores nothing
        if (tid == 0) out_counts[sr.row] = 0;
        return;
    }
    float* st = sr.st;                                                  // channel c's row at st + c rf
    float* win = sm;                                                    // [C][WL]: the history, then the packets written
    float* sum = win + C * WL;                                          // [H]: the channel sum of a search
    float* per = sum + H;                                               // [C][tmax]: the period being repeated
    int* tg = reinterpret_cast<int*>(per + (int64_t)C * p.tmax);        // [R]: the ring tags
    int* cp = tg + R;                                                   // [M]: the ring slot of each arrival, or -1
    int* kind = cp + p.M;                                               // [max_out]: the tag of each packet written
    const int64_t o_ring = JB_HEAD + R, o_hist = o_ring + (int64_t)R * P, o_per = o_hist + H;
    for (int i = tid; i < R; i += blockDim.x) tg[i] = __float_as_int(st[JB_HEAD + i]);
    for (int c = 0; c < C; ++c) {
        for (int i = tid; i < H; i += blockDim.x) win[c * WL + i] = st[c * rf + o_hist + i];
        for (int i = tid; i < p.tmax; i += blockDim.x) per[c * p.tmax + i] = st[c * rf + o_per + i];
    }
    __syncthreads();
    // thread 0's bookkeeping; in the adaptive form warp 0 enters too, and between thread 0's arrivals and its release
    // at now it keeps the slot's statistics and finds its deadline
    __shared__ int nm_s;
    if (Adaptive ? tid < 32 : tid == 0) {
        int started = __float_as_int(st[JB_STARTED]) != 0, next = int_word(st[JB_NEXT], JB_SEQ - 1);
        int pos = int_word(st[JB_POS], R - 1), pend = int_word(st[JB_PEND], W);
        int lost = 0, late = 0, dup = 0, dropped = 0, restarts = 0;
        const auto slot = [&](int d) { return (pos + pend + d) % R; };
        const auto held = [&](int d) { return tg[slot(d)] == ((next + d) & (JB_SEQ - 1)) + 1; };
        int far = -1;                                                   // the farthest stored packet in the window
        if (!Adaptive || tid == 0)
            for (int d = 0; d < W; ++d) if (held(d)) far = d;
        // timed: the anchor (a_s, a_t), the clock of this call and the deadline releases
        int a_s = 0, expired = 0;
        uint32_t a_t = 0, now = 0;
        if constexpr (Timed) {
            a_s = int_word(st[JB_ANCHOR_SEQ], JB_SEQ - 1), a_t = (uint32_t)__float_as_int(st[JB_ANCHOR_T]);
            now = (uint32_t)*ck.now;
        }
        // the concealment has gone silent: no deadline releases, and the next arrival at or past next restarts
        const auto stalled = [&] { return Timed && jb_ser(next - a_s - 1) >= ck.stall; };
        const int32_t* sq = seqs + (int64_t)sr.row * p.M;
        int* mb = kind + p.max_out;                                     // adaptive: [M] the bins of the measured arrivals
        int nm = 0;
        if (!Adaptive || tid == 0) {                                    // the arrivals
            for (int j = 0; j < cnt; ++j) {
                cp[j] = -1;
                const int s = sq[j];
                if (s < 0 || s >= JB_SEQ) continue;                         // no sequence number: skipped
                // adaptive: the packet's arrival (now without arrival times, or when it lies after now), and the
                // bin of its lateness against the anchor in force (for the packets measured: not the slot's first)
                uint32_t arr = now;
                const bool first = !started;
                if constexpr (Adaptive)
                    if (ad.arrivals) {
                        const uint32_t a = (uint32_t)ad.arrivals[(int64_t)sr.row * p.M + j];
                        if ((int)(a - now) < 0) arr = a;
                    }
                const auto measure = [&] {
                    mb[nm++] = jb_bin((int)(arr - (a_t + (uint32_t)jb_ser(s - a_s) * ck.period)), ad.w);
                };
                if (!started) started = 1, next = s, a_s = s;
                int d = (s - next) & (JB_SEQ - 1);
                if (d >= JB_SEQ / 2) d -= JB_SEQ;
                bool recover = false;
                if (d < 0) {
                    late = min(late + 1, INT32_MAX - 1);
                    if constexpr (Adaptive) if (!stalled()) measure();     // a late packet is measured
                    continue;
                }
                if (d < W && !stalled()) {
                    if (held(d)) { dup = min(dup + 1, INT32_MAX - 1); continue; }
                    if constexpr (Adaptive) if (!first) measure();
                } else {                                                    // beyond the window (or stalled): a restart
                    for (int e = 0; e < W; ++e) {
                        if (held(e)) dropped = min(dropped + 1, INT32_MAX - 1);
                        tg[slot(e)] = 0;
                    }
                    restarts = min(restarts + 1, INT32_MAX - 1);
                    next = s, d = 0, far = -1, recover = true, a_s = s;
                }
                if constexpr (Timed)                            // the first packet, a restart, or a new highest
                    if (jb_ser(s - a_s) >= 0) a_s = s, a_t = arr;
                const int at = slot(d);
                tg[at] = s + 1;
                for (int k = 0; k < j; ++k) if (cp[k] == at) cp[k] = -1;    // a slot freed and reused in this call
                cp[j] = at;
                far = max(far, d);
                for (;;) {                                                  // the release rule
                    int t;
                    if (held(0)) t = (next + 1) | (recover ? JB_RECOVER : 0), recover = false;
                    else if (far >= p.D + 1) t = JB_LOST, lost = min(lost + 1, INT32_MAX - 1);
                    else break;
                    if (pend == W) {                                        // the backlog is full: its oldest goes
                        tg[pos] = 0;
                        pos = (pos + 1) % R, --pend;
                        dropped = min(dropped + 1, INT32_MAX - 1);
                    }
                    tg[(pos + pend) % R] = t;
                    ++pend, next = (next + 1) & (JB_SEQ - 1), --far;
                }
            }
        }
        int deadline = ck.deadline;
        if constexpr (Adaptive) {                                       // a slot that has started: its statistics
            if (tid == 0) nm_s = started ? nm : -1;
            __syncwarp();
            deadline = nm_s >= 0 ? jb_stats(st + rf - JB_STATS, mb, nm_s, ad) : ad.hi;
        }
        if (!Adaptive || tid == 0) {
            if constexpr (Timed) {
                // the release rule once more at now, with a third way to release next: it expired (packet s is
                // expected at a_t + (s - a_s) period) and the slot has not stalled
                while (started) {
                    int t;
                    if (held(0)) t = next + 1;
                    else if (far >= p.D + 1) t = JB_LOST, lost = min(lost + 1, INT32_MAX - 1);
                    else if (!stalled() && (int)(now - (a_t + (uint32_t)jb_ser(next - a_s) * ck.period)) >= deadline)
                        t = JB_LOST, lost = min(lost + 1, INT32_MAX - 1), expired = min(expired + 1, INT32_MAX - 1);
                    else break;
                    if (pend == W) {
                        tg[pos] = 0;
                        pos = (pos + 1) % R, --pend;
                        dropped = min(dropped + 1, INT32_MAX - 1);
                    }
                    tg[(pos + pend) % R] = t;
                    ++pend, next = (next + 1) & (JB_SEQ - 1), --far;
                }
            }
            const int n_out = min(pend, p.max_out);
            for (int k = 0; k < n_out; ++k) {                               // what each written packet is
                // a released packet plays whatever its number: a restart may lie between it and next; a malformed
                // tag conceals
                const int at = (pos + k) % R, t = tg[at], s1 = t & ~JB_RECOVER;
                kind[k] = s1 >= 1 && s1 <= JB_SEQ ? t : JB_LOST;
                tg[at] = 0;
            }
            pos = (pos + n_out) % R, pend -= n_out;
            int nheld = 0;
            for (int d = 0; d < W; ++d) nheld += held(d);
            st[JB_STARTED] = __int_as_float(started);
            st[JB_NEXT] = __int_as_float(next);
            st[JB_POS] = __int_as_float(pos);
            st[JB_PEND] = __int_as_float(pend);
            st[JB_C_LOST] = add_word(st[JB_C_LOST], lost);
            st[JB_C_LATE] = add_word(st[JB_C_LATE], late);
            st[JB_C_DUP] = add_word(st[JB_C_DUP], dup);
            st[JB_C_DROPPED] = add_word(st[JB_C_DROPPED], dropped);
            st[JB_C_RESTARTS] = add_word(st[JB_C_RESTARTS], restarts);
            st[JB_HELD] = __int_as_float(nheld);
            if constexpr (Timed) {
                st[JB_ANCHOR_SEQ] = __int_as_float(a_s);
                st[JB_ANCHOR_T] = __int_as_float((int)a_t);
                st[JB_C_EXPIRED] = add_word(st[JB_C_EXPIRED], expired);
            }
            out_counts[sr.row] = n_out;
            n_out_s = n_out;
        }
    }
    __syncthreads();
    const int n_out = n_out_s;
    for (int i = tid; i < R; i += blockDim.x) st[JB_HEAD + i] = __int_as_float(tg[i]);
    const int64_t per_row = (int64_t)C * P;
    for (int64_t e = tid; e < (int64_t)cnt * per_row; e += blockDim.x) {   // the stored packets into the ring
        const int j = (int)(e / per_row), r = (int)(e - j * per_row), c = r / P, i = r - c * P;
        if (cp[j] >= 0) st[c * rf + o_ring + (int64_t)cp[j] * P + i] = jb_clean(row_ch(x, x_row, x_ch, sr.row, c)[(int64_t)j * P + i]);
    }
    __syncthreads();                                                    // the ring, visible to the block
    int run = int_word(st[JB_RUN], p.gb), tau = __float_as_int(st[JB_TAU]);
    if (tau < p.tmin || tau > p.tmax) tau = 0;
    const int pos0 = int_word(st[JB_POS], R - 1) - n_out;               // the ring slot of the first packet written
    for (int k = 0; k < n_out; ++k) {
        const int t = kind[k], base = k * P;
        if (tau == 0 && t != JB_LOST && !(t & JB_RECOVER)) {            // a packet in order: copied as it is
            const int at = (pos0 + k + R) % R;
            for (int e = tid; e < C * P; e += blockDim.x) {
                const int c = e / P, i = e - c * P;
                const float v = st[c * rf + o_ring + (int64_t)at * P + i];
                win[c * WL + H + base + i] = v;
                row_ch(y, y_row, y_ch, sr.row, c)[base + i] = v;
            }
            __syncthreads();
            continue;
        }
        if (tau == 0) {                                                 // a run starts: find its period
            tau = jb_pitch(win, WL, base, C, sum, sc, lt, &tau_s, p);
            run = 0;
            for (int e = tid; e < C * tau; e += blockDim.x) {
                const int c = e / tau, i = e - c * tau;
                per[c * p.tmax + i] = win[c * WL + base + H - tau + i];
            }
            if (tid == 0) st[JB_PITCH] = __int_as_float(tau);
            __syncthreads();
        }
        const int at = (pos0 + k + R) % R;
        for (int e = tid; e < C * P; e += blockDim.x) {
            const int c = e / P, i = e - c * P;
            const int q = min(run + i, p.gb);
            const float cont = jb_gain(q, p) * per[c * p.tmax + (run + i) % tau];
            float v = cont;
            if (t != JB_LOST) {                                         // the fade from the concealment to the packet
                const float r = st[c * rf + o_ring + (int64_t)at * P + i];
                if (i < p.lr) v = fmaf(0.5f - 0.5f * cospif((float)(i + 1) / (float)(p.lr + 1)), r - cont, cont);
                else v = r;
            }
            win[c * WL + H + base + i] = v;
            row_ch(y, y_row, y_ch, sr.row, c)[base + i] = v;
        }
        if (t == JB_LOST) run = min(run + P, p.gb);
        else tau = 0, run = 0;
        __syncthreads();
    }
    for (int c = 0; c < C; ++c) {
        for (int i = tid; i < H; i += blockDim.x) st[c * rf + o_hist + i] = win[c * WL + (int64_t)n_out * P + i];
        for (int i = tid; i < p.tmax; i += blockDim.x) st[c * rf + o_per + i] = per[c * p.tmax + i];
    }
    if (tid == 0) {
        st[JB_RUN] = __int_as_float(tau ? run : 0);
        st[JB_TAU] = __int_as_float(tau);
    }
}

template <bool Timed>
__global__ void __launch_bounds__(RS_TILE)
jitter_buffer_kernel_t(const float* __restrict__ x, int64_t x_row, int64_t x_ch, const int32_t* __restrict__ seqs,
                       const int32_t* __restrict__ counts, float* __restrict__ y, int64_t y_row, int64_t y_ch,
                       int32_t* __restrict__ out_counts, int C, const int32_t* __restrict__ slots, float* __restrict__ state,
                       int n_slots, const __grid_constant__ JbParams p, const JbClock ck) {
    jb_row<Timed ? JB_TIMED : JB_UNTIMED>(x, x_row, x_ch, seqs, counts, y, y_row, y_ch, out_counts, C, slots, state,
                                          n_slots, p, ck, JbAdapt{});
}

__global__ void __launch_bounds__(RS_TILE)
jitter_buffer_adaptive_kernel(const float* __restrict__ x, int64_t x_row, int64_t x_ch, const int32_t* __restrict__ seqs,
                              const int32_t* __restrict__ counts, float* __restrict__ y, int64_t y_row, int64_t y_ch,
                              int32_t* __restrict__ out_counts, int C, const int32_t* __restrict__ slots,
                              float* __restrict__ state, int n_slots, const __grid_constant__ JbParams p, const JbClock ck,
                              const __grid_constant__ JbAdapt ad) {
    jb_row<JB_ADAPTIVE>(x, x_row, x_ch, seqs, counts, y, y_row, y_ch, out_counts, C, slots, state, n_slots, p, ck, ad);
}

// the parameters of a jitter buffer and the shared-memory bytes of a call of `arrivals` packets per row (the adaptive
// form's rows end in the statistics block and stage the bins of the arrivals too): 0, or an error code (1 invalid, 2 the
// staging exceeds shared memory) with its message
static int jb_params(const std::string& who, int32_t channels, int32_t rate, int32_t packet, int32_t depth, int32_t window,
                     int32_t max_out, int32_t arrivals, JbParams* p, int* smem, bool adaptive = false) {
    if (channels <= 0) return fail(1, who + ": channels must be positive");
    if (rate < 8000 || rate > 384000) return fail(1, who + ": rate " + std::to_string(rate) + " lies outside [8000, 384000] Hz");
    if (packet < 1) return fail(1, who + ": packet " + std::to_string(packet) + " is not positive");
    if (window < 1 || window > JB_MAX_WINDOW)
        return fail(1, who + ": window " + std::to_string(window) + " lies outside [1, " + std::to_string(JB_MAX_WINDOW) + "]");
    if (depth < 0 || depth >= window)
        return fail(1, who + ": depth " + std::to_string(depth) + " lies outside [0, window - 1 = " + std::to_string(window - 1) + "]");
    if (max_out < 1) return fail(1, who + ": max_out " + std::to_string(max_out) + " is not positive");
    const auto samples = [rate](double s) { return (int32_t)std::floor(s * rate + 0.5); };
    p->P = packet, p->W = window, p->R = 2 * window, p->D = depth, p->M = arrivals, p->max_out = max_out;
    p->tmin = samples(0.0025), p->tmax = samples(0.015), p->wc = samples(0.020);
    p->hist = p->wc + p->tmax;
    p->lr = std::min(samples(0.004), packet);
    p->ga = samples(0.010), p->gb = samples(0.060);
    p->rf = JB_HEAD + p->R + (int64_t)p->R * packet + p->hist + p->tmax + (adaptive ? JB_STATS : 0);
    if ((int64_t)channels * p->rf > INT32_MAX)
        return fail(1, who + ": a slot of " + std::to_string(channels) + " channels, window " + std::to_string(window) +
                           " and packets of " + std::to_string(packet) + " samples is too large");
    const int64_t floats = (int64_t)channels * (p->hist + (int64_t)max_out * packet) + p->hist +
                           (int64_t)channels * p->tmax + p->R + arrivals + max_out + (adaptive ? arrivals : 0);
    return staging(who, floats, std::to_string(channels) + " channels at " + std::to_string(rate) + " Hz with " +
                                    std::to_string(max_out) + " packets of " + std::to_string(packet) +
                                    " samples written per row are too large", "words per row", smem);
}
}  // namespace l2h

extern "C" int l2h_jitter_buffer_layout(int32_t channels, int32_t rate, int32_t packet, int32_t depth, int32_t window,
                                        int32_t max_out, int32_t* row_floats) {
    using namespace l2h;
    if (!row_floats) return fail(1, "l2h_jitter_buffer_layout: null pointer");
    JbParams p;
    if (int rc = jb_params("l2h_jitter_buffer_layout", channels, rate, packet, depth, window, max_out, 1, &p, nullptr))
        return rc;
    *row_floats = (int32_t)p.rf;
    return 0;
}

extern "C" int l2h_jitter_buffer_adaptive_layout(int32_t channels, int32_t rate, int32_t packet, int32_t depth,
                                                 int32_t window, int32_t max_out, int32_t* row_floats) {
    using namespace l2h;
    if (!row_floats) return fail(1, "l2h_jitter_buffer_adaptive_layout: null pointer");
    JbParams p;
    if (int rc = jb_params("l2h_jitter_buffer_adaptive_layout", channels, rate, packet, depth, window, max_out, 1, &p,
                           nullptr, true))
        return rc;
    *row_floats = (int32_t)p.rf;
    return 0;
}

namespace l2h {
constexpr auto jitter_buffer_kernel = jitter_buffer_kernel_t<false>;

// the three entries: the checks of l2h_jitter_buffer, then one launch of the untimed kernel (now_dev null), the timed one
// or, with `ad` (whose lo, hi and late rate r are set), the adaptive one
static int jb_call(const std::string& who, const float* x_dev, int64_t x_row_stride, int64_t x_ch_stride, int32_t max_in,
                   const int32_t* seqs_dev, const int32_t* counts_dev, float* y_dev, int64_t y_row_stride,
                   int64_t y_ch_stride, int32_t* out_counts_dev, int32_t n, int32_t channels, const int32_t* slots_dev,
                   float* state_dev, int32_t n_slots, int32_t rate, int32_t packet, int32_t depth, int32_t window,
                   int32_t max_out, const int32_t* now_dev, int32_t deadline_us, void* stream, JbAdapt* ad = nullptr) {
    if (int rc = slot_call(who, {x_dev, seqs_dev, counts_dev, y_dev, out_counts_dev, slots_dev, state_dev},
                           "n, channels, max_in and n_slots", {n, channels, max_in, n_slots}, n, channels, n_slots))
        return rc;
    JbParams p;
    int smem;
    if (int rc = jb_params(who, channels, rate, packet, depth, window, max_out, max_in, &p, &smem, ad != nullptr))
        return rc;
    const Rows x{"x", x_row_stride, x_ch_stride, (int64_t)max_in * packet},
        y{"y", y_row_stride, y_ch_stride, (int64_t)max_out * packet};
    if (x.len > INT32_MAX) return fail(1, who + ": max_in * packet is too large");
    if (int rc = disjoint(who, channels, {x, y})) return rc;
    if (overlap(y_dev, n, y, x_dev, n, x, channels, false)) return fail(1, who + ": y must not overlap x");
    JbClock ck{now_dev, deadline_us, 0, 0};
    if (now_dev) {
        // period = round(1e6 packet / rate) µs, exactly, taken mod 2^32 as the clock is; S = ceil(gb / packet)
        ck.period = (uint32_t)((2000000 * (int64_t)packet + rate) / (2 * (int64_t)rate));
        ck.stall = (p.gb + packet - 1) / packet;
    }
    if (ad) {
        // w = max(1, ceil(hi / 64)); N = max(1, round(5e6 / period)) with the period before it is taken mod 2^32
        const int64_t period = (2000000 * (int64_t)packet + rate) / (2 * (int64_t)rate);
        ad->w = (int32_t)std::max<int64_t>(1, ((int64_t)ad->hi + JB_BINS - 1) / JB_BINS);
        ad->mem = (int32_t)std::max<int64_t>(1, (10000000 + period) / (2 * period));
        if (smem > RS_SMEM_BYTES - 4096)
            if (cudaError_t e = full_staging(jitter_buffer_adaptive_kernel))
                return fail(3, who + ": " + cudaGetErrorString(e));
        jitter_buffer_adaptive_kernel<<<(unsigned)n, RS_TILE, smem, static_cast<cudaStream_t>(stream)>>>(
            x_dev, x_row_stride, x_ch_stride, seqs_dev, counts_dev, y_dev, y_row_stride, y_ch_stride, out_counts_dev,
            channels, slots_dev, state_dev, n_slots, p, ck, *ad);
        return launched(who);
    }
    const auto kernel = now_dev ? jitter_buffer_kernel_t<true> : jitter_buffer_kernel;
    if (smem > RS_SMEM_BYTES - 4096)                                    // then the static words need the opt-in
        if (cudaError_t e = full_staging(kernel)) return fail(3, who + ": " + cudaGetErrorString(e));
    kernel<<<(unsigned)n, RS_TILE, smem, static_cast<cudaStream_t>(stream)>>>(
        x_dev, x_row_stride, x_ch_stride, seqs_dev, counts_dev, y_dev, y_row_stride, y_ch_stride, out_counts_dev, channels,
        slots_dev, state_dev, n_slots, p, ck);
    return launched(who);
}
}  // namespace l2h

extern "C" int l2h_jitter_buffer(const float* x_dev, int64_t x_row_stride, int64_t x_ch_stride, int32_t max_in,
                                 const int32_t* seqs_dev, const int32_t* counts_dev, float* y_dev, int64_t y_row_stride,
                                 int64_t y_ch_stride, int32_t* out_counts_dev, int32_t n, int32_t channels,
                                 const int32_t* slots_dev, float* state_dev, int32_t n_slots, int32_t rate, int32_t packet,
                                 int32_t depth, int32_t window, int32_t max_out, void* stream) {
    return l2h::jb_call("l2h_jitter_buffer", x_dev, x_row_stride, x_ch_stride, max_in, seqs_dev, counts_dev, y_dev,
                        y_row_stride, y_ch_stride, out_counts_dev, n, channels, slots_dev, state_dev, n_slots, rate, packet,
                        depth, window, max_out, nullptr, 0, stream);
}

extern "C" int l2h_jitter_buffer_timed(const float* x_dev, int64_t x_row_stride, int64_t x_ch_stride, int32_t max_in,
                                       const int32_t* seqs_dev, const int32_t* counts_dev, float* y_dev,
                                       int64_t y_row_stride, int64_t y_ch_stride, int32_t* out_counts_dev, int32_t n,
                                       int32_t channels, const int32_t* slots_dev, float* state_dev, int32_t n_slots,
                                       int32_t rate, int32_t packet, int32_t depth, int32_t window, int32_t max_out,
                                       const int32_t* now_dev, int32_t deadline_us, void* stream) {
    using namespace l2h;
    const std::string who = "l2h_jitter_buffer_timed";
    if (!now_dev) return fail(1, who + ": null pointers");
    if (deadline_us < 0) return fail(1, who + ": deadline_us " + std::to_string(deadline_us) + " is negative");
    return jb_call(who, x_dev, x_row_stride, x_ch_stride, max_in, seqs_dev, counts_dev, y_dev, y_row_stride, y_ch_stride,
                   out_counts_dev, n, channels, slots_dev, state_dev, n_slots, rate, packet, depth, window, max_out,
                   now_dev, deadline_us, stream);
}

extern "C" int l2h_jitter_buffer_adaptive(const float* x_dev, int64_t x_row_stride, int64_t x_ch_stride, int32_t max_in,
                                          const int32_t* seqs_dev, const int32_t* counts_dev, float* y_dev,
                                          int64_t y_row_stride, int64_t y_ch_stride, int32_t* out_counts_dev, int32_t n,
                                          int32_t channels, const int32_t* slots_dev, float* state_dev, int32_t n_slots,
                                          int32_t rate, int32_t packet, int32_t depth, int32_t window, int32_t max_out,
                                          const int32_t* now_dev, const int32_t* arrivals_dev, int32_t lo_us,
                                          int32_t hi_us, double late_rate, void* stream) {
    using namespace l2h;
    const std::string who = "l2h_jitter_buffer_adaptive";
    if (!now_dev) return fail(1, who + ": null pointers");
    if (lo_us < 0 || hi_us < lo_us)
        return fail(1, who + ": lo_us " + std::to_string(lo_us) + " and hi_us " + std::to_string(hi_us) +
                           " do not satisfy 0 <= lo_us <= hi_us");
    if (!(late_rate > 0.0 && late_rate <= 0.5))
        return fail(1, who + ": late_rate " + std::to_string(late_rate) + " lies outside (0, 0.5]");
    // r = round(late_rate 2^16); the warm-up ceil(1 / late_rate), at most 2^31 - 1
    JbAdapt ad{arrivals_dev, lo_us, hi_us, 0, (int32_t)std::floor(late_rate * 65536.0 + 0.5),
               (int32_t)std::min(std::ceil(1.0 / late_rate), (double)INT32_MAX), 0};
    return jb_call(who, x_dev, x_row_stride, x_ch_stride, max_in, seqs_dev, counts_dev, y_dev, y_row_stride, y_ch_stride,
                   out_counts_dev, n, channels, slots_dev, state_dev, n_slots, rate, packet, depth, window, max_out,
                   now_dev, 0, stream, &ad);
}
