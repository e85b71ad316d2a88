// Separation-network kernels that are not plain row-GEMMs / LSTM recurrences.
// Reference: reference src/models/tfgridnet_realtime/tfgridnet_causal.py (cited per kernel).
// Activations are [B, T, F=97, C=64] fp32 rows of 256 B.
#pragma once
#include <cooperative_groups.h>

#include "common.cuh"
#include "sep_layout.h"

namespace l2h {

struct SepWeights {           // device pointers into the packed weight buffer
    const float* wat;         // [192][196]   analysis filters, transposed (n, r)
    const float* ws;          // [194][192]   synthesis filters (r, n)
    const float* wc;          // [64][36]     conv (o, c*9+i*3+j)
    const float* bc;          // [64]
    const float* we;          // [6208][256]  speaker projection
    const float* be;          // [6208]
    const float* lne_g;       // [6208]
    const float* lne_b;
    const float* wd;          // [64][4][9]   deconv (c, o, i*3+j)
    const float* bd;          // [4]
    int gen;                  // weight generation (bumped by every commit): part of the speaker-gate memo key
};

struct BlockWeights {
    const float *ln1_g, *ln1_b;       // [64]
    const float* wih1_t;              // [64][512]   (k, dir*256 + j*4+q)
    const float* b1;                  // [512]       b_ih + b_hh, same packing
    const float* whh1;                // [2][256][64]
    const float* wl1_t;               // [128][64]
    const float* bl1;                 // [64]
    const float *ln2_g, *ln2_b;
    const float* wih2_t;              // [64][256]
    const float* b2;                  // [256]
    const float* whh2;                // [256][64]   (row = gate column j*4+q)
    const float* whh2_t;              // [64][256]   the same matrix k-major (source of mid_pack)
    const float* mid_pack;            // [MID_PACK]  k-sliced copies of wl1_t, [wih2_t ; whh2_t], wl2_t, wqkv_t (mid_kernel.cuh)
    const float* wl2_t;               // [64][64]
    const float* bl2;
    const float* wqkv_t;              // [64][112]   cols: Q(h*6+e) | K(h*6+e) | V(h*16+c)
    const float* bqkv;                // [112]
    const float* slopes;              // [4]  PReLU of Q, K, V, proj
    const float* slope_vec;           // [112] the Q/K/V slopes per projection column (epilogue of the tensor-core QKV GEMM)
    const float *lnq_g, *lnq_b;       // [582]
    const float *lnk_g, *lnk_b;       // [582]
    const float *lnv_g, *lnv_b;       // [1552]
    const float* wp_t;                // [64][64]
    const float* bp;                  // [64]
    const float *lnp_g, *lnp_b;       // [6208]
};

// ------------------------------------------------------------------------------------------
// state init: zero everything, poison the cached embedding with NaN (forces the first gate build)
__global__ void state_init_kernel(float* state, int64_t total_floats, int64_t stride, int B) {
    const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t hdr = sizeof(StateHeader) / 4;
    for (int64_t i = i0; i < total_floats; i += (int64_t)gridDim.x * blockDim.x) {
        float v = 0.f;
        if (i >= hdr) {
            const int64_t o = (i - hdr) % stride;
            if (o < SPK) v = __int_as_float(0x7fc00000);
        }
        state[i] = v;
    }
}

// ---- call rows -> stream records, per-stream clocks (sep_layout.h) and the rows that store -------------------------
// Where the records of a slot-list call's rows live (l2h_sep_forward_slots): row b is record slots[b] of a state of
// `batch` records.  Dense calls pass the record stride instead (row b is record b).  The kernels that address records
// are templates over the two (`Map`): the dense forms compile to the arithmetic they had before slot lists existed.
struct Records {
    int64_t stride;            // floats per record
    const int32_t* slots;      // device, one entry per call row
    int32_t batch;             // records in the state
    const int32_t* hops;       // device, frames each row advances (l2h_sep_forward_slots_hops), or null: every row all of them
    int32_t frames;            // frames of the call (T)
};

// How many of a call's T frames row b advances: all of them for dense rows and plain slot lists; hops[b] for a ragged
// slot list, where an entry outside [0, T] counts as 0.  A ragged row computes all T frames (its first T_b are exactly
// those of a T_b-frame call: every stage is causal in time) but stores only what its T_b frames leave.
__device__ __forceinline__ int row_frames(int64_t, int, int T) { return T; }
__device__ __forceinline__ int row_frames(const Records& r, int b, int T) {
    if (r.hops == nullptr) return T;
    const int h = __ldg(r.hops + b);
    return (unsigned)h <= (unsigned)T ? h : 0;
}
// ... whether frame t (< T) is one of them, given T_b = row_frames(): always for a dense row
__device__ __forceinline__ bool row_has_frame(int64_t, int, int) { return true; }
__device__ __forceinline__ bool row_has_frame(const Records&, int t, int Tb) { return t < Tb; }
// ... and the samples of row b's x (extra = LOOKAHEAD) or y (extra = 0) those frames read or write: `len` for a dense row
__device__ __forceinline__ int row_len(int64_t, int, int, int len, int) { return len; }
__device__ __forceinline__ int row_len(const Records& r, int b, int T, int len, int extra) {
    return r.hops == nullptr ? len : min(len, HOP * row_frames(r, b, T) + extra);
}

// The one decision of which record call row b reads and writes, and whether the row stores anything (its record and its
// y row).  Dense rows store unless the activity mask of l2h_sep_forward_active clears them.  A slot-list entry outside
// [0, batch) marks a row that is computed from record 0 (so every read stays inside the state) and stores nothing, and so
// does a ragged row that advances no frame.
struct RowRecord { int64_t off; bool stores; };
__device__ __forceinline__ RowRecord row_record(int64_t stride, const uint8_t* active, int b) {
    return {(int64_t)(sizeof(StateHeader) / 4) + (int64_t)b * stride, active == nullptr || active[b] != 0};
}
__device__ __forceinline__ RowRecord row_record(const Records& r, const uint8_t*, int b) {
    const int s = __ldg(r.slots + b);
    const bool in = (unsigned)s < (unsigned)r.batch;
    return {(int64_t)(sizeof(StateHeader) / 4) + (int64_t)(in ? s : 0) * r.stride, in && row_frames(r, b, r.frames) > 0};
}
template <class Map> __device__ __forceinline__ float* stream_rec(float* state, const Map& r, int b) {
    return state + row_record(r, nullptr, b).off;
}
template <class Map> __device__ __forceinline__ const float* stream_rec(const float* state, const Map& r, int b) {
    return state + row_record(r, nullptr, b).off;
}
template <class Map> __device__ __forceinline__ bool stream_active(const Map& r, const uint8_t* active, int b) {
    return row_record(r, active, b).stores;
}
__device__ __forceinline__ long long rec_pos(const float* rec) { return *reinterpret_cast<const long long*>(rec + ST_POS); }
__device__ __forceinline__ int rec_par(const float* rec) { return __float_as_int(rec[ST_CALLS]) & 1; }

// End of a call, run by every thread of ONE CTA after all others have finished reading the clocks: the header advances by
// `frames` frames and one call, and the clock of every row that stores by one call and the frames it advances.
template <class Map>
__device__ void advance_clocks(float* state, Map recs, int n_streams, int frames, const uint8_t* active) {
    if (threadIdx.x == 0) {
        StateHeader* hdr = reinterpret_cast<StateHeader*>(state);
        hdr->pos += frames;
        hdr->ncalls += 1;
        hdr->done = 0;
    }
    for (int b = threadIdx.x; b < n_streams; b += blockDim.x) {
        if (!stream_active(recs, active, b)) continue;
        float* rec = stream_rec(state, recs, b);
        *reinterpret_cast<long long*>(rec + ST_POS) += row_frames(recs, b, frames);
        rec[ST_CALLS] = __int_as_float(__float_as_int(rec[ST_CALLS]) + 1);
    }
    __threadfence();
}

// The last CTA of a call's final kernel advances the clocks (advance_clocks).
template <class Map>
__device__ __forceinline__ void finish_call(float* state, Map recs, int n_streams, int frames, const uint8_t* active) {
    __shared__ int last;
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const int prev = atomicAdd(&reinterpret_cast<StateHeader*>(state)->done, 1);
        last = prev == (int)(gridDim.x * gridDim.y) - 1;
    }
    __syncthreads();
    if (last) advance_clocks(state, recs, n_streams, frames, active);
}

__global__ void advance_header_kernel(float* state, int64_t sstride, int n_streams, int frames) {
    advance_clocks(state, sstride, n_streams, frames, nullptr);
}

// l2h_sep_state_reset_streams: the listed records become fresh streams, as state_init_kernel leaves them (zero rings,
// h / c and tails, clock 0, NaN embedding = gate memo invalid).  grid (any, n), record of slots.s[blockIdx.y].
constexpr int RESET_MAX_SLOTS = 960;      // slots per launch: the kernel parameters stay under 4 KB
struct SlotList { int32_t s[RESET_MAX_SLOTS]; };
__global__ void reset_streams_kernel(float* state, int64_t sstride, SlotList slots) {
    float4* rec = reinterpret_cast<float4*>(stream_rec(state, sstride, slots.s[blockIdx.y]));
    const float nan = __int_as_float(0x7fc00000);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < sstride / 4; i += (int64_t)gridDim.x * blockDim.x)
        rec[i] = (i < SPK / 4) ? make_float4(nan, nan, nan, nan) : make_float4(0.f, 0.f, 0.f, 0.f);
}

__global__ void set_clip_base_kernel(float* state) {
    StateHeader* hdr = reinterpret_cast<StateHeader*>(state);
    hdr->clip_base = hdr->pos;
}

// ------------------------------------------------------------------------------------------
// K1 front: STFT analysis + channel regroup + causal 3x3 conv   (tfgridnet_causal.py:229-242)
// grid (T, B), 256 threads.  x: [B][NMIC][x_len] (samples past x_len read as zero: the mod-pad and
// look-ahead zeros of net.py:8-18,56-58).  Frames before the call start come from conv_buf.
constexpr size_t FRONT_SMEM = (size_t)NFFT * 196 * sizeof(float);     // analysis filters, staged by TMA

template <class Map>
__device__ void spk_gate_cta(const float* __restrict__ emb, float* __restrict__ pre, float* __restrict__ state,
                             Map recs, const SepWeights& w, int b, float* red, const uint8_t* __restrict__ active);

template <class Map>
__global__ void __launch_bounds__(256)
front_kernel_t(const float* __restrict__ x, int64_t x_bstride, int64_t x_cstride, int x_len,
               float* __restrict__ X, float* __restrict__ state, Map recs, SepWeights w, int T,
               int pos_rel, const float* __restrict__ emb, float* __restrict__ spk_pre, int frame_k, int frames_total,
               int sample_off, const uint8_t* __restrict__ active) {
    extern __shared__ __align__(16) float wat_s[];     // [192][196]
    __shared__ __align__(16) float xs[NMIC][448];
    __shared__ float U[3][4][100];      // [frame t-2..t][ch][1 + f], zero-padded in f
    __shared__ __align__(8) unsigned long long wbar;
    TraceScope trace_(TK_FRONT, X);
    griddep_launch();
    const int t = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    if (t == T) {                      // the extra CTA of this stream: speaker-gate memo
        griddep_wait();
        spk_gate_cta(emb, spk_pre, state, recs, w, b, &xs[0][0], active);
        return;
    }
    if (tid == 0) { mbar_init(&wbar, 1); mbar_fence_init(); }
    __syncthreads();
    if (tid == 0) mbar_expect_tx(&wbar, (unsigned)FRONT_SMEM);
    __syncthreads();
    tma_load_split(wat_s, w.wat, (unsigned)FRONT_SMEM, &wbar, tid, 256);     // 74 bulk copies in flight
    griddep_wait();
    // A "group" is what advances the clocks once: the T frames of an ordinary call, or the
    // frames_total one-frame calls of a pipelined graph (frame_k = index inside it).  gi = frame index in
    // the group.  All frames of a group read the tails the stream's PREVIOUS group left (parity of its call
    // count) and recompute what they need of their predecessors inside the group; only the group's last frame
    // writes the new tails (other parity) -- so the frames of a group never depend on each other here.
    const StateHeader* hdr = reinterpret_cast<const StateHeader*>(state);
    const int gi = frame_k + t, GN = row_frames(recs, b, (frames_total > 1) ? frames_total : T);
    float* st = stream_rec(state, recs, b);
    const int par = rec_par(st);
    const float* cb = st + ST_CONV + par * (2 * 4 * NF);
    float* cb_next = st + ST_CONV + (par ^ 1) * (2 * 4 * NF);

    for (int i = tid; i < 3 * 4 * 100; i += 256) (&U[0][0][0])[i] = 0.f;
    // pos_rel: x is a whole clip and this call starts at frame (pos - clip_base) of it
    const int s0 = HOP * (t - 2) + sample_off + (pos_rel ? (int)(hdr->pos - hdr->clip_base) * HOP : 0);
    const int xl = row_len(recs, b, T, x_len, LOOKAHEAD);
    for (int i = tid; i < NMIC * 448; i += 256) {
        const int m = i / 448, n = i % 448, s = s0 + n;
        xs[m][n] = (s >= 0 && s < xl) ? x[(int64_t)b * x_bstride + (int64_t)m * x_cstride + s] : 0.f;
    }
    __syncthreads();
    trace_.mark(0);
    // history frames from conv_buf: frame -2 -> slot 0, frame -1 -> slot 1
    for (int i = 0; i < 2; ++i) {
        const int g = gi - 2 + i;               // frame index in the group; < 0: before the group -> conv_buf
        if (g < 0)
            for (int e = tid; e < 4 * NF; e += 256) U[i][e / NF][1 + e % NF] = cb[(2 + g) * 4 * NF + e];
    }
    if (tid < NROW) {
        float acc[3][NMIC];
#pragma unroll
        for (int i = 0; i < 3; ++i) { acc[i][0] = 0.f; acc[i][1] = 0.f; }
        mbar_wait(&wbar, 0);
        trace_.mark(1);
#pragma unroll 8
        for (int n = 0; n < NFFT; ++n) {
            const float wv = wat_s[n * 196 + tid];
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                acc[i][0] = fmaf(wv, xs[0][HOP * i + n], acc[i][0]);
                acc[i][1] = fmaf(wv, xs[1][HOP * i + n], acc[i][1]);
            }
        }
        const int ri = tid / NF, f = tid % NF;      // rows 0..96 real, 97..193 imaginary
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            if (gi - 2 + i >= 0) {                  // channels: [Re m0, Re m1, Im m0, Im m1]
                U[i][ri * 2 + 0][1 + f] = acc[i][0];
                U[i][ri * 2 + 1][1 + f] = acc[i][1];
            }
        }
    }
    __syncthreads();
    trace_.mark(2);
    // conv: X[f][o] = b_o + sum_{c,i,j} Wc[o][c][i][j] * U[i][c][f-1+j]
    {
        const int o = tid & 63, fg = tid >> 6;
        float wr[36];
#pragma unroll
        for (int k = 0; k < 36; ++k) wr[k] = __ldg(w.wc + o * 36 + k);
        const float bias = __ldg(w.bc + o);
        // four rows at a time: four independent 36-long FMA chains per thread instead of one (a single chain makes the
        // conv the longest part of the frame); per output the same order of additions as before
        for (int f = fg; f < NF; f += 16) {
            float acc[4] = {bias, bias, bias, bias};
#pragma unroll
            for (int c = 0; c < 4; ++c)
#pragma unroll
                for (int i = 0; i < 3; ++i)
#pragma unroll
                    for (int j = 0; j < 3; ++j) {
                        const float wv = wr[c * 9 + i * 3 + j];
#pragma unroll
                        for (int u = 0; u < 4; ++u) acc[u] = fmaf(wv, U[i][c][min(f + 4 * u, NF - 1) + j], acc[u]);
                    }
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (f + 4 * u < NF) X[(((int64_t)b * T + t) * NF + f + 4 * u) * CH + o] = acc[u];
        }
    }
    trace_.mark(3);
    // next conv_buf = spectrogram rows of the last two frames of the group (a ragged row's own last two), written by its
    // last frame
    if (gi == GN - 1 && stream_active(recs, active, b)) {
        for (int e = tid; e < 4 * NF; e += 256) {
            cb_next[e] = U[1][e / NF][1 + e % NF];
            cb_next[4 * NF + e] = U[2][e / NF][1 + e % NF];
        }
    }
}

// K1 for calls of MANY frames: front_kernel's arithmetic frame by frame in the same order (bit-identical), but one CTA walks a
// contiguous chunk of a stream's frames: the 150 KB of analysis filters are staged once per CTA instead of once per frame,
// only the NEW frame's spectrum is computed (the two before it stay in a 3-slot ring; front_kernel recomputes them: 3x the STFT),
// and the next frame's samples are fetched while the current frame is worked on.  grid (n_chunks + 1, B): the last CTA of a
// stream is the speaker-gate memo.  Frames [c*chunk, min(T, (c+1)*chunk)) for CTA c.
template <class Map>
__global__ void __launch_bounds__(256)
front_many_kernel_t(const float* __restrict__ x, int64_t x_bstride, int64_t x_cstride, int x_len, float* __restrict__ X,
                    float* __restrict__ state, Map recs, SepWeights w, int T, int pos_rel, const float* __restrict__ emb,
                    float* __restrict__ spk_pre, int chunk, int n_chunks, int n_streams, int n_workers,
                    const uint8_t* __restrict__ active) {
    extern __shared__ __align__(16) float wat_s[];     // [192][196]
    __shared__ __align__(16) float xs[NMIC][NFFT];      // the samples of the frame being transformed (>= 288 floats: gate CTA scratch)
    __shared__ float U[3][4][100];      // ring: frame g -> slot (g + 3) % 3; [ch][1 + f], zero-padded in f
    __shared__ __align__(8) unsigned long long wbar;
    griddep_launch();
    const int tid = threadIdx.x;
    if ((int)blockIdx.x >= n_workers) {        // one more CTA per stream: speaker-gate memo
        griddep_wait();
        spk_gate_cta(emb, spk_pre, state, recs, w, (int)blockIdx.x - n_workers, &xs[0][0], active);
        return;
    }
    if (tid == 0) { mbar_init(&wbar, 1); mbar_fence_init(); }
    __syncthreads();
    if (tid == 0) { mbar_expect_tx(&wbar, (unsigned)FRONT_SMEM); tma_load_1d(wat_s, w.wat, (unsigned)FRONT_SMEM, &wbar); }
    for (int i = tid; i < 3 * 4 * 100; i += 256) (&U[0][0][0])[i] = 0.f;
    const int o = tid & 63, fg = tid >> 6;
    float wr[36];
#pragma unroll
    for (int k = 0; k < 36; ++k) wr[k] = __ldg(w.wc + o * 36 + k);
    const float bias = __ldg(w.bc + o);
    griddep_wait();
    const StateHeader* hdr = reinterpret_cast<const StateHeader*>(state);
    const int sbase = pos_rel ? (int)(hdr->pos - hdr->clip_base) * HOP : 0;
    mbar_wait(&wbar, 0);
    // one CTA walks (stream, chunk) items: frames [c*chunk, min(T, (c+1)*chunk)) of stream b
    for (int item = blockIdx.x; item < n_streams * n_chunks; item += n_workers) {
    const int b = item / n_chunks, c = item % n_chunks;
    const int t0 = c * chunk, t1 = min(T, t0 + chunk);
    float* st = stream_rec(state, recs, b);
    const int par = rec_par(st);
    const bool live = stream_active(recs, active, b);
    const int Tb = row_frames(recs, b, T), xl = row_len(recs, b, T, x_len, LOOKAHEAD);
    const float* cb = st + ST_CONV + par * (2 * 4 * NF);
    float* cb_next = st + ST_CONV + (par ^ 1) * (2 * 4 * NF);
    const float* xb = x + (int64_t)b * x_bstride;
    // samples of frame g: x[sbase + 128 g .. + 191] (zero outside the clip); thread tid fetches entries tid and tid + 256 of [2][192]
    auto fetch = [&](int g, float& a0, float& a1) {
        const int s0 = sbase + HOP * g;
        { const int m = tid / NFFT, n = tid % NFFT, sidx = s0 + n; a0 = (sidx >= 0 && sidx < xl) ? xb[(int64_t)m * x_cstride + sidx] : 0.f; }
        a1 = 0.f;
        if (tid + 256 < NMIC * NFFT) { const int i = tid + 256, m = i / NFFT, n = i % NFFT, sidx = s0 + n; a1 = (sidx >= 0 && sidx < xl) ? xb[(int64_t)m * x_cstride + sidx] : 0.f; }
    };
    auto put = [&](float a0, float a1) {
        (&xs[0][0])[tid] = a0;
        if (tid + 256 < NMIC * NFFT) (&xs[0][0])[tid + 256] = a1;
    };
    // spectrum of the frame whose samples are in xs -> ring slot of frame g: channels [Re m0, Re m1, Im m0, Im m1]
    auto stft = [&](int g) {
        if (tid < NROW) {
            float a0 = 0.f, a1 = 0.f;
#pragma unroll 8
            for (int n = 0; n < NFFT; ++n) {
                const float wv = wat_s[n * 196 + tid];
                a0 = fmaf(wv, xs[0][n], a0);
                a1 = fmaf(wv, xs[1][n], a1);
            }
            const int ri = tid / NF, f = tid % NF, slot = (g + 3) % 3;
            U[slot][ri * 2 + 0][1 + f] = a0;
            U[slot][ri * 2 + 1][1 + f] = a1;
        }
    };
    float n0, n1;
    // the two frames before the chunk: from the tails of the previous call (g < 0) or recomputed
    for (int g = t0 - 2; g < t0; ++g) {
        __syncthreads();
        if (g < 0) {
            for (int e = tid; e < 4 * NF; e += 256) U[(g + 3) % 3][e / NF][1 + e % NF] = cb[(2 + g) * 4 * NF + e];
        } else {
            fetch(g, n0, n1);
            put(n0, n1);
            __syncthreads();
            stft(g);
        }
    }
    __syncthreads();
    fetch(t0, n0, n1);
    for (int t = t0; t < t1; ++t) {
        put(n0, n1);
        __syncthreads();                           // samples of frame t visible; frame t-1's conv (reads all three slots) is done
        if (t + 1 < t1) fetch(t + 1, n0, n1);      // next frame's samples in flight under this frame's work
        stft(t);
        __syncthreads();
        // conv: X[f][o] = b_o + sum_{c,i,j} Wc[o][c][i][j] * U[frame t-2+i][c][f-1+j]
        {
            const float (*U0)[100] = U[(t - 2 + 3) % 3];
            const float (*U1)[100] = U[(t - 1 + 3) % 3];
            const float (*U2)[100] = U[(t + 3) % 3];
            for (int f = fg; f < NF; f += 16) {
                float acc[4] = {bias, bias, bias, bias};
#pragma unroll
                for (int cc = 0; cc < 4; ++cc)
#pragma unroll
                    for (int i = 0; i < 3; ++i) {
                        const float* ur = (i == 0) ? U0[cc] : (i == 1 ? U1[cc] : U2[cc]);
#pragma unroll
                        for (int j = 0; j < 3; ++j) {
                            const float wv = wr[cc * 9 + i * 3 + j];
#pragma unroll
                            for (int u = 0; u < 4; ++u) acc[u] = fmaf(wv, ur[min(f + 4 * u, NF - 1) + j], acc[u]);
                        }
                    }
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (f + 4 * u < NF) X[(((int64_t)b * T + t) * NF + f + 4 * u) * CH + o] = acc[u];
            }
        }
        if (t == Tb - 1 && live) {                 // next conv tails = spectrogram rows of the row's last two frames
            for (int e = tid; e < 4 * NF; e += 256) {
                cb_next[e] = U[(t - 1 + 3) % 3][e / NF][1 + e % NF];
                cb_next[4 * NF + e] = U[(t + 3) % 3][e / NF][1 + e % NF];
            }
        }
    }
    __syncthreads();                               // the item's last conv is done before the next item refills the ring
    }
}

// ------------------------------------------------------------------------------------------
// K6 speaker gate: g = LN_6208(W e + b), stored (f, c)   (tfgridnet_causal.py:247-248).
// The reference recomputes it on every call; it only changes when the embedding does, so it is
// memoised ON THE DEVICE: one extra CTA per stream rides along with front_kernel, compares the
// embedding with the one the cached gate was built from and returns at once if they are equal
// (the streaming steady state).  Otherwise that CTA rebuilds the gate (6208x256 GEMV + LayerNorm).
template <class Map>
__device__ void spk_gate_cta(const float* __restrict__ emb, float* __restrict__ pre, float* __restrict__ state,
                             Map recs, const SepWeights& w, int b, float* red /* >= 288 floats smem */,
                             const uint8_t* __restrict__ active) {
    if (!stream_active(recs, active, b)) return;     // a stream that skips this hop keeps its record as it is, memo included
    const int tid = threadIdx.x;
    float* st = stream_rec(state, recs, b);
    const float e = emb[(int64_t)b * SPK + tid];
    // memo key: the embedding AND the weight generation (a reused state must not keep a gate built from old weights)
    const int same = __syncthreads_and(e == st[ST_EMB + tid] && __float_as_int(st[ST_GEN]) == w.gen);
    if (same) return;
    float* es = red + 32;                      // [256] embedding
    es[tid] = e;
    __syncthreads();
    const int warp = tid >> 5, lane = tid & 31;
    const float4 e0 = *reinterpret_cast<const float4*>(es + lane * 4);
    const float4 e1 = *reinterpret_cast<const float4*>(es + 128 + lane * 4);
    float* p = pre + (int64_t)b * FC;
    for (int n0 = warp * 4; n0 < FC; n0 += 32) {          // 4 rows per warp per pass: 8 loads in flight per lane
        float4 a0[4], a1[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const float4* wr = reinterpret_cast<const float4*>(w.we + (int64_t)(n0 + r) * SPK);
            a0[r] = __ldg(wr + lane);
            a1[r] = __ldg(wr + 32 + lane);
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            float s = a0[r].x * e0.x + a0[r].y * e0.y + a0[r].z * e0.z + a0[r].w * e0.w +
                      a1[r].x * e1.x + a1[r].y * e1.y + a1[r].z * e1.z + a1[r].w * e1.w;
            s = warp_sum(s);
            if (lane == 0) p[n0 + r] = s + __ldg(w.be + n0 + r);
        }
    }
    __syncthreads();
    float s = 0.f;
    for (int i = tid; i < FC; i += 256) s += p[i];
    const float mu = block_sum(s, red) * (1.f / FC);
    float q = 0.f;
    for (int i = tid; i < FC; i += 256) { const float d = p[i] - mu; q += d * d; }
    const float rs = rsqrtf(block_sum(q, red) * (1.f / FC) + 1e-5f);
    for (int i = tid; i < FC; i += 256) {          // i = c*97 + f  ->  gate[f][c]
        const int c = i / NF, f = i % NF;
        st[ST_GATE + f * CH + c] = (p[i] - mu) * rs * __ldg(w.lne_g + i) + __ldg(w.lne_b + i);
    }
    st[ST_EMB + tid] = e;
    if (tid == 0) st[ST_GEN] = __int_as_float(w.gen);
}

// ------------------------------------------------------------------------------------------
// K/V history -> linear scratch for multi-frame calls.  Kall[b*4+h][0..48] = ring slots of frames
// pos-49 .. pos-1 of stream b's clock (frames before its start are zero = the reference's zero-initialised K_buf/V_buf).
template <class Map>
__global__ void kv_gather_kernel_t(const float* __restrict__ state, Map recs, int blk,
                                   float* __restrict__ Kall, float* __restrict__ Vall, int T) {
    griddep_launch();
    griddep_wait();
    const int i = blockIdx.x, bh = blockIdx.y, b = bh / NHEAD, h = bh % NHEAD;
    const float* rec = stream_rec(state, recs, b);
    const long long fr = rec_pos(rec) - (ATT - 1) + i;
    const int slot = (int)(((fr % RING) + RING) % RING);
    const float* sb = rec + ST_BLK + (int64_t)blk * BK_STRIDE;
    const float4* ks = reinterpret_cast<const float4*>(sb + BK_K + ((int64_t)h * RING + slot) * QK_LD);
    const float4* vs = reinterpret_cast<const float4*>(sb + BK_V + ((int64_t)h * RING + slot) * V_DIM);
    float4* kd = reinterpret_cast<float4*>(Kall + ((int64_t)bh * (ATT - 1 + T) + i) * QK_LD);
    float4* vd = reinterpret_cast<float4*>(Vall + ((int64_t)bh * (ATT - 1 + T) + i) * V_DIM);
    const bool live = fr >= 0;
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int k = threadIdx.x; k < QK_LD / 4; k += blockDim.x) kd[k] = live ? ks[k] : z;
    for (int k = threadIdx.x; k < V_DIM / 4; k += blockDim.x) vd[k] = live ? vs[k] : z;
}

// ------------------------------------------------------------------------------------------
// K4a qkv: Linear(64 -> 24|24|64) + PReLU + head split + LayerNorm over (F, E) per head, then
// append to the K/V history   (tfgridnet_causal.py:547-562, modules :354-387).
// grid (T, B), 384 threads (12 warps = {Q,K,V} x 4 heads for the LayerNorm phase).
constexpr int QKV_THREADS = 384;
constexpr int QKV_PLD = NQKV;                 // 112: a frame's projections are one contiguous 43 KB tile
constexpr int QKV_LNP = 4 * QK_LD + 2 * V_DIM;  // staged LayerNorm params: gq | bq | gk | bk | gv | bv
constexpr size_t QKV_SMEM = (size_t)(64 * 100 + 64 * NQKV + NF * QKV_PLD + QKV_LNP) * sizeof(float);
// with the projections given (`pre`), X and W_qkv are not staged: launches that pass `pre` need only this much, which lets
// two such CTAs, or one and a BiLSTM, share an SM
constexpr size_t QKV_PRE_SMEM = (size_t)(NF * QKV_PLD + QKV_LNP) * sizeof(float);

template <class Map>
__global__ void __launch_bounds__(QKV_THREADS)
qkv_kernel_t(const float* __restrict__ X, const float* __restrict__ pre, float* __restrict__ Qbuf,
             float* __restrict__ Kall, float* __restrict__ Vall, float* __restrict__ state, Map recs, int blk,
             BlockWeights w, int T, int frame_k, const uint8_t* __restrict__ active) {
    extern __shared__ __align__(16) float sm[];
    float* Xt = sm;                      // [64][100]  k-major, rows padded to 100 (zeros); not staged when pre != nullptr
    float* Ws = Xt + 64 * 100;           // [64][112]
    float* P = pre != nullptr ? sm : Ws + 64 * NQKV;     // [97][112]
    float* LNP = P + NF * QKV_PLD;       // gq[584] bq[584] gk[584] bk[584] gv[1552] bv[1552]
    __shared__ __align__(8) unsigned long long bars[2];
    const int t = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    TraceScope trace_(TK_QKV, X);
    griddep_launch();
    if (tid == 0) { mbar_init(&bars[0], 1); mbar_init(&bars[1], 1); mbar_fence_init(); }
    __syncthreads();
    // parameters: independent of the chain -> before the wait
    // (the 582-float vectors are followed by 2 floats of alignment padding in the packed buffer)
    if (tid == 0) mbar_expect_tx(&bars[0], (unsigned)(QKV_LNP * 4 + (pre == nullptr ? 64 * NQKV * 4 : 0)));
    __syncthreads();
    if (tid < 6) {
        const float* src = tid == 0 ? w.lnq_g : tid == 1 ? w.lnq_b : tid == 2 ? w.lnk_g : tid == 3 ? w.lnk_b : tid == 4 ? w.lnv_g : w.lnv_b;
        float* dst = LNP + (tid < 4 ? tid * QK_LD : 4 * QK_LD + (tid - 4) * V_DIM);
        tma_load_1d(dst, src, (tid < 4 ? QK_LD : V_DIM) * 4, &bars[0]);
    }
    if (pre == nullptr) tma_load_split(Ws, w.wqkv_t, 64 * NQKV * 4, &bars[0], tid, QKV_THREADS);
    griddep_wait();
    if (pre != nullptr) {            // projections already done by mid_kernel: bulk copies stage them
        if (tid == 0) mbar_expect_tx(&bars[1], NF * NQKV * 4);
        __syncthreads();
        tma_load_split(P, pre + ((int64_t)b * T + t) * NF * NQKV, NF * NQKV * 4, &bars[1], tid, QKV_THREADS);
        mbar_wait(&bars[1], 0);
        mbar_wait(&bars[0], 0);
    } else {
    mbar_wait(&bars[0], 0);
    const float* xr = X + ((int64_t)b * T + t) * NF * CH;
    for (int i = tid; i < 100 * 16; i += QKV_THREADS) {       // float4 loads; lanes along f -> conflict-free stores
        const int c4 = i / 100, f = i % 100;
        const float4 v = (f < NF) ? *reinterpret_cast<const float4*>(xr + f * CH + c4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
        Xt[(c4 * 4 + 0) * 100 + f] = v.x; Xt[(c4 * 4 + 1) * 100 + f] = v.y;
        Xt[(c4 * 4 + 2) * 100 + f] = v.z; Xt[(c4 * 4 + 3) * 100 + f] = v.w;
    }
    __syncthreads();
    // 4 rows x 4 cols register tiles: 25 row groups x 28 col groups
    for (int it = tid; it < 25 * 28; it += QKV_THREADS) {
        const int rg = it / 28, cg = it % 28;
        float2 acc[4][2];
#pragma unroll
        for (int i = 0; i < 4; ++i) { acc[i][0] = make_float2(0.f, 0.f); acc[i][1] = make_float2(0.f, 0.f); }
#pragma unroll 8
        for (int k = 0; k < 64; ++k) {
            const float4 a = *reinterpret_cast<const float4*>(Xt + k * 100 + rg * 4);
            const float4 bb = *reinterpret_cast<const float4*>(Ws + k * NQKV + cg * 4);
            const float2 b0 = make_float2(bb.x, bb.y), b1 = make_float2(bb.z, bb.w);
            const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 aa = make_float2(av[i], av[i]);
                acc[i][0] = ffma2(aa, b0, acc[i][0]);
                acc[i][1] = ffma2(aa, b1, acc[i][1]);
            }
        }
        const int n0 = cg * 4;
        const float slope = __ldg(w.slopes + (n0 < 24 ? 0 : (n0 < 48 ? 1 : 2)));   // 24, 48 are multiples of 4
        const float4 bias = __ldg(reinterpret_cast<const float4*>(w.bqkv + n0));
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int f = rg * 4 + i;
            if (f < NF) {
                P[f * QKV_PLD + n0 + 0] = prelu(acc[i][0].x + bias.x, slope);
                P[f * QKV_PLD + n0 + 1] = prelu(acc[i][0].y + bias.y, slope);
                P[f * QKV_PLD + n0 + 2] = prelu(acc[i][1].x + bias.z, slope);
                P[f * QKV_PLD + n0 + 3] = prelu(acc[i][1].y + bias.w, slope);
            }
        }
    }
    }
    __syncthreads();
    // LayerNorm per (which, head): one warp each
    const int warp = tid >> 5, lane = tid & 31;
    const int which = warp >> 2, h = warp & 3;
    const int d = (which == 2) ? VD : QE;
    const int n = NF * d;
    const int col0 = (which == 2) ? (48 + h * VD) : (which * 24 + h * QE);
    // element i = f*d + e lives at P[f][col0 + e]; walk (f, e) incrementally (no division in the loops)
    const int f0 = lane / d, e0 = lane % d, df = 32 / d, de = 32 % d;
    float s = 0.f;
    {
        int f = f0, e2 = e0;
        for (int i = lane; i < n; i += 32) {
            s += P[f * QKV_PLD + col0 + e2];
            e2 += de; f += df;
            if (e2 >= d) { e2 -= d; ++f; }
        }
    }
    const float mu = warp_sum(s) / (float)n;
    float q = 0.f;
    {
        int f = f0, e2 = e0;
        for (int i = lane; i < n; i += 32) {
            const float dv = P[f * QKV_PLD + col0 + e2] - mu;
            q += dv * dv;
            e2 += de; f += df;
            if (e2 >= d) { e2 -= d; ++f; }
        }
    }
    const float rs = rsqrtf(warp_sum(q) / (float)n + 1e-5f);
    const float* gam = LNP + (which == 0 ? 0 : (which == 1 ? 2 * QK_LD : 4 * QK_LD));
    const float* bet = LNP + (which == 0 ? QK_LD : (which == 1 ? 3 * QK_LD : 4 * QK_LD + V_DIM));
    float* rec = stream_rec(state, recs, b);
    const long long pos = rec_pos(rec) + frame_k;
    const int ld = (which == 2) ? V_DIM : QK_LD;
    float* dst0 = nullptr;   // linear scratch / Q buffer
    float* dst1 = nullptr;   // ring slot
    const int64_t bh = (int64_t)b * NHEAD + h;
    if (which == 0) {
        dst0 = Qbuf + (bh * T + t) * QK_LD;
    } else {
        float* sb = rec + ST_BLK + (int64_t)blk * BK_STRIDE;
        const int slot = (int)((pos + t) % RING);
        // the ring keeps the last ATT of the frames the row advances; a frame past them (t >= T_b + RING - ATT + 1) would
        // overwrite a row the next call's window still reads
        const int Tb = row_frames(recs, b, T);
        if (t >= Tb - ATT && row_has_frame(recs, t, Tb) && stream_active(recs, active, b))
            dst1 = sb + (which == 1 ? BK_K : BK_V) + ((int64_t)h * RING + slot) * ld;
        if (T > 1) dst0 = (which == 1 ? Kall : Vall) + (bh * (ATT - 1 + T) + (ATT - 1) + t) * ld;
    }
    {
        int f = f0, e2 = e0;
        for (int i = lane; i < n; i += 32) {
            const float v = (P[f * QKV_PLD + col0 + e2] - mu) * rs * gam[i] + bet[i];
            if (dst0) dst0[i] = v;
            if (dst1) dst1[i] = v;
            e2 += de; f += df;
            if (e2 >= d) { e2 -= d; ++f; }
        }
    }
    if (which != 2 && lane < 2) {        // zero the two pad columns of 582 -> 584
        if (dst0) dst0[QK_DIM + lane] = 0.f;
        if (dst1) dst1[QK_DIM + lane] = 0.f;
    }
}

// ------------------------------------------------------------------------------------------
// K4a for MANY frames (offline batches, many streams) when the projections come from a tensor-core GEMM: the same
// LayerNorm + head split + ring append as qkv_kernel, but persistent -- each CTA stages the LayerNorm parameters ONCE
// (22 KB) and walks frames fi = blockIdx.x, + gridDim.x, ... with the 43 KB projection tile of the next frame in flight
// (two TMA-filled buffers) while the 12 warps normalise the current one.  qkv_kernel's one-CTA-per-frame form pays
// the staging latency per frame; this form is bound by the 86 KB each frame moves.
constexpr size_t QKV_MANY_SMEM = (size_t)(2 * NF * QKV_PLD + QKV_LNP) * sizeof(float);

template <class Map>
__global__ void __launch_bounds__(QKV_THREADS)
qkv_many_kernel_t(const float* __restrict__ pre, float* __restrict__ Qbuf, float* __restrict__ Kall, float* __restrict__ Vall,
                  float* __restrict__ state, Map recs, int blk, BlockWeights w, int T, int n_frames,
                  const uint8_t* __restrict__ active) {
    extern __shared__ __align__(16) float sm[];
    float* Pb[2] = {sm, sm + NF * QKV_PLD};
    float* LNP = sm + 2 * NF * QKV_PLD;
    __shared__ __align__(8) unsigned long long bars[3];
    const int tid = threadIdx.x;
    griddep_launch();
    if (tid == 0) { mbar_init(&bars[0], 1); mbar_init(&bars[1], 1); mbar_init(&bars[2], 1); mbar_fence_init(); }
    __syncthreads();
    if (tid == 0) mbar_expect_tx(&bars[2], (unsigned)(QKV_LNP * 4));
    __syncthreads();
    if (tid < 6) {
        const float* src = tid == 0 ? w.lnq_g : tid == 1 ? w.lnq_b : tid == 2 ? w.lnk_g : tid == 3 ? w.lnk_b : tid == 4 ? w.lnv_g : w.lnv_b;
        float* dst = LNP + (tid < 4 ? tid * QK_LD : 4 * QK_LD + (tid - 4) * V_DIM);
        tma_load_1d(dst, src, (tid < 4 ? QK_LD : V_DIM) * 4, &bars[2]);
    }
    griddep_wait();
    int fi = blockIdx.x;
    if (fi < n_frames && tid == 0) {
        mbar_expect_tx(&bars[0], NF * NQKV * 4);
        tma_load_1d(Pb[0], pre + (int64_t)fi * NF * NQKV, NF * NQKV * 4, &bars[0]);
    }
    mbar_wait(&bars[2], 0);
    const int warp = tid >> 5, lane = tid & 31;
    const int which = warp >> 2, h = warp & 3;
    const int d = (which == 2) ? VD : QE;
    const int n = NF * d;
    const int col0 = (which == 2) ? (48 + h * VD) : (which * 24 + h * QE);
    const int f0 = lane / d, e0 = lane % d, df = 32 / d, de = 32 % d;
    const float* gam = LNP + (which == 0 ? 0 : (which == 1 ? 2 * QK_LD : 4 * QK_LD));
    const float* bet = LNP + (which == 0 ? QK_LD : (which == 1 ? 3 * QK_LD : 4 * QK_LD + V_DIM));
    const int ld = (which == 2) ? V_DIM : QK_LD;
    unsigned it = 0;
    for (; fi < n_frames; fi += gridDim.x, ++it) {
        const int cur = it & 1;
        const int nxt = fi + gridDim.x;
        if (nxt < n_frames && tid == 0) {                  // the other buffer was released by the barrier that ended the previous frame
            fence_proxy_async();
            mbar_expect_tx(&bars[cur ^ 1], NF * NQKV * 4);
            tma_load_1d(Pb[cur ^ 1], pre + (int64_t)nxt * NF * NQKV, NF * NQKV * 4, &bars[cur ^ 1]);
        }
        mbar_wait(&bars[cur], (it >> 1) & 1);
        const float* P = Pb[cur];
        const int b = fi / T, t = fi % T;
        float s = 0.f;
        {
            int f = f0, e2 = e0;
            for (int i = lane; i < n; i += 32) {
                s += P[f * QKV_PLD + col0 + e2];
                e2 += de; f += df;
                if (e2 >= d) { e2 -= d; ++f; }
            }
        }
        const float mu = warp_sum(s) / (float)n;
        float q = 0.f;
        {
            int f = f0, e2 = e0;
            for (int i = lane; i < n; i += 32) {
                const float dv = P[f * QKV_PLD + col0 + e2] - mu;
                q += dv * dv;
                e2 += de; f += df;
                if (e2 >= d) { e2 -= d; ++f; }
            }
        }
        const float rs = rsqrtf(warp_sum(q) / (float)n + 1e-5f);
        float* dst0 = nullptr;   // linear scratch / Q buffer
        float* dst1 = nullptr;   // ring slot
        const int64_t bh = (int64_t)b * NHEAD + h;
        if (which == 0) {
            dst0 = Qbuf + (bh * T + t) * QK_LD;
        } else {
            float* rec = stream_rec(state, recs, b);
            float* sb = rec + ST_BLK + (int64_t)blk * BK_STRIDE;
            const int slot = (int)((rec_pos(rec) + t) % RING);
            const int Tb = row_frames(recs, b, T);      // as in qkv_kernel
            if (t >= Tb - ATT && row_has_frame(recs, t, Tb) && stream_active(recs, active, b))
                dst1 = sb + (which == 1 ? BK_K : BK_V) + ((int64_t)h * RING + slot) * ld;
            if (T > 1) dst0 = (which == 1 ? Kall : Vall) + (bh * (ATT - 1 + T) + (ATT - 1) + t) * ld;
        }
        {
            int f = f0, e2 = e0;
            for (int i = lane; i < n; i += 32) {
                const float v = (P[f * QKV_PLD + col0 + e2] - mu) * rs * gam[i] + bet[i];
                if (dst0) dst0[i] = v;
                if (dst1) dst1[i] = v;
                e2 += de; f += df;
                if (e2 >= d) { e2 -= d; ++f; }
            }
        }
        if (which != 2 && lane < 2) {        // zero the two pad columns of 582 -> 584
            if (dst0) dst0[QK_DIM + lane] = 0.f;
            if (dst1) dst1[QK_DIM + lane] = 0.f;
        }
        __syncthreads();                     // every warp is done with buffer `cur`: it may be refilled
    }
}

// ------------------------------------------------------------------------------------------
// K4b local attention: each query attends to its own frame + the 49 previous ones, unmasked
// (tfgridnet_causal.py:564-581).  One CTA per (frame, head, stream): grid (T, 4, B), 256 threads.
// T == 1: K/V rows are ring slots (frame n lives in slot n mod RING); T > 1: rows t .. t+49 of the
// linear scratch.  Used when there are enough (frame, head, stream) items to fill the GPU but too few
// frames per stream to tile (e.g. 256 streams x 1 hop); see attn_cluster_kernel / attn_tile_kernel.
template <class Map>
__global__ void __launch_bounds__(256)
attn_kernel_t(const float* __restrict__ Qbuf, const float* __restrict__ Kall, const float* __restrict__ Vall,
              const float* __restrict__ state, Map recs, int blk, float* __restrict__ Z, int T, int frame_k) {
    __shared__ __align__(16) float qs[QK_LD];
    __shared__ float sc[64];
    griddep_launch();
    griddep_wait();
    const int t = blockIdx.x, h = blockIdx.y, b = blockIdx.z, tid = threadIdx.x;
    const int64_t bh = (int64_t)b * NHEAD + h;
    const float* kb;
    const float* vb;
    int first = 0, wrap = 0x7fffffff;       // window row j -> storage row (first + j) % wrap
    if (T == 1) {                           // ring: window = frames pos-49 .. pos of the stream's clock
        const float* rec = stream_rec(state, recs, b);
        const float* sb = rec + ST_BLK + (int64_t)blk * BK_STRIDE;
        kb = sb + BK_K + (int64_t)h * RING * QK_LD;
        vb = sb + BK_V + (int64_t)h * RING * V_DIM;
        const long long p0 = rec_pos(rec) + frame_k - (ATT - 1);
        first = (int)(((p0 % RING) + RING) % RING);
        wrap = RING;
    } else {
        kb = Kall + (bh * (ATT - 1 + T) + t) * QK_LD;
        vb = Vall + (bh * (ATT - 1 + T) + t) * V_DIM;
    }
    const float* q = Qbuf + (bh * T + t) * QK_LD;
    for (int i = tid; i < QK_LD / 4; i += 256)
        reinterpret_cast<float4*>(qs)[i] = reinterpret_cast<const float4*>(q)[i];
    __syncthreads();
    const int warp = tid >> 5, lane = tid & 31;
    const float scale = rsqrtf((float)QK_DIM);
    for (int j = warp; j < ATT; j += 8) {
        const float4* kr = reinterpret_cast<const float4*>(kb + (int64_t)((first + j) % wrap) * QK_LD);
        float4 kv[5];
#pragma unroll
        for (int u = 0; u < 5; ++u) {
            const int i = lane + 32 * u;
            kv[u] = (i < QK_LD / 4) ? kr[i] : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        float s = 0.f;
#pragma unroll
        for (int u = 0; u < 5; ++u) {
            const int i = lane + 32 * u;
            if (i < QK_LD / 4) {
                const float4 qv = reinterpret_cast<const float4*>(qs)[i];
                s += kv[u].x * qv.x + kv[u].y * qv.y + kv[u].z * qv.z + kv[u].w * qv.w;
            }
        }
        s = warp_sum(s);
        if (lane == 0) sc[j] = s * scale;
    }
    __syncthreads();
    if (warp == 0) {
        const float a0 = sc[lane];
        const float a1 = (lane + 32 < ATT) ? sc[lane + 32] : -INFINITY;
        const float mx = warp_max(fmaxf(a0, a1));
        const float e0 = __expf(a0 - mx);
        const float e1 = (lane + 32 < ATT) ? __expf(a1 - mx) : 0.f;
        const float inv = 1.f / warp_sum(e0 + e1);
        sc[lane] = e0 * inv;
        if (lane + 32 < ATT) sc[lane + 32] = e1 * inv;
    }
    __syncthreads();
    float* zr = Z + ((int64_t)b * T + t) * NF * CH;
    for (int c4 = tid; c4 < V_DIM / 4; c4 += 256) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int j0 = 0; j0 < ATT; j0 += 10) {       // 10 value rows in flight per thread
            float4 v[10];
#pragma unroll
            for (int u = 0; u < 10; ++u)
                v[u] = reinterpret_cast<const float4*>(vb + (int64_t)((first + j0 + u) % wrap) * V_DIM)[c4];
#pragma unroll
            for (int u = 0; u < 10; ++u) {
                const float p = sc[j0 + u];
                acc.x = fmaf(p, v[u].x, acc.x); acc.y = fmaf(p, v[u].y, acc.y);
                acc.z = fmaf(p, v[u].z, acc.z); acc.w = fmaf(p, v[u].w, acc.w);
            }
        }
        const int f = c4 >> 2, c0 = (c4 & 3) * 4;            // feature f*16 + c -> channel h*16 + c
        *reinterpret_cast<float4*>(zr + f * CH + h * VD + c0) = acc;
    }
}

// K4b'' query-tiled local attention for multi-frame calls: consecutive queries share 49 of their 50
// window rows, so one CTA serves ATT_TQ consecutive queries of a (stream, head) from ONE pass over the
// ATT_TQ + 49 rows of the linear K/V scratch: ~7x less L2 traffic than one CTA per query.
// grid (ceil(T/ATT_TQ), 4, B), 256 threads (8 warps = 8 queries in the softmax phase).
constexpr int ATT_TQ = 8;
constexpr int ATT_TR = ATT_TQ + ATT - 1;        // 57 rows per tile

__global__ void __launch_bounds__(256)
attn_tile_kernel(const float* __restrict__ Qbuf, const float* __restrict__ Kall, const float* __restrict__ Vall,
                 float* __restrict__ Z, int T) {
    __shared__ __align__(16) float qs[ATT_TQ][QK_LD];    // 18.7 KB
    __shared__ float sc[ATT_TQ][ATT_TR + 3];             // scores / probabilities, [query][tile row]
    griddep_launch();
    griddep_wait();
    const int t0 = blockIdx.x * ATT_TQ, h = blockIdx.y, b = blockIdx.z, tid = threadIdx.x;
    const int nq = min(ATT_TQ, T - t0);
    const int64_t bh = (int64_t)b * NHEAD + h;
    const float* kb = Kall + (bh * (ATT - 1 + T) + t0) * QK_LD;       // tile row r = scratch row t0 + r
    const float* vb = Vall + (bh * (ATT - 1 + T) + t0) * V_DIM;
    const int nrow = nq + ATT - 1;
    for (int i = tid; i < ATT_TQ * (QK_LD / 4); i += 256) {
        const int qi = i / (QK_LD / 4), c4 = i % (QK_LD / 4);
        reinterpret_cast<float4*>(&qs[qi][0])[c4] =
            (qi < nq) ? reinterpret_cast<const float4*>(Qbuf + (bh * T + t0 + qi) * QK_LD)[c4] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();
    const int warp = tid >> 5, lane = tid & 31;
    const float scale = rsqrtf((float)QK_DIM);
    for (int r = warp; r < nrow; r += 8) {           // one warp per key row, dotted with all queries that see it
        const float4* kr = reinterpret_cast<const float4*>(kb + (int64_t)r * QK_LD);
        float4 kv[5];
#pragma unroll
        for (int u = 0; u < 5; ++u) {
            const int i = lane + 32 * u;
            kv[u] = (i < QK_LD / 4) ? kr[i] : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int qi = 0; qi < ATT_TQ; ++qi) {
            // query qi sees tile rows qi .. qi+49
            if (qi < nq && r >= qi && r < qi + ATT) {          // warp-uniform
                float s = 0.f;
#pragma unroll
                for (int u = 0; u < 5; ++u) {
                    const int i = lane + 32 * u;
                    if (i < QK_LD / 4) {
                        const float4 qv = reinterpret_cast<const float4*>(&qs[qi][0])[i];
                        s += kv[u].x * qv.x + kv[u].y * qv.y + kv[u].z * qv.z + kv[u].w * qv.w;
                    }
                }
                s = warp_sum(s);
                if (lane == 0) sc[qi][r] = s * scale;
            }
        }
    }
    __syncthreads();
    if (warp < nq) {                                 // softmax of query `warp` over its 50 rows
        const int qi = warp;
        const float a0 = sc[qi][qi + lane];
        const float a1 = (lane + 32 < ATT) ? sc[qi][qi + lane + 32] : -INFINITY;
        const float mx = warp_max(fmaxf(a0, a1));
        const float e0 = __expf(a0 - mx);
        const float e1 = (lane + 32 < ATT) ? __expf(a1 - mx) : 0.f;
        const float inv = 1.f / warp_sum(e0 + e1);
        sc[qi][qi + lane] = e0 * inv;
        if (lane + 32 < ATT) sc[qi][qi + lane + 32] = e1 * inv;
    }
    __syncthreads();
    for (int c4 = tid; c4 < V_DIM / 4; c4 += 256) {
        float4 acc[ATT_TQ];
#pragma unroll
        for (int qi = 0; qi < ATT_TQ; ++qi) acc[qi] = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int r0 = 0; r0 < nrow; r0 += 8) {       // 8 value rows in flight per thread
            float4 v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u)
                v[u] = (r0 + u < nrow) ? reinterpret_cast<const float4*>(vb + (int64_t)(r0 + u) * V_DIM)[c4]
                                       : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int r = r0 + u;
#pragma unroll
                for (int qi = 0; qi < ATT_TQ; ++qi) {
                    if (r < nrow && r >= qi && r < qi + ATT) {       // uniform across the CTA
                        const float p = sc[qi][r];
                        acc[qi].x = fmaf(p, v[u].x, acc[qi].x); acc[qi].y = fmaf(p, v[u].y, acc[qi].y);
                        acc[qi].z = fmaf(p, v[u].z, acc[qi].z); acc[qi].w = fmaf(p, v[u].w, acc[qi].w);
                    }
                }
            }
        }
        const int f = c4 >> 2, c0 = (c4 & 3) * 4;
#pragma unroll
        for (int qi = 0; qi < ATT_TQ; ++qi)
            if (qi < nq)
                *reinterpret_cast<float4*>(Z + (((int64_t)b * T + t0 + qi) * NF + f) * CH + h * VD + c0) = acc[qi];
    }
}

// K4b' cluster attention for few frames in flight: the 50-row window of one (stream, frame, head) is
// split over a thread-block CLUSTER of 8 CTAs (8 SMs); every CTA reduces its rows to an
// un-normalised partial (max, sum, o[1552]) in its own shared memory, then the cluster merges the
// partials through distributed shared memory (each CTA owns 1/8 of the output columns and reads
// that slice from its 7 peers) and writes the final, normalised head output.  No scratch round trip
// through L2/HBM, no separate merge pass.  grid (T, 4*8, B), cluster (1, 8, 1), 256 threads.
constexpr int ATT_CL = 8;

template <class Map>
__global__ void __launch_bounds__(256)
attn_cluster_kernel_t(const float* __restrict__ Qbuf, const float* __restrict__ Kall, const float* __restrict__ Vall,
                      const float* __restrict__ state, Map recs, int blk, float* __restrict__ Z, int T,
                      int frame_k) {
    namespace cg = cooperative_groups;
    __shared__ __align__(16) float qs[QK_LD];
    __shared__ __align__(16) float os[V_DIM];     // this CTA's partial output
    __shared__ float ml[2];                        // its running max and sum
    __shared__ float sc[16];
    __shared__ float coef[ATT_CL];
    TraceScope trace_(TK_ATTN, Qbuf);
    griddep_launch();
    griddep_wait();
    cg::cluster_group cluster = cg::this_cluster();
    const int t = blockIdx.x, h = blockIdx.y / ATT_CL, rk = blockIdx.y % ATT_CL, b = blockIdx.z, tid = threadIdx.x;
    const int base = ATT / ATT_CL, rem = ATT % ATT_CL;           // 6 rows each, the first 2 ranks take 7
    const int j0 = rk * base + min(rk, rem), nr = base + (rk < rem ? 1 : 0);
    const int64_t bh = (int64_t)b * NHEAD + h;
    const float* kb;
    const float* vb;
    int first = j0, wrap = 0x7fffffff;      // window row j -> storage row (first + j) % wrap
    if (T == 1) {                           // ring: window = frames pos-49 .. pos of the stream's clock, frame n in slot n mod RING
        const float* rec = stream_rec(state, recs, b);
        const float* sb = rec + ST_BLK + (int64_t)blk * BK_STRIDE;
        kb = sb + BK_K + (int64_t)h * RING * QK_LD;
        vb = sb + BK_V + (int64_t)h * RING * V_DIM;
        const long long p0 = rec_pos(rec) + frame_k - (ATT - 1) + j0;
        first = (int)(((p0 % RING) + RING) % RING);
        wrap = RING;
    } else {
        kb = Kall + (bh * (ATT - 1 + T) + t) * QK_LD;
        vb = Vall + (bh * (ATT - 1 + T) + t) * V_DIM;
    }
    const float* q = Qbuf + (bh * T + t) * QK_LD;
    for (int i = tid; i < QK_LD / 4; i += 256)
        reinterpret_cast<float4*>(qs)[i] = reinterpret_cast<const float4*>(q)[i];
    __syncthreads();
    const int warp = tid >> 5, lane = tid & 31;
    const float scale = rsqrtf((float)QK_DIM);
    if (warp < nr) {                               // one warp per key row (nr <= 7)
        const float4* kr = reinterpret_cast<const float4*>(kb + (int64_t)((first + warp) % wrap) * QK_LD);
        float4 kv[5];
#pragma unroll
        for (int u = 0; u < 5; ++u) {
            const int i = lane + 32 * u;
            kv[u] = (i < QK_LD / 4) ? kr[i] : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        float s = 0.f;
#pragma unroll
        for (int u = 0; u < 5; ++u) {
            const int i = lane + 32 * u;
            if (i < QK_LD / 4) {
                const float4 qv = reinterpret_cast<const float4*>(qs)[i];
                s += kv[u].x * qv.x + kv[u].y * qv.y + kv[u].z * qv.z + kv[u].w * qv.w;
            }
        }
        s = warp_sum(s);
        if (lane == 0) sc[warp] = s * scale;
    }
    __syncthreads();
    if (warp == 0) {
        const float a0 = (lane < nr) ? sc[lane] : -INFINITY;
        const float mx = warp_max(a0);
        const float e0 = (lane < nr) ? __expf(a0 - mx) : 0.f;
        const float lsum = warp_sum(e0);
        if (lane < nr) sc[lane] = e0;
        if (lane == 0) { ml[0] = mx; ml[1] = lsum; }
    }
    __syncthreads();
    for (int c4 = tid; c4 < V_DIM / 4; c4 += 256) {
        float4 v[7];
#pragma unroll
        for (int j = 0; j < 7; ++j)
            v[j] = (j < nr) ? reinterpret_cast<const float4*>(vb + (int64_t)((first + j) % wrap) * V_DIM)[c4]
                            : make_float4(0.f, 0.f, 0.f, 0.f);
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < 7; ++j) {
            const float p = (j < nr) ? sc[j] : 0.f;
            acc.x = fmaf(p, v[j].x, acc.x); acc.y = fmaf(p, v[j].y, acc.y);
            acc.z = fmaf(p, v[j].z, acc.z); acc.w = fmaf(p, v[j].w, acc.w);
        }
        reinterpret_cast<float4*>(os)[c4] = acc;
    }
    cluster.sync();                                // every CTA's partial is complete and visible cluster-wide
    // ---- merge through distributed shared memory ---------------------------------------------------
    if (tid < ATT_CL) {
        const float* pml = cluster.map_shared_rank(ml, tid);
        sc[8 + tid] = pml[0];                      // peer maxima
        coef[tid] = pml[1];                        // peer sums (turned into weights below)
    }
    __syncthreads();
    if (tid == 0) {
        float mstar = -INFINITY;
        for (int p = 0; p < ATT_CL; ++p) mstar = fmaxf(mstar, sc[8 + p]);
        float den = 0.f, wgt[ATT_CL];
        for (int p = 0; p < ATT_CL; ++p) { wgt[p] = __expf(sc[8 + p] - mstar); den += wgt[p] * coef[p]; }
        const float inv = 1.f / den;
        for (int p = 0; p < ATT_CL; ++p) coef[p] = wgt[p] * inv;
    }
    __syncthreads();
    constexpr int COLS = (V_DIM / 4 + ATT_CL - 1) / ATT_CL;      // 49 float4 columns per CTA
    float* zr = Z + ((int64_t)b * T + t) * NF * CH;
    if (tid < COLS) {
        const int c4 = rk * COLS + tid;
        if (c4 < V_DIM / 4) {
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int p = 0; p < ATT_CL; ++p) {
                const float4 v = reinterpret_cast<const float4*>(cluster.map_shared_rank(os, p))[c4];
                const float cf = coef[p];
                acc.x = fmaf(cf, v.x, acc.x); acc.y = fmaf(cf, v.y, acc.y);
                acc.z = fmaf(cf, v.z, acc.z); acc.w = fmaf(cf, v.w, acc.w);
            }
            const int f = c4 >> 2, c0 = (c4 & 3) * 4;            // feature f*16 + c -> channel h*16 + c
            *reinterpret_cast<float4*>(zr + f * CH + h * VD + c0) = acc;
        }
    }
    cluster.sync();                                // nobody leaves while a peer may still read its shared memory
}

// ------------------------------------------------------------------------------------------
// K4c attention output: Linear(64->64) + PReLU + LayerNorm over (F, C) + residual
// (tfgridnet_causal.py:583-588); for block 0 the speaker gate that the reference applies to the
// input of block 1 (:250-251) is folded into this epilogue.  grid (T, B), 256 threads.
// The residual rows, the gate and the LayerNorm parameters are read once per element, so none is staged in shared memory
// (the residual rows go to registers during the projection, the rest is read where it is used): 67 KB per CTA lets three
// of them, or one next to a BiLSTM, share an SM.
constexpr size_t AOUT_SMEM = (size_t)(64 * 100 + 64 * 64 + NF * 64) * sizeof(float);
constexpr int AOUT_EPI = (FC / 4 + 255) / 256;      // float4s of the frame per thread in the epilogue

template <class Map>
__global__ void __launch_bounds__(256)
attn_out_kernel_t(const float* __restrict__ Z, float* __restrict__ X, const float* __restrict__ state,
                  Map recs, BlockWeights w, int apply_gate, int T) {
    extern __shared__ __align__(16) float sm[];
    __shared__ float red[32];
    float* Zt = sm;                 // [64][100]
    float* Ws = Zt + 64 * 100;      // [64][64]
    float* P = Ws + 64 * 64;        // [97][64]
    __shared__ __align__(8) unsigned long long bars[1];
    const int t = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    float* xr = X + ((int64_t)b * T + t) * NF * CH;
    const float* gate = stream_rec(state, recs, b) + ST_GATE;
    TraceScope trace_(TK_ATTN_OUT, Z);
    griddep_launch();
    if (tid == 0) { mbar_init(&bars[0], 1); mbar_fence_init(); }
    __syncthreads();
    // parameters: before the dependency wait
    if (tid == 0) mbar_expect_tx(&bars[0], 64 * 64 * 4);
    __syncthreads();
    tma_load_split(Ws, w.wp_t, 64 * 64 * 4, &bars[0], tid, 256);
    griddep_wait();
    // chain data: the residual rows, in flight during the projection
    float4 xv[AOUT_EPI];
#pragma unroll
    for (int j = 0; j < AOUT_EPI; ++j) {
        const int i = tid + j * 256;
        xv[j] = (i < FC / 4) ? reinterpret_cast<const float4*>(xr)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    {
        const float* zr = Z + ((int64_t)b * T + t) * NF * CH;
        for (int i = tid; i < 100 * 16; i += 256) {
            const int c4 = i / 100, f = i % 100;
            const float4 v = (f < NF) ? *reinterpret_cast<const float4*>(zr + f * CH + c4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
            Zt[(c4 * 4 + 0) * 100 + f] = v.x; Zt[(c4 * 4 + 1) * 100 + f] = v.y;
            Zt[(c4 * 4 + 2) * 100 + f] = v.z; Zt[(c4 * 4 + 3) * 100 + f] = v.w;
        }
    }
    mbar_wait(&bars[0], 0);
    __syncthreads();
    const float slope = __ldg(w.slopes + 3);
    for (int it = tid; it < 25 * 16; it += 256) {
        const int rg = it / 16, cg = it % 16;
        float2 acc[4][2];
#pragma unroll
        for (int i = 0; i < 4; ++i) { acc[i][0] = make_float2(0.f, 0.f); acc[i][1] = make_float2(0.f, 0.f); }
#pragma unroll 8
        for (int k = 0; k < 64; ++k) {
            const float4 a = *reinterpret_cast<const float4*>(Zt + k * 100 + rg * 4);
            const float4 bb = *reinterpret_cast<const float4*>(Ws + k * 64 + cg * 4);
            const float2 b0 = make_float2(bb.x, bb.y), b1 = make_float2(bb.z, bb.w);
            const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 aa = make_float2(av[i], av[i]);
                acc[i][0] = ffma2(aa, b0, acc[i][0]);
                acc[i][1] = ffma2(aa, b1, acc[i][1]);
            }
        }
        const int n0 = cg * 4;
        const float4 bias = __ldg(reinterpret_cast<const float4*>(w.bp + n0));
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int f = rg * 4 + i;
            if (f < NF) {
                float4 o;
                o.x = prelu(acc[i][0].x + bias.x, slope);
                o.y = prelu(acc[i][0].y + bias.y, slope);
                o.z = prelu(acc[i][1].x + bias.z, slope);
                o.w = prelu(acc[i][1].y + bias.w, slope);
                *reinterpret_cast<float4*>(P + f * 64 + n0) = o;
            }
        }
    }
    __syncthreads();
    float s = 0.f;
    for (int i = tid; i < FC; i += 256) s += P[i];
    const float mu = block_sum(s, red) * (1.f / FC);
    float q = 0.f;
    for (int i = tid; i < FC; i += 256) { const float d = P[i] - mu; q += d * d; }
    const float rs = rsqrtf(block_sum(q, red) * (1.f / FC) + 1e-5f);
#pragma unroll
    for (int j = 0; j < AOUT_EPI; ++j) {
        const int i = tid + j * 256;
        if (i < FC / 4) {
            float4 x4 = xv[j];
            const float4 p4 = reinterpret_cast<const float4*>(P)[i];
            const float4 g4 = __ldg(reinterpret_cast<const float4*>(w.lnp_g) + i);
            const float4 b4 = __ldg(reinterpret_cast<const float4*>(w.lnp_b) + i);
            x4.x += (p4.x - mu) * rs * g4.x + b4.x; x4.y += (p4.y - mu) * rs * g4.y + b4.y;
            x4.z += (p4.z - mu) * rs * g4.z + b4.z; x4.w += (p4.w - mu) * rs * g4.w + b4.w;
            if (apply_gate) {
                const float4 t4 = __ldg(reinterpret_cast<const float4*>(gate) + i);
                x4.x *= t4.x; x4.y *= t4.y; x4.z *= t4.z; x4.w *= t4.w;
            }
            reinterpret_cast<float4*>(xr)[i] = x4;
        }
    }
}

// ------------------------------------------------------------------------------------------
// K5 back: causal 3x3 transposed conv (64 -> 4) + Re/Im regroup + synthesis filterbank +
// overlap-add   (tfgridnet_causal.py:256-273; net.py:61 drops the look-ahead tail).
// grid (BACK_CL * T, B) in clusters of BACK_CL CTAs, 256 threads.  y: [B][NSRC][y_len], frame t writes
// samples 128 t .. 128 t + 127.  One frame is one cluster: CTA `part` owns a quarter of the frequency bins
// -- it stages those rows (+ halo) of the four frames it needs by TMA, runs the deconv for them, and sums
// the synthesis filterbank over ITS rows only (its 2 x ~24 filter rows, 37 KB, prefetched by TMA before the
// dependency wait).  The four partial windows meet in CTA 0 through distributed shared memory, in a fixed
// order, and CTA 0 does the overlap-add and the store.  (v1 ran the frame in one CTA, which made it the
// slowest stage of the one-hop pipeline once the mid section was split.)
// The last CTA to finish advances the header and the clocks of the active streams (finish_call).
constexpr int BACK_CL = 4;
constexpr int BACK_FMAX = (NF + BACK_CL - 1) / BACK_CL;       // 25 bins per CTA at most
constexpr size_t BACK_SMEM = (size_t)(4 * (BACK_FMAX + 2) * 64 + 2 * BACK_FMAX * NFFT + 2 * NSRC * NROW + NSRC * NFFT) * sizeof(float);

__device__ __forceinline__ int back_f0(int part) { return (part * NF) / BACK_CL; }

template <class Map>
__global__ void __launch_bounds__(256)
back_kernel_t(const float* __restrict__ X, float* __restrict__ y, int64_t y_bstride, int64_t y_cstride,
              int y_len, float* __restrict__ state, Map recs, SepWeights w, int T, int pos_rel, int frame_k,
              int frames_total, int sample_off, int64_t hist_stride, const uint8_t* __restrict__ active) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    extern __shared__ __align__(16) float sm[];
    float* Xs = sm;                                    // [4 slots: frame t-3+i][nf + 2 rows: f0-1 .. f1][64]
    float* Wf = Xs + 4 * (BACK_FMAX + 2) * 64;         // [2: re, im][nf][192] this CTA's synthesis filter rows
    float* R = Wf + 2 * BACK_FMAX * NFFT;              // [2: frame t-1, t][2 ears][194]  (own bins only)
    float* wacc = R + 2 * NSRC * NROW;                 // [2 ears][192] partial synthesis sums
    __shared__ __align__(8) unsigned long long bars[2];
    const int part = (int)cluster.block_rank();
    const int t = blockIdx.x / BACK_CL, b = blockIdx.y, tid = threadIdx.x;
    const int f0 = back_f0(part), f1 = back_f0(part + 1), nf = f1 - f0;
    const int ld = nf + 2;                             // staged rows per frame slot: bins f0-1 .. f1
    TraceScope trace_(TK_BACK, X);
    griddep_launch();
    if (tid == 0) {
        mbar_init(&bars[0], 1); mbar_init(&bars[1], 1); mbar_fence_init();
        // this CTA's filter rows: weights, so they can be on their way before the dependency wait
        mbar_expect_tx(&bars[1], 2 * nf * NFFT * 4);
        tma_load_1d(Wf, w.ws + (int64_t)f0 * NFFT, nf * NFFT * 4, &bars[1]);
        tma_load_1d(Wf + nf * NFFT, w.ws + (int64_t)(NF + f0) * NFFT, nf * NFFT * 4, &bars[1]);
    }
    // group bookkeeping as in front_kernel: gi = frame index in the group, frames before the group come
    // from the deconv tails the previous group left, frames inside it from X (T > 1) or from the
    // workspace slots of the previous one-frame calls of the pipelined graph (hist_stride apart)
    const int gi = frame_k + t, GN = row_frames(recs, b, (frames_total > 1) ? frames_total : T);
    // zero the halo rows that fall outside 0 .. 96 and whole slots that stay empty
    for (int i = tid; i < 4 * ld * 64; i += 256) {
        const int slot = i / (ld * 64), r = (i / 64) % ld;
        const int g = gi - 3 + slot, f = f0 - 1 + r;
        if (f < 0 || f >= NF || g < -2) Xs[i] = 0.f;
    }
    float wr[2][36];
    {
        const int lane = tid & 31;
#pragma unroll
        for (int u = 0; u < 2; ++u)
#pragma unroll
            for (int k = 0; k < 36; ++k) wr[u][k] = __ldg(w.wd + (lane + 32 * u) * 36 + k);
    }
    __syncthreads();
    griddep_wait();
    trace_.mark(0);
    const StateHeader* hdr = reinterpret_cast<const StateHeader*>(state);
    const int soff = sample_off + (pos_rel ? (int)(hdr->pos - hdr->clip_base) * HOP : 0);
    float* st = stream_rec(state, recs, b);
    const int par = rec_par(st);
    const bool live = stream_active(recs, active, b);
    const float* db = st + ST_DECONV + par * (2 * FC);
    float* db_next = st + ST_DECONV + (par ^ 1) * (2 * FC);
    const float* ib = st + ST_ISTFT + par * (NSRC * NROW);
    float* ib_next = st + ST_ISTFT + (par ^ 1) * (NSRC * NROW);
    const int lo = max(f0 - 1, 0), hi = min(f1 + 1, NF);          // staged bins that exist: [lo, hi)
    if (tid == 0) {
        int nfr = 0;
        for (int slot = 0; slot < 4; ++slot) nfr += (gi - 3 + slot >= -2) ? 1 : 0;
        fence_proxy_async();
        mbar_expect_tx(&bars[0], nfr * (hi - lo) * 64 * 4);
        for (int slot = 0; slot < 4; ++slot) {
            const int g = gi - 3 + slot;
            if (g < -2) continue;
            const float* src;
            if (g < 0) src = db + (2 + g) * FC;
            else if (frames_total > 1) src = X - (int64_t)(3 - slot) * hist_stride + (int64_t)b * FC;   // slot of one-frame call g
            else src = X + ((int64_t)b * T + (t - 3 + slot)) * FC;
            tma_load_1d(Xs + (slot * ld + (lo - (f0 - 1))) * 64, src + lo * 64, (hi - lo) * 64 * 4, &bars[0]);
        }
    }
    mbar_wait(&bars[0], 0);
    trace_.mark(1);
    // deconv of the own bins for frames t (fi = 1) and, when it is inside this call, t-1 (fi = 0)
    {
        const int warp = tid >> 5, lane = tid & 31;
        for (int fi = (gi >= 1 ? 0 : 1); fi < 2; ++fi) {
            for (int f = f0 + warp; f < f1; f += 8) {
                float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int i = 0; i < 3; ++i)
#pragma unroll
                    for (int j = 0; j < 3; ++j) {
                        // frame (t-1+fi) - i  -> slot (2 + fi - i) ; bin f+1-j -> staged row (f+1-j) - (f0-1)
                        const float* xp = Xs + ((2 + fi - i) * ld + (f + 2 - j - f0)) * 64;
                        const float x0 = xp[lane], x1 = xp[lane + 32];
#pragma unroll
                        for (int o = 0; o < 4; ++o) {
                            acc[o] = fmaf(wr[0][o * 9 + i * 3 + j], x0, acc[o]);
                            acc[o] = fmaf(wr[1][o * 9 + i * 3 + j], x1, acc[o]);
                        }
                    }
#pragma unroll
                for (int o = 0; o < 4; ++o) {
                    const float v = warp_sum(acc[o]);
                    // channel o = 2*ear + ri  ->  R[ear][ri*97 + f]
                    if (lane == 0) R[(fi * NSRC + (o >> 1)) * NROW + (o & 1) * NF + f] = v + __ldg(w.bd + o);
                }
            }
        }
        if (gi == 0)                                   // the previous group's last spectrum (own bins)
            for (int i = tid; i < NSRC * 2 * nf; i += 256) {
                const int idx = (i / (2 * nf)) * NROW + ((i / nf) & 1) * NF + f0 + i % nf;
                R[idx] = ib[idx];
            }
    }
    // next deconv tails (frames GN-2, GN-1) come straight from the staged frames of the group's last frame
    if (gi == GN - 1 && live) {
        for (int i = tid; i < nf * 16; i += 256) {
            const int r = i / 16, c4 = i % 16;
            reinterpret_cast<float4*>(db_next + (f0 + r) * 64)[c4] = reinterpret_cast<const float4*>(Xs + (2 * ld + 1 + r) * 64)[c4];
            reinterpret_cast<float4*>(db_next + FC + (f0 + r) * 64)[c4] = reinterpret_cast<const float4*>(Xs + (3 * ld + 1 + r) * 64)[c4];
        }
    }
    __syncthreads();                        // R (own bins) complete
    trace_.mark(2);
    // synthesis over the own filter rows: w_t[n] (n < 128) from R_t, w_{t-1}[n] (n >= 128) from R_{t-1}
    mbar_wait(&bars[1], 0);
#pragma unroll
    for (int u = 0; u < 2; ++u) {
        const int item = tid + 256 * u;
        if (item < NSRC * NFFT) {
            const int ear = item / NFFT, n = item % NFFT;
            const float* rr = R + (((n < HOP) ? 1 : 0) * NSRC + ear) * NROW + f0;
            float acc = 0.f;
            for (int ri = 0; ri < 2; ++ri) {
                const float* wf = Wf + ri * nf * NFFT + n;
                const float* rv = rr + ri * NF;
#pragma unroll 5
                for (int r = 0; r < nf; ++r) acc = fmaf(rv[r], wf[r * NFFT], acc);
            }
            wacc[item] = acc;
        }
    }
    if (gi == GN - 1 && live)
        for (int i = tid; i < NSRC * 2 * nf; i += 256) {
            const int idx = (i / (2 * nf)) * NROW + ((i / nf) & 1) * NF + f0 + i % nf;
            ib_next[idx] = R[NSRC * NROW + idx];
        }
    trace_.mark(3);
    cluster.sync();                         // all four partial windows are complete and visible cluster-wide
    trace_.mark(4);
    if (part == 0 && live) {
        const int yl = row_len(recs, b, T, y_len, 0);
        for (int i = tid; i < NSRC * HOP; i += 256) {
            const int ear = i / HOP, n = i % HOP;
            const int s = HOP * t + n + soff;
            if (s < yl) {
                float v = 0.f, tail = 0.f;
#pragma unroll
                for (int p = 0; p < BACK_CL; ++p) {
                    const float* pw = cluster.map_shared_rank(wacc, p);
                    v += pw[ear * NFFT + n];
                    if (n < LOOKAHEAD) tail += pw[ear * NFFT + HOP + n];
                }
                if (n < LOOKAHEAD) v += tail;               // overlap-add of the previous frame's tail
                y[(int64_t)b * y_bstride + (int64_t)ear * y_cstride + s] = v;
            }
        }
    }
    trace_.mark(5);
    cluster.sync();                         // nobody leaves while CTA 0 may still read its shared memory
    trace_.mark(6);
    // ordinary call: the last CTA to finish advances the clocks (a pipelined graph runs several back_kernels
    // at once and advances them with advance_header_kernel after all of its frames instead)
    if (frames_total == 1) finish_call(state, recs, gridDim.y, T, active);
}


// K5 for calls of MANY frames (whole utterances, offline batches): the same arithmetic as back_kernel, frame by frame in the
// same order (results are bit-identical), but one cluster walks a contiguous CHUNK of frames of a stream: its synthesis
// filter slices (37 KB per CTA) are loaded once instead of once per frame, every frame's rows are staged once (4-slot ring,
// the next frame's TMA in flight under the current frame's work) instead of four times, and the deconvolved spectrum of
// frame t-1 is carried in shared memory instead of being recomputed -- back_kernel's one-cluster-per-frame form launches
// 8 000 clusters of 4 CTAs per 16 x 500 frames.
// grid (BACK_CL * n_chunks, B) in clusters of BACK_CL, 256 threads; frames [c*chunk, min(T, (c+1)*chunk)) for cluster c.
constexpr size_t BACK_MANY_SMEM = (size_t)(4 * (BACK_FMAX + 2) * 64 + 2 * BACK_FMAX * NFFT + 2 * NSRC * NROW + 2 * NSRC * NFFT) * sizeof(float);

template <class Map>
__global__ void __launch_bounds__(256)
back_many_kernel_t(const float* __restrict__ X, float* __restrict__ y, int64_t y_bstride, int64_t y_cstride, int y_len,
                   float* __restrict__ state, Map recs, SepWeights w, int T, int pos_rel, int chunk, int n_chunks, int n_streams,
                   const uint8_t* __restrict__ active) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    extern __shared__ __align__(16) float sm[];
    float* Xs = sm;                                    // ring [4: frame g -> slot (g + 4) & 3][nf + 2 rows: f0-1 .. f1][64]
    float* Wf = Xs + 4 * (BACK_FMAX + 2) * 64;         // [2: re, im][nf][192] this CTA's synthesis filter rows
    float* R = Wf + 2 * BACK_FMAX * NFFT;              // [2: frame g -> g & 1][2 ears][194]  (own bins only)
    float* wacc = R + 2 * NSRC * NROW;                 // [2: alternating per frame][2 ears][192] partial synthesis sums
    __shared__ __align__(8) unsigned long long fbar;   // filter
    __shared__ __align__(8) unsigned long long xbar[4];// one per ring slot
    const int part = (int)cluster.block_rank();
    const int cl = blockIdx.x / BACK_CL, n_cl = gridDim.x / BACK_CL, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int f0 = back_f0(part), f1 = back_f0(part + 1), nf = f1 - f0;
    const int ld = nf + 2;
    griddep_launch();
    if (tid == 0) {
        mbar_init(&fbar, 1);
        for (int i = 0; i < 4; ++i) mbar_init(&xbar[i], 1);
        mbar_fence_init();
        mbar_expect_tx(&fbar, 2 * nf * NFFT * 4);
        tma_load_1d(Wf, w.ws + (int64_t)f0 * NFFT, nf * NFFT * 4, &fbar);
        tma_load_1d(Wf + nf * NFFT, w.ws + (int64_t)(NF + f0) * NFFT, nf * NFFT * 4, &fbar);
    }
    for (int i = tid; i < 4 * ld * 64; i += 256) {      // halo rows outside 0 .. 96 stay zero for the whole walk
        const int f = f0 - 1 + (i / 64) % ld;
        if (f < 0 || f >= NF) Xs[i] = 0.f;
    }
    float wr[2][36];
#pragma unroll
    for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int k = 0; k < 36; ++k) wr[u][k] = __ldg(w.wd + (lane + 32 * u) * 36 + k);
    float bd[4];
#pragma unroll
    for (int o = 0; o < 4; ++o) bd[o] = __ldg(w.bd + o);
    __syncthreads();
    griddep_wait();
    const StateHeader* hdr = reinterpret_cast<const StateHeader*>(state);
    const int soff = pos_rel ? (int)(hdr->pos - hdr->clip_base) * HOP : 0;
    const int lo = max(f0 - 1, 0), hi = min(f1 + 1, NF);          // staged bins that exist: [lo, hi)
    // ring-slot barriers: bit s of usebits = parity the NEXT staging into slot s completes; waitbits = parity to wait for the latest one
    unsigned usebits = 0u, waitbits = 0u;
    unsigned nframe = 0u;                               // frames this cluster has finished (selects the wacc buffer)
    mbar_wait(&fbar, 0);
    // one cluster walks (stream, chunk) items: frames [c*chunk, min(T, (c+1)*chunk)) of stream b
    for (int item = cl; item < n_streams * n_chunks; item += n_cl) {
        const int b = item / n_chunks, c = item % n_chunks;
        const int t0 = c * chunk, t1 = min(T, t0 + chunk);
        float* st = stream_rec(state, recs, b);
        const int par = rec_par(st);
        const bool live = stream_active(recs, active, b);
        const int Tb = row_frames(recs, b, T), yl = row_len(recs, b, T, y_len, 0);
        const float* db = st + ST_DECONV + par * (2 * FC);
        float* db_next = st + ST_DECONV + (par ^ 1) * (2 * FC);
        const float* ib = st + ST_ISTFT + par * (NSRC * NROW);
        float* ib_next = st + ST_ISTFT + (par ^ 1) * (NSRC * NROW);
        // frame g of this call: g >= 0 from X, g = -1, -2 from the deconv tails the previous call left
        auto stage = [&](int g) {                                     // bookkeeping by every thread, the copy by thread 0
            const int slot = (g + 4) & 3;
            waitbits = (waitbits & ~(1u << slot)) | (((usebits >> slot) & 1u) << slot);
            usebits ^= 1u << slot;
            if (tid == 0) {
                const float* src = (g < 0) ? db + (2 + g) * FC : X + ((int64_t)b * T + g) * FC;
                fence_proxy_async();
                mbar_expect_tx(&xbar[slot], (hi - lo) * 64 * 4);
                tma_load_1d(Xs + (slot * ld + (lo - (f0 - 1))) * 64, src + lo * 64, (hi - lo) * 64 * 4, &xbar[slot]);
            }
        };
        auto wait_frame = [&](int g) { const int slot = (g + 4) & 3; mbar_wait(&xbar[slot], (waitbits >> slot) & 1u); };
        // deconv of the own bins for frame g (needs frames g, g-1, g-2 in the ring) -> R[g & 1]
        auto deconv = [&](int g) {
            float* Rg = R + (g & 1) * NSRC * NROW;
            for (int f = f0 + warp; f < f1; f += 8) {
                float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int i = 0; i < 3; ++i)
#pragma unroll
                    for (int j = 0; j < 3; ++j) {
                        const float* xp = Xs + ((((g - i) + 4) & 3) * ld + (f + 2 - j - f0)) * 64;
                        const float x0 = xp[lane], x1 = xp[lane + 32];
#pragma unroll
                        for (int o = 0; o < 4; ++o) {
                            acc[o] = fmaf(wr[0][o * 9 + i * 3 + j], x0, acc[o]);
                            acc[o] = fmaf(wr[1][o * 9 + i * 3 + j], x1, acc[o]);
                        }
                    }
#pragma unroll
                for (int o = 0; o < 4; ++o) {
                    const float v = warp_sum(acc[o]);
                    if (lane == 0) Rg[(o >> 1) * NROW + (o & 1) * NF + f] = v + bd[o];
                }
            }
        };
        // prologue of the item: frames t0-3 .. t0 into the ring (those that exist: >= -2), then the spectrum of frame t0-1
        __syncthreads();                               // the previous item's readers of the ring and of R are done
        const int gfirst = max(t0 - 3, -2);
        for (int g = gfirst; g <= t0; ++g) stage(g);
        for (int g = gfirst; g < t0; ++g) wait_frame(g);
        if (t0 == 0) {                                 // the previous call's last spectrum (own bins)
            for (int i = tid; i < NSRC * 2 * nf; i += 256) {
                const int idx = (i / (2 * nf)) * NROW + ((i / nf) & 1) * NF + f0 + i % nf;
                R[NSRC * NROW + idx] = ib[idx];        // frame -1 -> slot (-1) & 1 = 1
            }
        } else {
            deconv(t0 - 1);
        }
        for (int t = t0; t < t1; ++t, ++nframe) {
            wait_frame(t);
            __syncthreads();                           // frame t-1's readers of frame t-3's slot are done; R[(t-1)&1] complete
            if (t + 1 < t1) stage(t + 1);              // into the slot of frame t-3
            deconv(t);
            if (t == Tb - 1 && live) {                 // next deconv tails: the row's last two frames (own bins)
                for (int i = tid; i < nf * 16; i += 256) {
                    const int r = i / 16, c4 = i % 16;
                    reinterpret_cast<float4*>(db_next + (f0 + r) * 64)[c4] =
                        reinterpret_cast<const float4*>(Xs + ((((t - 1) + 4) & 3) * ld + 1 + r) * 64)[c4];
                    reinterpret_cast<float4*>(db_next + FC + (f0 + r) * 64)[c4] =
                        reinterpret_cast<const float4*>(Xs + (((t + 4) & 3) * ld + 1 + r) * 64)[c4];
                }
            }
            __syncthreads();                           // R[t & 1] (own bins) complete
            float* wa = wacc + (nframe & 1u) * NSRC * NFFT;
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int it2 = tid + 256 * u;
                if (it2 < NSRC * NFFT) {
                    const int ear = it2 / NFFT, n = it2 % NFFT;
                    const float* rr = R + ((((n < HOP) ? t : t - 1) & 1) * NSRC + ear) * NROW + f0;
                    float acc = 0.f;
                    for (int ri = 0; ri < 2; ++ri) {
                        const float* wf = Wf + ri * nf * NFFT + n;
                        const float* rv = rr + ri * NF;
#pragma unroll 5
                        for (int r = 0; r < nf; ++r) acc = fmaf(rv[r], wf[r * NFFT], acc);
                    }
                    wa[it2] = acc;
                }
            }
            if (t == Tb - 1 && live)
                for (int i = tid; i < NSRC * 2 * nf; i += 256) {
                    const int idx = (i / (2 * nf)) * NROW + ((i / nf) & 1) * NF + f0 + i % nf;
                    ib_next[idx] = R[(t & 1) * NSRC * NROW + idx];
                }
            cluster.sync();                            // the four partial windows of frame t are complete and visible cluster-wide
            if (part == 0 && live) {                   // (wacc is double-buffered: the peers go on with the next frame meanwhile)
                for (int i = tid; i < NSRC * HOP; i += 256) {
                    const int ear = i / HOP, n = i % HOP;
                    const int s2 = HOP * t + n + soff;
                    if (s2 < yl) {
                        float v = 0.f, tail = 0.f;
#pragma unroll
                        for (int p = 0; p < BACK_CL; ++p) {
                            const float* pw = cluster.map_shared_rank(wa, p);
                            v += pw[ear * NFFT + n];
                            if (n < LOOKAHEAD) tail += pw[ear * NFFT + HOP + n];
                        }
                        if (n < LOOKAHEAD) v += tail;               // overlap-add of the previous frame's tail
                        y[(int64_t)b * y_bstride + (int64_t)ear * y_cstride + s2] = v;
                    }
                }
            }
        }
    }
    cluster.sync();                         // nobody leaves while CTA 0 may still read its shared memory
    finish_call(state, recs, n_streams, T, active);      // the last CTA to finish advances the clocks
}

// ------------------------------------------------------------------------------------------
// Tail of the attention output for calls with many rows, where the Linear(64->64) + PReLU ran as a tensor-core GEMM
// into P: LayerNorm over the frame's (F, C) = 6208 values + residual (+ the speaker gate after block 0)
// (tfgridnet_causal.py:583-588, :250-251).  Same arithmetic as the tail of attn_out_kernel.  grid (T, B), 256 threads.
template <class Map>
__global__ void __launch_bounds__(256)
ln_frame_res_kernel_t(const float* __restrict__ P, float* __restrict__ X, const float* __restrict__ state, Map recs,
                      BlockWeights w, int apply_gate, int T) {
    __shared__ float red[32];
    __shared__ __align__(16) float Ps[FC];
    const int t = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    griddep_launch();
    griddep_wait();
    const int64_t off = ((int64_t)b * T + t) * FC;
    float s = 0.f;
    for (int i = tid; i < FC / 4; i += 256) {
        const float4 v = reinterpret_cast<const float4*>(P + off)[i];
        reinterpret_cast<float4*>(Ps)[i] = v;
        s += (v.x + v.y) + (v.z + v.w);
    }
    const float mu = block_sum(s, red) * (1.f / FC);
    float q = 0.f;
    for (int i = tid; i < FC; i += 256) { const float d = Ps[i] - mu; q += d * d; }
    const float rs = rsqrtf(block_sum(q, red) * (1.f / FC) + 1e-5f);
    const float* gate = stream_rec(state, recs, b) + ST_GATE;
    float* xr = X + off;
    for (int i = tid; i < FC / 4; i += 256) {
        float4 x4 = reinterpret_cast<const float4*>(xr)[i];
        const float4 p4 = reinterpret_cast<const float4*>(Ps)[i];
        const float4 g4 = __ldg(reinterpret_cast<const float4*>(w.lnp_g) + i);
        const float4 b4 = __ldg(reinterpret_cast<const float4*>(w.lnp_b) + i);
        x4.x += (p4.x - mu) * rs * g4.x + b4.x; x4.y += (p4.y - mu) * rs * g4.y + b4.y;
        x4.z += (p4.z - mu) * rs * g4.z + b4.z; x4.w += (p4.w - mu) * rs * g4.w + b4.w;
        if (apply_gate) {
            const float4 gt = reinterpret_cast<const float4*>(gate)[i];
            x4.x *= gt.x; x4.y *= gt.y; x4.z *= gt.z; x4.w *= gt.w;
        }
        reinterpret_cast<float4*>(xr)[i] = x4;
    }
}

// ------------------------------------------------------------------------------------------
// One inter-LSTM step for many streams, cell part only (tfgridnet_causal.py:524-532 with T = 1): the gate
// pre-activations [rows][256] (column j*4+q, q in i,f,g,o; = LN(x) W_ih^T + h W_hh^T + b from ONE tensor-core GEMM
// over the concatenated k = [x | h]) and the carried cell state give the new (h, c), written back to the per-stream
// state records, and h again as contiguous rows for the Linear that follows.  One thread per (row, hidden unit).
template <class Map>
__global__ void __launch_bounds__(256)
lstm_cell_rows_kernel_t(const float* __restrict__ gates, float* __restrict__ state, Map recs, int blk, float* __restrict__ Hout,
                        int rows, const uint8_t* __restrict__ active) {
    griddep_launch();
    griddep_wait();
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= (int64_t)rows * 64) return;
    const int row = (int)(i >> 6), j = (int)(i & 63);
    const int b = row / NF, f = row % NF;
    const float4 g = *reinterpret_cast<const float4*>(gates + (int64_t)row * 256 + j * 4);
    float* base = stream_rec(state, recs, b) + ST_BLK + (int64_t)blk * BK_STRIDE;
    float* hp = base + BK_H + f * 64 + j;
    float* cp = base + BK_C + f * 64 + j;
    constexpr float LOG2E = 1.4426950408889634f;
    const float ig = __fdividef(1.f, 1.f + ex2_ftz(-LOG2E * g.x));
    const float fg = __fdividef(1.f, 1.f + ex2_ftz(-LOG2E * g.y));
    const float gg = __fdividef(2.f, 1.f + ex2_ftz(-2.f * LOG2E * g.z)) - 1.f;
    const float og = __fdividef(1.f, 1.f + ex2_ftz(-LOG2E * g.w));
    const float c = fg * *cp + ig * gg;
    const float h = og * (__fdividef(2.f, 1.f + ex2_ftz(-2.f * LOG2E * c)) - 1.f);
    if (stream_active(recs, active, b)) {
        *cp = c;
        *hp = h;
    }
    Hout[i] = h;
}

// Slot-list calls read the carried inter-LSTM state of their records through a base pointer and a stride in two places,
// and a slot list cannot be expressed that way: the one-hop tensor-core chain's inter-step GEMM (a strided tensor map over
// the records' h) and the recurrence over T of multi-hop calls (LstmArgs::h_state / c_state).  Once per call, before any
// block reads them, this copies the h (and, with Cg, the c) of every block of every row's record to Hg[blk][row][f][c]
// (Cg alike) for those to use instead.  One thread per float4.
__global__ void __launch_bounds__(256)
gather_h_kernel(const float* __restrict__ state, Records recs, int n_blocks, int n_streams, float* __restrict__ Hg,
                float* __restrict__ Cg) {
    constexpr int PER = FC / 4;                        // float4s of one block's h
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= (int64_t)n_blocks * n_streams * PER) return;
    const int k = (int)(i % PER), row = (int)(i / PER);
    const int b = row % n_streams, blk = row / n_streams;
    const float* h = stream_rec(state, recs, b) + ST_BLK + (int64_t)blk * BK_STRIDE + BK_H;
    reinterpret_cast<float4*>(Hg)[i] = reinterpret_cast<const float4*>(h)[k];
    if (Cg != nullptr) reinterpret_cast<float4*>(Cg)[i] = reinterpret_cast<const float4*>(h + (BK_C - BK_H))[k];
}

// Multi-hop slot-list calls: after the last block's recurrence, the new (h, c) that gather_h_kernel's copy carried through
// the call go back to the records of the rows that store (an entry outside the state stores nothing).  One thread per float4.
__global__ void __launch_bounds__(256)
scatter_hc_kernel(float* __restrict__ state, Records recs, int n_blocks, int n_streams, const float* __restrict__ Hg,
                  const float* __restrict__ Cg) {
    constexpr int PER = FC / 4;
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= (int64_t)n_blocks * n_streams * PER) return;
    const int k = (int)(i % PER), row = (int)(i / PER);
    const int b = row % n_streams, blk = row / n_streams;
    const RowRecord r = row_record(recs, nullptr, b);
    if (!r.stores) return;
    float* h = state + r.off + ST_BLK + (int64_t)blk * BK_STRIDE + BK_H;
    reinterpret_cast<float4*>(h)[k] = reinterpret_cast<const float4*>(Hg)[i];
    reinterpret_cast<float4*>(h + (BK_C - BK_H))[k] = reinterpret_cast<const float4*>(Cg)[i];
}

// Ragged slot-list calls (l2h_sep_forward_slots_hops), inter LSTM over T: the gate pre-activations GX [B][T][97][256]
// (column j*4 + q, q = i, f, g, o) of the frames t >= T_b a row does not advance become i = -inf, f = +inf, g = 0, so that
// the recurrence carries c through them unchanged (sigma(+inf) = 1, sigma(-inf) = 0) and ends with the c of frame T_b - 1.
// grid (T, B), 256 threads; CTAs of frames a row advances return at once.
__global__ void __launch_bounds__(256)
inter_gate_mask_kernel(float* __restrict__ gx, Records recs, int T) {
    const int t = blockIdx.x, b = blockIdx.y;
    if (t < row_frames(recs, b, T)) return;
    float* g = gx + ((int64_t)b * T + t) * NF * 256;
    for (int u = threadIdx.x; u < NF * 64; u += 256) {
        g[4 * u + 0] = -INFINITY;
        g[4 * u + 1] = INFINITY;
        g[4 * u + 2] = 0.f;
    }
}

// ... and its h: the recurrence ends with the h of frame T - 1, a row with 0 < T_b < T carries that of frame T_b - 1, which
// is its row of the recurrence's output Y [B][T][97][64].  That row goes into Hg [B][97][64] (the block's part of
// gather_h_kernel's copy) before Y is reused.  grid (B), 256 threads.
__global__ void __launch_bounds__(256)
inter_h_last_kernel(const float* __restrict__ Y, float* __restrict__ Hg, Records recs, int T) {
    const int b = blockIdx.x;
    const int Tb = row_frames(recs, b, T);
    if (Tb <= 0 || Tb >= T) return;
    const float4* src = reinterpret_cast<const float4*>(Y + ((int64_t)b * T + Tb - 1) * FC);
    float4* dst = reinterpret_cast<float4*>(Hg + (int64_t)b * FC);
    for (int i = threadIdx.x; i < FC / 4; i += 256) dst[i] = src[i];
}

// the dense forms (call row b = record b); the `_t<Records>` forms serve slot-list calls (l2h_sep_forward_slots)
constexpr auto front_kernel = front_kernel_t<int64_t>;
constexpr auto front_many_kernel = front_many_kernel_t<int64_t>;
constexpr auto qkv_kernel = qkv_kernel_t<int64_t>;
constexpr auto qkv_many_kernel = qkv_many_kernel_t<int64_t>;
constexpr auto attn_kernel = attn_kernel_t<int64_t>;
constexpr auto attn_cluster_kernel = attn_cluster_kernel_t<int64_t>;
constexpr auto attn_out_kernel = attn_out_kernel_t<int64_t>;
constexpr auto back_kernel = back_kernel_t<int64_t>;
constexpr auto back_many_kernel = back_many_kernel_t<int64_t>;
constexpr auto ln_frame_res_kernel = ln_frame_res_kernel_t<int64_t>;
constexpr auto lstm_cell_rows_kernel = lstm_cell_rows_kernel_t<int64_t>;
constexpr auto kv_gather_kernel = kv_gather_kernel_t<int64_t>;

}  // namespace l2h
