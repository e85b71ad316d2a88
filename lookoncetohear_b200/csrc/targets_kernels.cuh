// Kernels of the calls that extract several targets per mixture (l2h_sep_forward_targets, l2h_sep_forward_targets_groups,
// l2h_sep_forward_targets_rows).
// The front and block 0 do not depend on the speaker, so such a call runs them once per mixture, without the gate; the two
// kernels below then give each target row its own gated copy of block 0's output.  (Included after every other kernel
// header: defining them earlier in the module would move the code generated for kernels that do not use them.)
#pragma once
#include "sep_kernels.cuh"

namespace l2h {

// The speaker-gate memo of every target row: one CTA per row, as the extra CTA of front_kernel builds or validates it in a
// dense call.  grid (target rows), 256 threads.
template <class Map>
__global__ void __launch_bounds__(256)
spk_gate_kernel_t(const float* __restrict__ emb, float* __restrict__ spk_pre, float* __restrict__ state, Map recs, SepWeights w) {
    __shared__ __align__(16) float red[288];
    griddep_launch();
    griddep_wait();
    spk_gate_cta(emb, spk_pre, state, recs, w, (int)blockIdx.x, red, nullptr);
}

// X[r] = X0[i] * gate of target row r's record, elementwise over the [T][97][64] rows, where mixture i owns row r: block
// 0's output of mixture i becomes block 1's input for each of its targets.  The owner is r / n_targets (the dense targets
// call: owner == nullptr) or owner[r] (a call over listed rows, see target_lists_kernel); a row with no owner (-1) copies
// mixture 0's row ungated, so it stays finite, and stores nothing downstream.  The multiply is the one attn_out_kernel /
// ln_frame_res_kernel / tail_kernel apply with their gate flag (tfgridnet_causal.py:250-251); with one block the gate never
// applies (apply_gate = 0) and this is a plain copy.  X0 and X do not overlap.  grid (T, target rows), 256 threads.
template <class Map>
__global__ void __launch_bounds__(256)
gate_fanout_kernel_t(const float* __restrict__ X0, float* __restrict__ X, const float* __restrict__ state, Map recs,
                     const int32_t* __restrict__ owner, int n_targets, int T, int apply_gate) {
    griddep_launch();
    griddep_wait();
    const int t = blockIdx.x, r = blockIdx.y;
    const int i = owner == nullptr ? r / n_targets : __ldg(owner + r);
    const bool gated = apply_gate && i >= 0;
    const float4* src = reinterpret_cast<const float4*>(X0 + ((int64_t)max(i, 0) * T + t) * FC);
    float4* dst = reinterpret_cast<float4*>(X + ((int64_t)r * T + t) * FC);
    const float4* gate = reinterpret_cast<const float4*>(stream_rec(state, recs, r) + ST_GATE);
    for (int j = threadIdx.x; j < FC / 4; j += 256) {
        float4 v = src[j];
        if (gated) {
            const float4 g = gate[j];
            v.x *= g.x; v.y *= g.y; v.z *= g.z; v.w *= g.w;
        }
        dst[j] = v;
    }
}

// The lists of a call over a state's listeners, built at the start of the call before any kernel reads them.  Call row i
// (a listener, one mixture) owns the target rows start[i] .. start[i+1]-1:
//   l2h_sep_forward_targets_rows:   start[i] = offsets[i], clamped here to be non-decreasing and <= rows (a bad list gives
//                                   empty listeners, never a read out of bounds); target row r is record records[r]
//   l2h_sep_forward_targets_groups: start[i] = i*K (offsets == nullptr); target row i*K + k is record groups[i]*K + k, or
//                                   -1 for a group outside [0, batch / K)
// Written: rec[rows], the target rows' records (-1: the row stores nothing); rec_hops[rows] with `hops`, the frames each
// advances (its listener's count, 0 for no listener); owner[rows], the call row that owns each target row (-1: none, the
// rows from start[n] on); lead[n], each listener's lead record, the record of its first target row, which holds its conv
// tails and block 0 (-1: no target row, or a lead outside the state, and then none of the listener's rows stores);
// start[n + 1] with offsets.  One CTA of 1024 threads.
__device__ __forceinline__ int listed_record(const int32_t* records, const int32_t* groups, int K, int batch, int i, int r,
                                             int first) {
    if (records == nullptr) {
        const int g = __ldg(groups + i);
        return (unsigned)g < (unsigned)(batch / K) ? g * K + (r - first) : -1;
    }
    const int s = __ldg(records + r);
    return (unsigned)s < (unsigned)batch ? s : -1;
}
__global__ void __launch_bounds__(1024)
target_lists_kernel(const int32_t* __restrict__ records, const int32_t* __restrict__ offsets, const int32_t* __restrict__ groups,
                    const int32_t* __restrict__ hops, int n, int K, int rows, int batch, int32_t* __restrict__ rec,
                    int32_t* __restrict__ rec_hops, int32_t* __restrict__ owner, int32_t* __restrict__ lead, int32_t* start) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (offsets != nullptr) {      // start = the running maximum of the offsets clamped to [0, rows], 1024 entries per pass
        __shared__ int wmax[32];
        __shared__ int carry;
        if (tid == 0) carry = 0;
        __syncthreads();
        for (int base = 0; base <= n; base += 1024) {
            const int i = base + tid;
            int v = i <= n ? min(max(__ldg(offsets + i), 0), rows) : 0;
            for (int d = 1; d < 32; d <<= 1) {
                const int u = __shfl_up_sync(0xffffffffu, v, d);
                if (lane >= d) v = max(v, u);
            }
            if (lane == 31) wmax[warp] = v;
            __syncthreads();
            if (warp == 0) {
                int w = wmax[lane];
                for (int d = 1; d < 32; d <<= 1) {
                    const int u = __shfl_up_sync(0xffffffffu, w, d);
                    if (lane >= d) w = max(w, u);
                }
                wmax[lane] = w;
            }
            __syncthreads();
            if (warp > 0) v = max(v, wmax[warp - 1]);
            v = max(v, carry);
            if (i <= n) start[i] = v;
            __syncthreads();
            if (tid == 1023) carry = v;
            __syncthreads();
        }
    }
    const auto first = [&](int i) { return offsets != nullptr ? start[i] : i * K; };
    const auto lead_of = [&](int i) {
        const int f = first(i);
        return f < first(i + 1) ? listed_record(records, groups, K, batch, i, f, f) : -1;
    };
    for (int i = tid; i < n; i += 1024) lead[i] = lead_of(i);
    for (int r = tid; r < rows; r += 1024) {
        int i;      // the listener whose rows hold r: the last i with start[i] <= r, if i < n
        if (offsets != nullptr) {
            int lo = 0, hi = n + 1;      // the count of start[0 .. n] <= r
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (start[mid] <= r) lo = mid + 1; else hi = mid;
            }
            i = lo - 1 < n ? lo - 1 : -1;
        } else {
            i = r / K < n ? r / K : -1;
        }
        owner[r] = i;
        rec[r] = i >= 0 && lead_of(i) >= 0 ? listed_record(records, groups, K, batch, i, r, first(i)) : -1;
        if (hops != nullptr) rec_hops[r] = i >= 0 ? __ldg(hops + i) : 0;
    }
}

constexpr auto spk_gate_kernel = spk_gate_kernel_t<int64_t>;
constexpr auto gate_fanout_kernel = gate_fanout_kernel_t<int64_t>;

// Launchers of the kernels above, shared by the engine (sep_engine.cu) and the kernel tests (tests/kernels/
// kernel_harness.cu), in the convention of sep_launch.cuh.
// spk_gate_kernel: one CTA per target row
template <class Map>
inline cudaError_t launch_spk_gate(bool pdl, cudaStream_t st, int rows, const float* emb, float* spk_pre, float* state, Map recs,
                                   const SepWeights& w) {
    return launch_k(pdl, spk_gate_kernel_t<Map>, dim3(rows), dim3(256), 0, st, emb, spk_pre, state, recs, w);
}
// gate_fanout_kernel: grid (T, target rows)
template <class Map>
inline cudaError_t launch_gate_fanout(bool pdl, cudaStream_t st, int rows, const float* X0, float* X, const float* state, Map recs,
                                      const int32_t* owner, int n_targets, int T, int apply_gate) {
    return launch_k(pdl, gate_fanout_kernel_t<Map>, dim3(T, rows), dim3(256), 0, st, X0, X, state, recs, owner, n_targets, T,
                    apply_gate);
}
// target_lists_kernel: one CTA of 1024 threads.  `lists` is the call's int32 buffer of 5 rows + 1 entries (rows >= n):
// rec [rows], rec_hops [rows], owner [rows], lead [n] at 3 rows, start [n + 1] at 4 rows.
inline cudaError_t launch_target_lists(cudaStream_t st, const int32_t* records, const int32_t* offsets, const int32_t* groups,
                                       const int32_t* hops, int n, int K, int rows, int batch, int32_t* lists) {
    const int64_t R = rows;
    return launch_k(false, target_lists_kernel, dim3(1), dim3(1024), 0, st, records, offsets, groups, hops, n, K, rows, batch, lists,
                    lists + R, lists + 2 * R, lists + 3 * R, lists + 4 * R);
}

// ---- adding and dropping the targets of a running listener (l2h_sep_forward_targets_rows_history, l2h_sep_join_targets,
// l2h_sep_state_move_lead) ---------------------------------------------------------------------------------------------
// A block-0 history is [state batch][F][97*64] fp32, keyed by record: the ring of the last F frames of block 0's ungated
// output of a lead record, frame n of the record's own clock in slot n mod F.

// Rows tick: listener i's last min(h_i, F) frames of block 0's output X0 [M][T][97][64] (frames h_i - F <= t < h_i) go into
// the ring of its lead record, at the lead's clock from before the call: no two CTAs write one slot, and a tick of more
// frames than the ring holds leaves its last F.  `lead` is the map of block 0's rows (the lead list and the listeners'
// hop counts): a listener that stores nothing writes nothing.  grid (T, M), 256 threads.
__global__ void __launch_bounds__(256)
history_put_kernel(const float* __restrict__ X0, const float* __restrict__ state, Records lead, float* __restrict__ hist, int F,
                   int T) {
    griddep_launch();
    griddep_wait();
    const int t = blockIdx.x, i = blockIdx.y;
    const RowRecord r = row_record(lead, nullptr, i);
    const int h = row_frames(lead, i, T);
    if (!r.stores || t >= h || t + F < h) return;
    const long long fr = rec_pos(state + r.off) + t;
    const float4* src = reinterpret_cast<const float4*>(X0 + ((int64_t)i * T + t) * FC);
    float4* dst = reinterpret_cast<float4*>(hist + ((int64_t)__ldg(lead.slots + i) * F + (int)(fr % F)) * FC);
    for (int j = threadIdx.x; j < FC / 4; j += 256) dst[j] = src[j];
}

// Join, first kernel: row j is live when records[j] and leads[j] both lie in [0, batch), and records[j] is neither another
// row's record nor any row's lead (such rows would race with each other; they store nothing).  Its record becomes a fresh record,
// as reset_streams_kernel leaves it, except for its clock: p - W_j, where p is the clock of leads[j] and W_j = min(w_max, p)
// the frames the row replays.  CTA 0 of each row also writes the row's entries of the call's lists: rec[j] (the record, -1
// for a row that is not live), used[j] = W_j (0 if not live), owner[j] (j, -1 if not live), and used_out[j] if given.
// grid (any, J), 256 threads.
static_assert(ST_GEN % 4 == 0 && ST_CALLS == ST_GEN + 1 && ST_POS == ST_GEN + 2, "one float4 holds the memo generation and clock");
__global__ void __launch_bounds__(256)
join_start_kernel(float* __restrict__ state, int64_t ss, int batch, const int32_t* __restrict__ records,
                  const int32_t* __restrict__ leads, int w_max, int32_t* __restrict__ rec, int32_t* __restrict__ used,
                  int32_t* __restrict__ owner, int32_t* __restrict__ used_out, int J) {
    const int j = blockIdx.y;
    const int s = __ldg(records + j), l = __ldg(leads + j);
    bool clash = false;
    for (int k = threadIdx.x; k < J; k += blockDim.x) clash |= (k != j && __ldg(records + k) == s) || __ldg(leads + k) == s;
    const bool live = !__syncthreads_or(clash) && (unsigned)s < (unsigned)batch && (unsigned)l < (unsigned)batch;
    const long long p = live ? rec_pos(stream_rec(state, ss, l)) : 0;
    const int W = (int)min((long long)w_max, p);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        rec[j] = live ? s : -1;
        used[j] = live ? W : 0;
        owner[j] = live ? j : -1;
        if (used_out != nullptr) used_out[j] = live ? W : 0;
    }
    if (!live) return;
    float4* r = reinterpret_cast<float4*>(stream_rec(state, ss, s));
    const long long start = p - W;
    const float nan = __int_as_float(0x7fc00000);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ss / 4; i += (int64_t)gridDim.x * blockDim.x)
        r[i] = i < SPK / 4 ? make_float4(nan, nan, nan, nan)
             : i == ST_GEN / 4 ? make_float4(0.f, 0.f, __int_as_float((int)(start & 0xffffffffLL)), __int_as_float((int)(start >> 32)))
                               : make_float4(0.f, 0.f, 0.f, 0.f);
}

// Join, the replayed frames: X0[j][t] = frame (clock of record j) + t of the ring of leads[j], for t < used[j]; the other
// frames (and rows that are not live) are zero.  `recs` is the join's row map (rec, used).  grid (T, J), 256 threads.
__global__ void __launch_bounds__(256)
history_get_kernel(const float* __restrict__ hist, int F, const float* __restrict__ state, Records recs,
                   const int32_t* __restrict__ leads, float* __restrict__ X0, int T) {
    griddep_launch();
    griddep_wait();
    const int t = blockIdx.x, j = blockIdx.y;
    const RowRecord r = row_record(recs, nullptr, j);
    float4* dst = reinterpret_cast<float4*>(X0 + ((int64_t)j * T + t) * FC);
    if (!r.stores || t >= row_frames(recs, j, T)) {
        for (int i = threadIdx.x; i < FC / 4; i += 256) dst[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        return;
    }
    const long long fr = rec_pos(state + r.off) + t;
    const float4* src = reinterpret_cast<const float4*>(hist + ((int64_t)__ldg(leads + j) * F + (int)(fr % F)) * FC);
    for (int i = threadIdx.x; i < FC / 4; i += 256) dst[i] = src[i];
}

// l2h_sep_state_move_lead: the speaker-independent part of record olds[i] goes to record news[i]: block 0 (K/V rings and
// (h, c)) whole, and the current copy of the conv tails (parity of olds[i]'s calls) into the copy news[i]'s parity makes
// current.  Nothing else of news[i] changes.  grid (any, n), 256 threads.
constexpr int MOVE_MAX_PAIRS = RESET_MAX_SLOTS / 2;      // the kernel parameters stay under 4 KB
struct PairList { int32_t from[MOVE_MAX_PAIRS], to[MOVE_MAX_PAIRS]; };
__global__ void __launch_bounds__(256)
move_lead_kernel(float* __restrict__ state, int64_t ss, PairList pairs) {
    constexpr int64_t CONV = 2 * 4 * NF;                   // one parity of the conv tails
    static_assert(CONV % 4 == 0, "float4 copies");
    const float* src = stream_rec(state, ss, pairs.from[blockIdx.y]);
    float* dst = stream_rec(state, ss, pairs.to[blockIdx.y]);
    const float4* s0 = reinterpret_cast<const float4*>(src + ST_BLK);
    float4* d0 = reinterpret_cast<float4*>(dst + ST_BLK);
    const float4* sc = reinterpret_cast<const float4*>(src + ST_CONV + rec_par(src) * CONV);
    float4* dc = reinterpret_cast<float4*>(dst + ST_CONV + rec_par(dst) * CONV);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < BK_STRIDE / 4 + CONV / 4; i += (int64_t)gridDim.x * blockDim.x) {
        if (i < BK_STRIDE / 4) d0[i] = s0[i];
        else dc[i - BK_STRIDE / 4] = sc[i - BK_STRIDE / 4];
    }
}

// move_lead_kernel over the host pairs from[i] -> to[i], i < n: one launch per MOVE_MAX_PAIRS of them, each of ~2 CTAs per
// SM over all its pairs, as reset_streams
inline cudaError_t launch_move_lead(cudaStream_t st, float* state, int64_t ss, const int32_t* from, const int32_t* to, int n) {
    for (int i0 = 0; i0 < n; i0 += MOVE_MAX_PAIRS) {
        const int k = std::min(MOVE_MAX_PAIRS, n - i0);
        PairList pl{};
        std::copy(from + i0, from + i0 + k, pl.from);
        std::copy(to + i0, to + i0 + k, pl.to);
        const unsigned per_rec = (unsigned)std::max(1, 2 * NUM_SMS / k);
        if (cudaError_t e = launch_k(false, move_lead_kernel, dim3(per_rec, k), dim3(256), 0, st, state, ss, pl)) return e;
    }
    return cudaSuccess;
}
inline cudaError_t launch_history_put(bool pdl, cudaStream_t st, int M, const float* X0, const float* state, Records lead, float* hist,
                                      int F, int T) {
    return launch_k(pdl, history_put_kernel, dim3(T, M), dim3(256), 0, st, X0, state, lead, hist, F, T);
}
inline cudaError_t launch_join_start(cudaStream_t st, int J, float* state, int64_t ss, int batch, const int32_t* records,
                                     const int32_t* leads, int w_max, int32_t* lists, int32_t* used_out) {
    const int64_t R = J;
    const unsigned per_rec = (unsigned)std::max(1, 2 * NUM_SMS / J);      // as reset_streams: ~2 CTAs per SM over all records
    return launch_k(false, join_start_kernel, dim3(per_rec, J), dim3(256), 0, st, state, ss, batch, records, leads, w_max, lists,
                    lists + R, lists + 2 * R, used_out, J);
}
inline cudaError_t launch_history_get(bool pdl, cudaStream_t st, int J, const float* hist, int F, const float* state, Records recs,
                                      const int32_t* leads, float* X0, int T) {
    return launch_k(pdl, history_get_kernel, dim3(T, J), dim3(256), 0, st, hist, F, state, recs, leads, X0, T);
}

}  // namespace l2h
