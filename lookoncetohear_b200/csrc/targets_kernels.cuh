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

}  // namespace l2h
