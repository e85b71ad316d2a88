// Kernels of the calls that extract several targets per mixture (l2h_sep_forward_targets, l2h_sep_forward_targets_groups).
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

// X[i*K + k] = X0[i] * gate of target row i*K + k's record, elementwise over the [T][97][64] rows: block 0's output of
// mixture i becomes block 1's input for each of its K targets.  The multiply is the one attn_out_kernel /
// ln_frame_res_kernel / tail_kernel apply with their gate flag (tfgridnet_causal.py:250-251); with one block the gate never
// applies (apply_gate = 0) and this is a plain copy.  X0 and X do not overlap.  grid (T, target rows), 256 threads.
template <class Map>
__global__ void __launch_bounds__(256)
gate_fanout_kernel_t(const float* __restrict__ X0, float* __restrict__ X, const float* __restrict__ state, Map recs,
                     int n_targets, int T, int apply_gate) {
    griddep_launch();
    griddep_wait();
    const int t = blockIdx.x, r = blockIdx.y;
    const float4* src = reinterpret_cast<const float4*>(X0 + ((int64_t)(r / n_targets) * T + t) * FC);
    float4* dst = reinterpret_cast<float4*>(X + ((int64_t)r * T + t) * FC);
    const float4* gate = reinterpret_cast<const float4*>(stream_rec(state, recs, r) + ST_GATE);
    for (int i = threadIdx.x; i < FC / 4; i += 256) {
        float4 v = src[i];
        if (apply_gate) {
            const float4 g = gate[i];
            v.x *= g.x; v.y *= g.y; v.z *= g.z; v.w *= g.w;
        }
        dst[i] = v;
    }
}

// A call over a list of a state's groups (l2h_sep_forward_targets_groups): call row i is group groups[i], whose K records
// g*K .. g*K + K-1 are its targets.  The front and block 0 address the lead records through the group list itself (record
// stride K * stride); this builds the record list of the K*n target rows, and with `hops` their hop list, for everything
// after block 0.  Target row i*K + k is record groups[i]*K + k and advances hops[i] frames; a group outside [0, n_groups)
// gives -1, a record outside the state: its K rows store nothing.  One thread per target row.
__global__ void __launch_bounds__(256)
group_rows_kernel(const int32_t* __restrict__ groups, const int32_t* __restrict__ hops, int n_groups, int n_targets, int rows,
                  int32_t* __restrict__ rec, int32_t* __restrict__ rec_hops) {
    const int r = (int)blockIdx.x * 256 + threadIdx.x;
    if (r >= rows) return;
    const int i = r / n_targets;
    const int g = __ldg(groups + i);
    rec[r] = (unsigned)g < (unsigned)n_groups ? g * n_targets + r % n_targets : -1;
    if (hops != nullptr) rec_hops[r] = __ldg(hops + i);
}

constexpr auto spk_gate_kernel = spk_gate_kernel_t<int64_t>;
constexpr auto gate_fanout_kernel = gate_fanout_kernel_t<int64_t>;

}  // namespace l2h
