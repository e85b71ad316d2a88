// On-GPU evaluation epilogue (SURVEY.md section 8 f-2): the three per-mixture figures the reference's evaluation
// driver computes on the CPU after `outputs.cpu()` -- reference src/ts_hear_test.py:139-146 --
//   output_sisnr  = mean over ears of SI-SNR(estimate, target)
//   si_snr_i      = mean over ears of SI-SNR(estimate, target) - SI-SNR(mixture, target)
//   embedding_sim = cosine_similarity(embedding, embedding_gt)
// so that the device->host traffic of an evaluation step shrinks from the separated audio to three floats per mixture.
// SI-SNR as torchmetrics' scale_invariant_signal_noise_ratio, in its order and all in double, per channel row:
//   1. the means of estimate, target (and mixture);
//   2. the centred sums <p~,t~>, <t~,t~> and alpha = (<p~,t~>+eps)/(<t~,t~>+eps);
//   3. the residual energy |alpha t~ - p~|^2 summed directly;
// then 10 log10((alpha^2 <t~,t~>+eps)/(|alpha t~ - p~|^2+eps)), eps = float32 eps.  Three passes over the row instead of
// one-pass raw sums: spt - sp st / n and friends cancel catastrophically once the signals carry a DC offset.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>

#include "../../include/lookonce_b200.h"
#include "host_errors.h"

namespace l2h {

__device__ __forceinline__ double blk_sum(double v, double* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = (threadIdx.x & 31) < (blockDim.x >> 5) ? red[threadIdx.x & 31] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    return t;
}

constexpr double SI_EPS = 1.1920928955078125e-07;          // torch.finfo(torch.float32).eps

__device__ __forceinline__ double si_snr_db(double sig, double noise) {
    return 10.0 * log10((sig + SI_EPS) / (noise + SI_EPS));
}

// one CTA per mixture; 256 threads
__global__ void __launch_bounds__(256)
eval_metrics_kernel(const float* __restrict__ est, const float* __restrict__ tgt, const float* __restrict__ mix, int ch, int n,
                    const float* __restrict__ emb, const float* __restrict__ emb_gt, int dim, float* __restrict__ out) {
    __shared__ double red[32];
    const int b = blockIdx.x, tid = threadIdx.x;
    double acc_s = 0.0, acc_i = 0.0;
    for (int c = 0; c < ch; ++c) {
        const int64_t off = ((int64_t)b * ch + c) * n;
        const float *p = est + off, *t = tgt + off, *m = mix ? mix + off : nullptr;
        double sp = 0, st = 0, sm = 0;
        for (int i = tid; i < n; i += 256) {
            sp += p[i]; st += t[i];
            if (m) sm += m[i];
        }
        const double mp = blk_sum(sp, red) / n, mt = blk_sum(st, red) / n, mm = m ? blk_sum(sm, red) / n : 0.0;
        double spt = 0, stt = 0, smt = 0;
        for (int i = tid; i < n; i += 256) {
            const double tc = t[i] - mt;
            spt += (p[i] - mp) * tc; stt += tc * tc;
            if (m) smt += (m[i] - mm) * tc;
        }
        const double tt = blk_sum(stt, red);
        const double ap = (blk_sum(spt, red) + SI_EPS) / (tt + SI_EPS);
        const double am = m ? (blk_sum(smt, red) + SI_EPS) / (tt + SI_EPS) : 0.0;
        double rp = 0, rm = 0;
        for (int i = tid; i < n; i += 256) {
            const double tc = t[i] - mt;
            const double ep = ap * tc - (p[i] - mp);
            rp += ep * ep;
            if (m) { const double em = am * tc - (m[i] - mm); rm += em * em; }
        }
        const double s_est = si_snr_db(ap * ap * tt, blk_sum(rp, red));
        acc_s += s_est;
        if (m) acc_i += s_est - si_snr_db(am * am * tt, blk_sum(rm, red));
    }
    double cs = 0.0;
    if (emb && emb_gt) {
        double xy = 0, xx = 0, yy = 0;
        for (int i = tid; i < dim; i += 256) {
            const double x = emb[(int64_t)b * dim + i], y = emb_gt[(int64_t)b * dim + i];
            xy += x * y; xx += x * x; yy += y * y;
        }
        xy = blk_sum(xy, red); xx = blk_sum(xx, red); yy = blk_sum(yy, red);
        cs = xy / (fmax(sqrt(xx), 1e-8) * fmax(sqrt(yy), 1e-8));       // F.cosine_similarity, eps = 1e-8
    }
    if (tid == 0) {
        out[b * 3 + 0] = (float)(acc_s / ch);
        out[b * 3 + 1] = (float)(acc_i / ch);
        out[b * 3 + 2] = (float)cs;
    }
}
}  // namespace l2h

extern "C" int l2h_eval_metrics(const float* est_dev, const float* target_dev, const float* mixture_dev, int32_t batch, int32_t channels,
                                int32_t n_samples, const float* emb_dev, const float* emb_gt_dev, int32_t emb_dim, float* out_dev,
                                void* stream) {
    using namespace l2h;
    if (!est_dev || !target_dev || !out_dev || batch <= 0 || channels <= 0 || n_samples <= 1)
        return fail(1, "l2h_eval_metrics: bad argument");
    eval_metrics_kernel<<<batch, 256, 0, static_cast<cudaStream_t>(stream)>>>(est_dev, target_dev, mixture_dev, channels, n_samples,
                                                                                emb_dev, emb_gt_dev, emb_dim, out_dev);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(3, std::string("eval_metrics_kernel: ") + cudaGetErrorString(e));
    return 0;
}
