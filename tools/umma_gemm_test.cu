// Standalone correctness + throughput harness for csrc/umma_gemm.cuh (wgmma / tensor-map TMA GEMM).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -o tools/umma_gemm_test tools/umma_gemm_test.cu lookoncetohear_b200/csrc/umma_gemm.cu
// Every case is checked against a double-precision CPU product of the same fp32 inputs.
#include <cuda_runtime.h>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>
#include "../lookoncetohear_b200/csrc/umma_host.cuh"

using namespace l2h;
using namespace l2h::umma;

#define CKC(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(2); } } while (0)

static std::mt19937 rng(1234);
static std::vector<float> randv(size_t n, float sc = 1.f, bool small_int = false) {
    std::vector<float> v(n);
    static unsigned long long st = 0x9E3779B97F4A7C15ull;
    for (auto& x : v) {
        st ^= st << 13; st ^= st >> 7; st ^= st << 17;
        if (small_int) x = (float)((int)((st >> 20) % 9) - 4);
        else x = sc * 1.7320508f * ((float)((st >> 11) & 0xFFFFFF) / 8388608.f - 1.f);     // uniform, unit variance * sc
    }
    return v;
}
template <class T> static T* dcopy(const std::vector<T>& h) {
    T* d; CKC(cudaMalloc(&d, h.size() * sizeof(T) + 256)); CKC(cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice)); return d;
}

struct Case {
    const char* name;
    // A: [nseq][Ls][C] fp32; row (seq, p) uses window positions p+dp+pos_bias, channels all C, w taps => K = w*C
    int nseq, Ls, C, w, rows_per_seq, pos_bias;
    int N; int passes; bool ln; bool bias; bool prelu_vec; bool res; bool small_int; float alpha;
    bool b_by_seq; bool mn_major; bool two_src; int n_inner;   // n_inner: split seq into (inner, outer) for the tensor map
};

static int run_case(const Case& c, bool timing = false) {
    const int K = c.w * c.C * (c.two_src ? 2 : 1);
    const int nz = c.b_by_seq ? c.nseq : 1;
    std::vector<float> A = randv((size_t)c.nseq * c.Ls * c.C, 1.f, c.small_int);
    std::vector<float> A1 = c.two_src ? randv((size_t)c.nseq * c.Ls * c.C, 1.f, c.small_int) : std::vector<float>(4);
    std::vector<float> W = randv((size_t)nz * c.N * K, c.small_int ? 1.f : 0.2f, c.small_int);   // [z][N][K]
    std::vector<float> bias = randv(c.N), slopes = randv(c.N, 0.3f), g = randv(64), bt = randv(64);
    const int64_t Mrows = (int64_t)c.nseq * c.rows_per_seq;
    std::vector<float> R = c.res ? randv((size_t)Mrows * c.N) : std::vector<float>(4);
    float *dA = dcopy(A), *dA1 = dcopy(A1), *dW = dcopy(W), *dbias = dcopy(bias), *dsl = dcopy(slopes), *dg = dcopy(g), *dbt = dcopy(bt), *dR = dcopy(R);
    float* dC; CKC(cudaMalloc(&dC, (size_t)Mrows * c.N * sizeof(float))); CKC(cudaMemset(dC, 0xff, (size_t)Mrows * c.N * sizeof(float)));
    // B planes
    const int64_t ldb = c.mn_major ? ((c.N + 7) & ~7) : ((K + 7) & ~7);
    const int64_t brows = c.mn_major ? K : c.N;
    const int64_t zs = brows * ldb, ps = zs * nz;
    __nv_bfloat16* dB; CKC(cudaMalloc(&dB, 2 * ps * sizeof(__nv_bfloat16))); CKC(cudaMemset(dB, 0, 2 * ps * sizeof(__nv_bfloat16)));
    for (int z = 0; z < nz; ++z) {
        const float* src = dW + (size_t)z * c.N * K;
        if (!c.mn_major) CKC(split_planes(src, K, 1, c.N, K, ldb, dB + z * zs, dB + ps + z * zs, 0));
        else CKC(split_planes(src, 1, K, K, c.N, ldb, dB + z * zs, dB + ps + z * zs, 0));     // [k][n] = W[n][k]
    }
    GemmDesc d;
    const int n_inner = c.n_inner > 0 ? c.n_inner : c.nseq;
    d.a0.base = dA; d.a0.channels = c.C; d.a0.n_pos = c.Ls; d.a0.pos_stride = c.C;
    d.a0.n_inner = n_inner; d.a0.inner_stride = (int64_t)c.Ls * c.C; d.a0.n_outer = c.nseq / n_inner; d.a0.outer_stride = (int64_t)n_inner * c.Ls * c.C;
    if (c.two_src) { d.a1 = d.a0; d.a1.base = dA1; }
    set_window_chunks(d, c.C, c.w, c.ln);
    if (c.two_src) {
        const int n0 = d.n_chunks;
        for (int j = 0; j < n0; ++j) { d.chunks[n0 + j] = d.chunks[j]; d.chunks[n0 + j].flags = 1; }    // second source, no LN
        d.n_chunks = 2 * n0;
    }
    if (c.C % 64 != 0) { set_plain_chunks(d, c.C, false); }     // single tap, ragged K (zero fill)
    d.rows_per_seq = c.rows_per_seq; d.nseq = c.nseq; d.pos_bias = c.pos_bias;
    d.b.base = dB; d.b.ld = ldb; d.b.z_stride = zs; d.b.plane_stride = ps; d.b.nz = nz; d.b.mn_major = c.mn_major; d.b_by_seq = c.b_by_seq;
    d.N = c.N; d.K = K; d.passes = c.passes;
    d.C = dC; d.ldc = c.N; d.c_seq_stride = (int64_t)c.rows_per_seq * c.N;
    if (c.res) d.R = dR;
    if (c.bias) d.bias = dbias;
    if (c.prelu_vec) d.prelu_vec = dsl;
    if (c.ln) { d.ln_g = dg; d.ln_b = dbt; }
    d.alpha = c.alpha;
    std::string why;
    cudaError_t e = launch(d, 0, &why);
    if (e != cudaSuccess) { printf("[%s] launch failed: %s (%s)\n", c.name, cudaGetErrorString(e), why.c_str()); return 1; }
    e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { printf("[%s] kernel failed: %s\n", c.name, cudaGetErrorString(e)); exit(3); }
    if (timing) {
        cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
        for (int i = 0; i < 3; ++i) launch(d, 0);
        cudaEventRecord(e0);
        const int reps = 10;
        for (int i = 0; i < reps; ++i) launch(d, 0);
        cudaEventRecord(e1); CKC(cudaEventSynchronize(e1));
        float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= reps;
        const double fl = 2.0 * (double)Mrows * c.N * K;
        const double bytes = (double)Mrows * (c.C * (c.two_src ? 2 : 1) + c.N) * 4.0;
        printf("[%s] M=%lld N=%d K=%d passes=%d: %.1f us  %.1f TFLOP/s (x%d MMA passes = %.1f bf16 TF/s)  %.0f GB/s (A once + C)\n", c.name,
               (long long)Mrows, c.N, K, c.passes, ms * 1e3, fl / ms * 1e-9, c.passes, c.passes * fl / ms * 1e-9, bytes / ms * 1e-6);
    }
    std::vector<float> Cg((size_t)Mrows * c.N);
    CKC(cudaMemcpy(Cg.data(), dC, Cg.size() * sizeof(float), cudaMemcpyDeviceToHost));
    // CPU reference on a sample of rows
    double num = 0, den = 0, maxabs = 0; int bad = 0;
    const int64_t step = std::max<int64_t>(1, Mrows / 600);
    std::vector<double> a(K);
    for (int64_t m = 0; m < Mrows; m += step) {
        const int seq = (int)(m / c.rows_per_seq), p = (int)(m % c.rows_per_seq);
        for (int src = 0; src < (c.two_src ? 2 : 1); ++src) {
            const std::vector<float>& AA = src ? A1 : A;
            for (int t = 0; t < c.w; ++t) {
                const int pos = p + t + c.pos_bias;
                double mu = 0, var = 0;
                std::vector<double> row(c.C, 0.0);
                if (pos >= 0 && pos < c.Ls)
                    for (int ch = 0; ch < c.C; ++ch) row[ch] = AA[((size_t)seq * c.Ls + pos) * c.C + ch];
                if (c.ln && src == 0) {
                    for (int ch = 0; ch < c.C; ++ch) mu += row[ch];
                    mu /= c.C;
                    for (int ch = 0; ch < c.C; ++ch) var += (row[ch] - mu) * (row[ch] - mu);
                    var /= c.C;
                    for (int ch = 0; ch < c.C; ++ch) row[ch] = (row[ch] - mu) / std::sqrt(var + 1e-5) * g[ch] + bt[ch];
                }
                for (int ch = 0; ch < c.C; ++ch) a[(size_t)src * c.w * c.C + t * c.C + ch] = row[ch];
            }
        }
        const float* Wz = W.data() + (size_t)(c.b_by_seq ? seq : 0) * c.N * K;
        for (int n = 0; n < c.N; ++n) {
            double s = 0;
            for (int k = 0; k < K; ++k) s += a[k] * (double)Wz[(size_t)n * K + k];
            s *= c.alpha;
            if (c.bias) s += bias[n];
            if (c.prelu_vec) s = s >= 0 ? s : s * slopes[n];
            if (c.res) s += R[(size_t)m * c.N + n];
            const double got = Cg[(size_t)m * c.N + n];
            const double df = got - s;
            if (!(std::fabs(df) <= 1e30)) { if (bad < 3) printf("   non-finite at m=%lld n=%d: %f\n", (long long)m, n, got); ++bad; continue; }
            num += df * df; den += s * s; maxabs = std::max(maxabs, std::fabs(df));
        }
    }
    const double rel = std::sqrt(num / std::max(den, 1e-30));
    const double tol = c.small_int ? 1e-6 : (c.passes == 3 ? 5e-5 : (c.passes == 2 ? 8e-3 : 2e-2));
    const bool ok = bad == 0 && rel <= tol;
    printf("[%s] rel-L2 %.3e  max-abs %.3e  non-finite %d  -> %s\n", c.name, rel, maxabs, bad, ok ? "OK" : "FAIL");
    cudaFree(dA); cudaFree(dA1); cudaFree(dW); cudaFree(dbias); cudaFree(dsl); cudaFree(dg); cudaFree(dbt); cudaFree(dR); cudaFree(dC); cudaFree(dB);
    return ok ? 0 : 1;
}

int main(int argc, char** argv) {
    const bool perf = argc > 1 && atoi(argv[1]) != 0;
    const char* only = argc > 2 ? argv[2] : nullptr;      // run only the cases whose name contains this
    int fails = 0;
    //            name                  nseq  Ls    C   w  rows  pb   N   ps  ln    bias  pvec  res   int   alpha bseq  mn    two   inner
    const Case cases[] = {
        {"exact_k64_n64_p1",            1,  1000,  64, 1, 1000, 0,   64, 1, false, false, false, false, true,  1.f, false, false, false, 0},
        {"exact_k64_n64_p3",            1,  1000,  64, 1, 1000, 0,   64, 3, false, false, false, false, true,  1.f, false, false, false, 0},
        {"rand_k64_n64_p3",             1,  1000,  64, 1, 1000, 0,   64, 3, false, false, false, false, false, 1.f, false, false, false, 0},
        {"rand_k64_n64_p1",             1,  1000,  64, 1, 1000, 0,   64, 1, false, false, false, false, false, 1.f, false, false, false, 0},
        {"rand_k128_n256_p2",           1,  3000, 128, 1, 3000, 0,  256, 2, false, true,  false, true,  false, 1.f, false, false, false, 0},
        {"win4_k256_n512_p2_stream",   37,    65,  64, 4,   62, 0,  512, 2, true,  true,  false, false, false, 1.f, false, false, false, 0},
        {"k256_n512_bias_prelu",        1,  3000, 256, 1, 3000, 0,  512, 3, false, true,  true,  false, false, 1.f, false, false, false, 0},
        {"ln_k64_n256_res",             1,  5000,  64, 1, 5000, 0,  256, 3, true,  true,  false, true,  false, 1.f, false, false, false, 0},
        {"ln_k64_n512",                 1,  2000,  64, 1, 2000, 0,  512, 3, true,  true,  false, false, false, 1.f, false, false, false, 0},
        {"n112_k64",                    1,   700,  64, 1,  700, 0,  112, 3, false, true,  true,  false, false, 1.f, false, false, false, 0},
        {"win4_short_seq_ln",          37,    65,  64, 4,   62, 0,  512, 3, true,  true,  false, false, false, 1.f, false, false, false, 0},
        {"win4_long_seq_halo",          5,   300, 128, 4,  303, -3,  64, 3, false, true,  false, true,  false, 1.f, false, false, false, 0},
        {"win4_long_seq_inner_outer",   6,   200,  64, 4,  197, 0,  512, 3, true,  true,  false, false, false, 1.f, false, false, false, 3},
        {"batched_k520_n300_alpha",     3,   300, 520, 1,  300, 0,  300, 3, false, false, false, false, false, 0.25f, true, false, false, 0},
        {"batched_mn_k300_n1040",       3,   150, 300, 1,  150, 0, 1040, 3, false, false, false, false, false, 1.f, true,  true,  false, 0},
        {"mn_k128_n208",                1,   400, 128, 1,  400, 0,  208, 3, false, true,  false, false, false, 1.f, false, true,  false, 0},
        {"two_src_k128_n256",           1,  1500,  64, 1, 1500, 0,  256, 3, true,  true,  false, false, false, 1.f, false, false, true,  0},
        {"k4160_n256",                  1,   600, 4160, 1, 600, 0,  256, 3, false, true,  false, false, false, 1.f, false, false, false, 0},
    };
    for (const Case& c : cases) if (!only || strstr(c.name, only)) fails += run_case(c);
    if (perf) {
        const Case pc[] = {
            {"perf_k64_n512_ln_p3",     1, 1 << 20,  64, 1, 1 << 20, 0, 512, 3, true,  true, false, false, false, 1.f, false, false, false, 0},
            {"perf_k64_n512_ln_p1",     1, 1 << 20,  64, 1, 1 << 20, 0, 512, 1, true,  true, false, false, false, 1.f, false, false, false, 0},
            {"perf_k64_n64_res_p3",     1, 1 << 21,  64, 1, 1 << 21, 0,  64, 3, false, true, false, true,  false, 1.f, false, false, false, 0},
            {"perf_k128_n64_res_p3",    1, 1 << 20, 128, 1, 1 << 20, 0,  64, 3, false, true, false, true,  false, 1.f, false, false, false, 0},
            {"perf_win4_k256_n512_p3",  1300, 65,    64, 4, 62,      0, 512, 3, true,  true, false, false, false, 1.f, false, false, false, 0},
            {"perf_k4160_n256_p3",      1, 40000, 4160, 1, 40000,    0, 256, 3, false, true, false, false, false, 1.f, false, false, false, 0},
            {"perf_qk_k520_n1280_p3",   32, 1251,   520, 1, 1251,    0, 1280, 3, false, false, false, false, false, 1.f, true, false, false, 0},
            {"perf_pv_k1280_n1040_p3",  32, 1251,  1280, 1, 1251,    0, 1040, 3, false, false, false, false, false, 1.f, true, true,  false, 0},
            {"perf_pv_k1280_n1040_p1",  32, 1251,  1280, 1, 1251,    0, 1040, 1, false, false, false, false, false, 1.f, true, true,  false, 0},
        };
        for (const Case& c : pc) if (!only || strstr(c.name, only)) fails += run_case(c, true);
    }
    printf("%s: %d failing case(s)\n", fails ? "FAILED" : "ALL OK", fails);
    return fails ? 1 : 0;
}
