// Packed fp32 weights of an engine (host side, shared by the separation and the enrollment engine): the host staging
// buffer, the table of reference tensor names, the device copy and the bf16 hi/lo planes of the tensor-core B operands.
//
// The layout is fixed when the engine is created: `alloc` hands out 4-float-aligned offsets into one buffer, each slot
// says how one reference tensor lands there, `bind` records which weight-struct field points at which offset, and `plane`
// registers a k-major matrix to be split into bf16 planes.  A commit is `finish` (every slot loaded; accumulate slots
// summed on the host), then `upload` (device buffers on the current device, bound fields pointed into them, planes split).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>

#include <algorithm>
#include <cstring>
#include <functional>
#include <iterator>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "host_errors.h"
#include "umma_host.cuh"

namespace l2h {

// LSTM gate-row permutation: packed row j*4+q <- reference row q*64+j
inline int perm_row(int p) { return (p & 3) * 64 + (p >> 2); }

struct WeightPack {
    using Repack = std::function<void(const float* src, float* host)>;   // host = base of the packed host buffer
    enum Kind {
        COPY,         // memcpy to [off, off + numel)
        REPACK,       // `repack` at load
        ACCUMULATE,   // kept until commit, then `repack` adds it into [off, off + numel), which was zeroed first (so
                      // several tensors can sum into one destination: an LSTM's b_ih + b_hh)
        IGNORED,      // accepted and counted, not used
    };
    struct Slot {
        Kind kind;
        int64_t off, numel;   // numel = element count of the reference tensor
        Repack repack;
        bool loaded = false;
        std::vector<float> raw;   // ACCUMULATE: the loaded tensor
    };
    struct PlaneSrc { int64_t wt_off; int K, N, ld, col0; int64_t plane_off; };

    std::vector<float> host;                                 // packed staging buffer
    std::map<std::string, Slot> slots;                       // alphabetical: the order of l2h_sep_weight_info and of the sums
    std::vector<std::pair<const float**, int64_t>> fields;   // weight-struct fields and the offsets they point at
    std::vector<PlaneSrc> plane_srcs;
    int64_t planes_total = 0;                                // elements of one plane set; the lo planes follow the hi planes
    float* dev = nullptr;
    __nv_bfloat16* planes = nullptr;
    int device = -1;                                         // ordinal that holds `dev` and `planes`
    bool committed = false;

    int64_t alloc(int64_t n) {
        const int64_t o = (int64_t)host.size();
        host.resize((o + n + 3) & ~int64_t(3), 0.f);
        return o;
    }
    int64_t plain(const std::string& name, int64_t n) {
        const int64_t o = alloc(n);
        slots[name] = Slot{COPY, o, n, nullptr};
        return o;
    }
    void repacked(const std::string& name, int64_t numel, Repack fn) { slots[name] = Slot{REPACK, 0, numel, std::move(fn)}; }
    void accumulate(const std::string& name, int64_t off, int64_t numel, Repack fn) {
        slots[name] = Slot{ACCUMULATE, off, numel, std::move(fn)};
    }
    void ignore(const std::string& name, int64_t numel) { slots[name] = Slot{IGNORED, 0, numel, nullptr}; }
    void bind(const float** field, int64_t off) { fields.push_back({field, off}); }

    // bf16 hi/lo planes [2][N][ld] of the k-major fp32 matrix [K][N] at `wt_off`, made at upload; returns the plane offset.
    // With col0 > 0 the matrix fills columns col0 .. col0+K-1 of the plane registered just before it (operands
    // concatenated along k).
    int64_t plane(int64_t wt_off, int K, int N, int ld, int col0 = 0) {
        const int64_t at = col0 > 0 ? plane_srcs.back().plane_off : planes_total;
        if (col0 == 0) planes_total += ((int64_t)N * ld + 63) & ~int64_t(63);
        plane_srcs.push_back({wt_off, K, N, ld, col0, at});
        return at;
    }
    umma::BPlanes bplanes(int64_t plane_off, int ld) const {
        umma::BPlanes b;
        b.base = planes + plane_off; b.ld = ld; b.plane_stride = planes_total; b.nz = 1;
        return b;
    }

    int load(const char* name, const float* data, int64_t numel) {
        auto it = slots.find(name);
        if (it == slots.end()) return fail(2, std::string("unknown weight name: ") + name);
        Slot& s = it->second;
        if (numel != s.numel) return fail(1, std::string("wrong element count for ") + name);
        if (s.kind == COPY) memcpy(host.data() + s.off, data, numel * sizeof(float));
        else if (s.kind == REPACK) s.repack(data, host.data());
        else if (s.kind == ACCUMULATE) s.raw.assign(data, data + numel);
        s.loaded = true;
        committed = false;
        return 0;
    }
    void counts(int32_t* n_expected, int32_t* n_loaded) const {
        int n = 0;
        for (const auto& kv : slots) n += kv.second.loaded ? 1 : 0;
        if (n_expected) *n_expected = (int32_t)slots.size();
        if (n_loaded) *n_loaded = n;
    }
    int info(int32_t index, const char** name, int64_t* numel) const {
        if (index < 0 || index >= (int32_t)slots.size()) return fail(1, "weight index out of range");
        auto it = std::next(slots.begin(), index);
        if (name) *name = it->first.c_str();             // owned by the pack, valid until it is destroyed
        if (numel) *numel = it->second.numel;
        return 0;
    }

    // commit, step 1: the host buffer is complete (an engine may derive more packed data from it before `upload`)
    int finish() {
        for (const auto& kv : slots)
            if (!kv.second.loaded) return fail(4, "weight not loaded: " + kv.first);
        for (const auto& kv : slots)
            if (kv.second.kind == ACCUMULATE) std::fill(host.begin() + kv.second.off, host.begin() + kv.second.off + kv.second.numel, 0.f);
        for (const auto& kv : slots)
            if (kv.second.kind == ACCUMULATE) kv.second.repack(kv.second.raw.data(), host.data());
        return 0;
    }
    // commit, step 2: copy to the current device (buffers that live on another device are released and made again here)
    // and split the planes; synchronises `st`
    int upload(cudaStream_t st) {
        int cur = -1;
        CK(cudaGetDevice(&cur));
        if (dev != nullptr && device != cur) release();
        if (dev == nullptr) {
            CK(cudaMalloc(&dev, host.size() * sizeof(float)));
            device = cur;
            for (auto& f : fields) *f.first = dev + f.second;
            CK(cudaMalloc(&planes, 2 * planes_total * sizeof(__nv_bfloat16)));
        }
        CK(cudaMemcpyAsync(dev, host.data(), host.size() * sizeof(float), cudaMemcpyHostToDevice, st));
        for (const auto& p : plane_srcs)        // k-major fp32 [K][N] -> bf16 hi/lo planes [N][ld]
            CK(umma::split_planes(dev + p.wt_off, 1, p.N, p.N, p.K, p.ld, planes + p.plane_off + p.col0,
                                  planes + planes_total + p.plane_off + p.col0, st));
        CK(cudaStreamSynchronize(st));
        committed = true;
        return 0;
    }
    // frees the device buffers on the device that holds them; the host side stays, so a later upload makes them again
    void release() {
        int cur = -1;
        const bool sw = device >= 0 && cudaGetDevice(&cur) == cudaSuccess && cur != device;
        if (sw) cudaSetDevice(device);
        if (dev) cudaFree(dev);
        if (planes) cudaFree(planes);
        if (sw) cudaSetDevice(cur);
        dev = nullptr;
        planes = nullptr;
        device = -1;
        committed = false;
    }
};

}  // namespace l2h
