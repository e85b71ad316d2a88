// PTX wrappers shared by the tensor-core kernels (umma_gemm_kernel, tc_lstm_kernel): mbarrier, tensor-map TMA, Hopper
// warpgroup MMA (wgmma) and its shared-memory matrix descriptors.  Device-inline only: safe to include from every
// translation unit.
#pragma once
#include "umma_gemm.cuh"

namespace l2h {
namespace umma {

// ---- PTX wrappers ---------------------------------------------------------------------------------------------
L2H_DEVINL void mbar_arrive(unsigned long long* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// bounded wait: a protocol bug must not hang the GPU -- trap after ~2 s.  (No printf here: a call between wgmma
// instructions of one pipeline makes ptxas serialize the MMAs.)
L2H_DEVINL void mbar_wait_to(unsigned long long* bar, unsigned parity) {
    const unsigned addr = smem_u32(bar);
    const long long t0 = clock64();
    for (;;) {
        unsigned ok;
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}"
                     : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
        if (ok) return;
        if (clock64() - t0 > 4000000000ll) __trap();
    }
}
L2H_DEVINL void tma_load_4d(unsigned dst, const CUtensorMap* tm, unsigned long long* bar, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                 ::"r"(dst), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
L2H_DEVINL void tmap_prefetch(const CUtensorMap* tm) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(tm) : "memory");
}

// ---- warpgroup MMA (sm_90a) ------------------------------------------------------------------------------------
// D[64 x N] (+)= A[64 x 16] . B[16 x N], bf16 operands from shared memory (descriptors), fp32 accumulators in the
// registers of the issuing warpgroup.  Accumulator fragment of thread t = 32 w + l: element 4 i + e holds row
// 16 w + l / 4 + 8 (e >> 1), column 8 i + 2 (l % 4) + (e & 1).  TB = 1: B is MN-major (transposed) in shared memory.
// scale_d = 0 overwrites D (first product of a tile), 1 accumulates.
L2H_DEVINL void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
L2H_DEVINL void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
L2H_DEVINL void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// the accumulator registers must not be touched by other instructions while an MMA group is in flight
template <int R>
L2H_DEVINL void wg_fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

template <int TB>
L2H_DEVINL void wgmma_n32(float (&d)[16], unsigned long long da, unsigned long long db, int scale_d) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, %19;\n}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(da), "l"(db), "r"(scale_d), "n"(TB));
}
template <int TB>
L2H_DEVINL void wgmma_n64(float (&d)[32], unsigned long long da, unsigned long long db, int scale_d) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, %35;\n}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(da), "l"(db), "r"(scale_d), "n"(TB));
}
template <int TB>
L2H_DEVINL void wgmma_n128(float (&d)[64], unsigned long long da, unsigned long long db, int scale_d) {
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, %67;\n}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(da), "l"(db), "r"(scale_d), "n"(TB));
}

template <int N, int TB>
L2H_DEVINL void wgmma_bf16(float (&d)[N / 2], unsigned long long da, unsigned long long db, int scale_d) {
    static_assert(N == 32 || N == 64 || N == 128, "wgmma shape");
    if constexpr (N == 32) wgmma_n32<TB>(d, da, db, scale_d);
    else if constexpr (N == 64) wgmma_n64<TB>(d, da, db, scale_d);
    else wgmma_n128<TB>(d, da, db, scale_d);
}

// shared-memory matrix descriptor (sm_90 wgmma): start address, leading/stride byte offsets (>>4), SWIZZLE_128B
// (layout type 1 in bits 62-63).  K-major operand tile: rows of 128 B (64 bf16 along K), 8-row groups 1024 B apart
// (SBO), LBO unused (16).  MN-major operand tile: k rows of 128 B (64 bf16 along N), 8-row groups 1024 B apart (SBO),
// the next 64 columns `lbo_bytes` further (LBO).  Advancing the start address by 32 B steps 16 k inside a K-major
// swizzle row; by 2048 B (16 rows) in an MN-major tile.
L2H_DEVINL unsigned long long smem_desc(unsigned addr, unsigned lbo_bytes, unsigned sbo_bytes) {
    unsigned long long d = 0;
    d |= (unsigned long long)((addr & 0x3FFFFu) >> 4);
    d |= (unsigned long long)((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= (unsigned long long)((sbo_bytes >> 4) & 0x3FFFu) << 32;
    d |= 1ull << 62;
    return d;
}

L2H_DEVINL unsigned pack_bf16x2(float lo_elem, float hi_elem) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(lo_elem, hi_elem);
    return *reinterpret_cast<const unsigned*>(&h);
}

}  // namespace umma
}  // namespace l2h
