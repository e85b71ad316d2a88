// Device side of umma_gemm: the wgmma kernel.  Included by umma_gemm.cu only.
#pragma once
#include "umma_ptx.cuh"

namespace l2h {
namespace umma {

// ---------------------------------------------------------------------------------------------------------------
// Shared-memory map (all regions 1024-byte aligned):
//   [fp32 staging ring: nstg x 32 KB][A operand ring: nop x planes x 16 KB][B: resident (all k-chunks) or ring of nop]
//   [epilogue transpose buffers: 8 warps x 2 KB]
// Tile schedule: CTA c owns column tile nt = c % n_tiles_n for its whole life (so a resident B is loaded once) and
// walks the row tiles gi, gi + groups, ... with gi = c / n_tiles_n; the n_tiles_n CTAs of a group read the same A tile
// at about the same time (L2 hits).  BN = column tile (64 or 128), TB = 1: B is MN-major.
template <int BN, int TB>
__global__ void __launch_bounds__(NTHREADS, 1)
umma_gemm_kernel(const __grid_constant__ Params p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) unsigned long long bar_stg_full[MAX_NSTG], bar_stg_empty[MAX_NSTG];
    __shared__ __align__(8) unsigned long long bar_op_full[4], bar_op_empty[4];
    __shared__ __align__(8) unsigned long long bar_b_full;
    __shared__ float ln_s[128];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // programmatic dependent launch: the successor may become resident now; THIS kernel's barrier set-up and its
    // weight-slab loads run under the predecessor's tail, and only the roles that touch chain data (the TMA producer
    // before the first activation tile, the math warps before residual reads / stores) wait for the predecessor
    griddep_launch();
    const unsigned smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;     // SWIZZLE_128B atoms need 1024-byte alignment
    const int passes = p.passes, nop = p.nop, NSTG = p.nstg;
    const int planes_a = passes > 1 ? 2 : 1;          // passes: 1 = a_hi b_hi; 2 = + a_lo b_hi (bf16 weights, split activations);
    const int planes = passes > 2 ? 2 : 1;            //         3 = + a_hi b_lo (bf16x3: fp32-grade products).  `planes` = B planes
    const unsigned opA_bytes = (unsigned)planes_a * OPA_PLANE;
    constexpr int NB64 = (BN + 63) >> 6;
    const unsigned opB_plane = TB ? (unsigned)NB64 * 8192u : (unsigned)BN * 128u;
    const unsigned opB_bytes = (unsigned)planes * opB_plane;
    const bool resident = p.b_resident != 0;
    const unsigned stg0 = smem0, opA0 = stg0 + (unsigned)NSTG * STG_BYTES, opB0 = opA0 + (unsigned)nop * opA_bytes;
    const unsigned epi0 = opB0 + (unsigned)(resident ? p.n_chunks : nop) * opB_bytes;

    if (tid == 0) {
        for (int i = 0; i < MAX_NSTG; ++i) { mbar_init(&bar_stg_full[i], 1); mbar_init(&bar_stg_empty[i], 4); }
        for (int i = 0; i < 4; ++i) { mbar_init(&bar_op_full[i], resident ? 4 : 5); mbar_init(&bar_op_empty[i], 8); }
        mbar_init(&bar_b_full, 1);
        mbar_fence_init();
        tmap_prefetch(&p.tmA0); tmap_prefetch(&p.tmA1); tmap_prefetch(&p.tmB);
    }
    if (tid < 128 && p.ln_g != nullptr) ln_s[tid] = tid < 64 ? __ldg(p.ln_g + tid) : __ldg(p.ln_b + tid - 64);
    __syncthreads();

    const int p_tiles = (p.rows_per_seq + p.P_TILE - 1) / p.P_TILE;
    const int s_tiles = (p.nseq + p.S_TILE - 1) / p.S_TILE;
    const int m_tiles = p_tiles * s_tiles;
    const int tile_rows = p.P_TILE * p.S_TILE;
    const int nt = blockIdx.x % p.n_tiles_n, gi = blockIdx.x / p.n_tiles_n, groups = gridDim.x / p.n_tiles_n;
    const int n0 = nt * BN;

    if (warp == 12) {
        // ===================== TMA producer ============================================================
        if (lane == 0) {
            const unsigned stg_tx = 2u * 128u * (unsigned)tile_rows;                       // two 32-float half boxes
            auto load_b = [&](unsigned dst, unsigned long long* bar, int j, int bz) {
                for (int pl = 0; pl < planes; ++pl) {
                    if (!TB) {
                        tma_load_4d(dst + pl * opB_plane, &p.tmB, bar, j * KC, n0, bz, pl);
                    } else {
                        for (int nb = 0; nb < NB64; ++nb)
                            tma_load_4d(dst + pl * opB_plane + nb * 8192, &p.tmB, bar, n0 + nb * 64, j * KC, bz, pl);
                    }
                }
            };
            if (resident) {                           // the whole [BN x K] weight slab, once
                mbar_expect_tx(&bar_b_full, opB_bytes * (unsigned)p.n_chunks);
                for (int j = 0; j < p.n_chunks; ++j) load_b(opB0 + j * opB_bytes, &bar_b_full, j, 0);
            }
            griddep_wait();                           // activations (and a batched B) come from the predecessor
            unsigned it = 0;
            for (int mt = gi; mt < m_tiles; mt += groups) {
                const int p0 = (mt % p_tiles) * p.P_TILE, seq0 = (mt / p_tiles) * p.S_TILE;
                const int s_in = seq0 % p.seq_inner, s_out = seq0 / p.seq_inner;
                const int bz = p.b_by_seq ? seq0 : 0;
                for (int j = 0; j < p.n_chunks; ++j, ++it) {
                    const KChunk kc = p.chunks[j];
                    const int s = it % NSTG, o = it % nop;
                    mbar_wait_to(&bar_stg_empty[s], ((it / NSTG) & 1) ^ 1);
                    mbar_expect_tx(&bar_stg_full[s], stg_tx);
                    const CUtensorMap* tm = (kc.flags & 1) ? &p.tmA1 : &p.tmA0;
                    const unsigned dst = stg0 + s * STG_BYTES;
                    tma_load_4d(dst, tm, &bar_stg_full[s], kc.c0, p0 + kc.dp + p.pos_bias, s_in, s_out);
                    tma_load_4d(dst + STG_BYTES / 2, tm, &bar_stg_full[s], kc.c0 + 32, p0 + kc.dp + p.pos_bias, s_in, s_out);
                    if (!resident) {
                        mbar_wait_to(&bar_op_empty[o], ((it / nop) & 1) ^ 1);
                        mbar_expect_tx(&bar_op_full[o], opB_bytes);
                        load_b(opB0 + o * opB_bytes, &bar_op_full[o], j, bz);
                    }
                }
            }
        }
    } else if (warp < 4) {
        // ===================== converter: fp32 staging -> bf16 hi/lo operand tile (thread = row) =======
        const int r = tid;
        const unsigned sw = (unsigned)(r & 7);
        unsigned it = 0;
        for (int mt = gi; mt < m_tiles; mt += groups) {
            for (int j = 0; j < p.n_chunks; ++j, ++it) {
                const int s = it % NSTG, o = it % nop;
                mbar_wait_to(&bar_stg_full[s], (it / NSTG) & 1);
                float v[64];
                const unsigned src = stg0 + s * STG_BYTES + (unsigned)r * 128u;
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (unsigned c = 0; c < 8; ++c) {
                        float4 t;
                        asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(t.x), "=f"(t.y), "=f"(t.z), "=f"(t.w)
                                     : "r"(src + h * (STG_BYTES / 2) + ((c ^ sw) << 4)));
                        v[h * 32 + c * 4 + 0] = t.x; v[h * 32 + c * 4 + 1] = t.y;
                        v[h * 32 + c * 4 + 2] = t.z; v[h * 32 + c * 4 + 3] = t.w;
                    }
                if (p.chunks[j].flags & 2) {        // LayerNorm over the 64 channels of this row (two-pass, biased var)
                    float sum = 0.f;
#pragma unroll
                    for (int i = 0; i < 64; ++i) sum += v[i];
                    const float mu = sum * (1.f / 64.f);
                    float q = 0.f;
#pragma unroll
                    for (int i = 0; i < 64; ++i) { v[i] -= mu; q = fmaf(v[i], v[i], q); }
                    const float rs = rsqrtf(q * (1.f / 64.f) + 1e-5f);
#pragma unroll
                    for (int i = 0; i < 64; ++i) v[i] = fmaf(v[i] * rs, ln_s[i], ln_s[64 + i]);
                }
                mbar_wait_to(&bar_op_empty[o], ((it / nop) & 1) ^ 1);
                const unsigned dst = opA0 + o * opA_bytes + (unsigned)r * 128u;
#pragma unroll
                for (unsigned c = 0; c < 8; ++c) {
                    unsigned hi[4], lo[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const float a0 = v[c * 8 + 2 * e], a1 = v[c * 8 + 2 * e + 1];
                        const __nv_bfloat162 h2 = __floats2bfloat162_rn(a0, a1);
                        hi[e] = *reinterpret_cast<const unsigned*>(&h2);
                        const float2 hf = __bfloat1622float2(h2);
                        lo[e] = pack_bf16x2(a0 - hf.x, a1 - hf.y);
                    }
                    const unsigned off = dst + ((c ^ sw) << 4);
                    asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(off), "r"(hi[0]), "r"(hi[1]), "r"(hi[2]), "r"(hi[3]) : "memory");
                    if (passes > 1)
                        asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(off + OPA_PLANE), "r"(lo[0]), "r"(lo[1]), "r"(lo[2]), "r"(lo[3]) : "memory");
                }
                fence_proxy_async();                 // generic-proxy writes -> visible to the tensor core (async proxy)
                __syncwarp();
                if (lane == 0) { mbar_arrive(&bar_op_full[o]); mbar_arrive(&bar_stg_empty[s]); }
            }
        }
    } else {
        // ===================== math: wgmma over 64 rows, then the epilogue of those rows ====================
        // Both warpgroups read the same B tile and their own half of the A tile.  A chunk's operand slot is handed back
        // when the NEXT chunk's MMAs have been issued and the chunk's own have completed (wait_group 1), so the tensor
        // core always has one chunk queued.  Epilogue: the accumulator fragment (thread = 2 rows x 2 columns per 8) of
        // each warp's 16 rows is transposed through 2 KB of swizzled shared memory per 32 columns and stored with 8 lanes
        // per row: one warp instruction writes four full 128-byte lines.  Bias / PReLU / residual are applied after the
        // transpose, where a lane's columns are fixed and the residual is read with the same coalesced pattern.
        const int wg = (warp - 4) >> 2, wq = warp & 3;
        const unsigned tb = epi0 + (unsigned)(warp - 4) * 2048u;
        const float slope1 = p.prelu ? __ldg(p.prelu) : 1.f;      // scalar PReLU slope (1 = identity)
        const bool has_prelu = p.prelu != nullptr || p.prelu_vec != nullptr;
        const int chunk = lane & 7, rsub = lane >> 3;
        const unsigned kstep_b = TB ? 128u : 2u;                  // 16 k: 32 B along a K-major row, 16 rows of 2048 B MN-major
        const unsigned b_lbo = TB ? 8192u : 16u;
        griddep_wait();                               // C may still be read, R still be written by the predecessor
        if (resident) mbar_wait_to(&bar_b_full, 0);
        unsigned it = 0;
        for (int mt = gi; mt < m_tiles; mt += groups) {
            float acc[BN / 2];
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
            int prev_o = -1;
            for (int j = 0; j < p.n_chunks; ++j, ++it) {
                const int o = it % nop;
                mbar_wait_to(&bar_op_full[o], (it / nop) & 1);
                const unsigned abase = opA0 + o * opA_bytes + (unsigned)wg * 8192u;
                const unsigned bbase = opB0 + (unsigned)(resident ? j : o) * opB_bytes;
                const unsigned long long da_hi = smem_desc(abase, 16, 1024);
                const unsigned long long da_lo = smem_desc(abase + OPA_PLANE, 16, 1024);
                const unsigned long long db_hi = smem_desc(bbase, b_lbo, 1024);
                const unsigned long long db_lo = smem_desc(bbase + opB_plane, b_lbo, 1024);
                wg_fence();
                for (int ps = 0; ps < passes; ++ps) {
                    const unsigned long long da = (ps == 1) ? da_lo : da_hi;
                    const unsigned long long db = (ps == 2) ? db_lo : db_hi;
#pragma unroll
                    for (unsigned kk = 0; kk < 4; ++kk)
                        wgmma_bf16<BN, TB>(acc, da + kk * 2, db + kk * kstep_b, (j | ps | (int)kk) != 0);
                }
                wg_commit();
                if (nop > 1) {
                    wg_wait<1>();
                    if (prev_o >= 0 && lane == 0) mbar_arrive(&bar_op_empty[prev_o]);
                    prev_o = o;
                } else {
                    wg_wait<0>();
                    if (lane == 0) mbar_arrive(&bar_op_empty[o]);
                }
            }
            wg_wait<0>();
            wg_fence_regs(acc);
            if (prev_o >= 0 && lane == 0) mbar_arrive(&bar_op_empty[prev_o]);

            const int p0 = (mt % p_tiles) * p.P_TILE, seq0 = (mt / p_tiles) * p.S_TILE;
            const int r = wg * 64 + wq * 16 + (lane & 15);       // tile row whose offsets this lane computes
            const int sl = r / p.P_TILE, pos = p0 + r % p.P_TILE, seq = seq0 + sl;
            const int valid = (r < tile_rows && pos < p.rows_per_seq && seq < p.nseq) ? 1 : 0;
            long long coff;
            if (p.c_inner > 1)
                coff = (long long)(seq / p.c_inner) * p.c_seq_stride + (long long)(seq % p.c_inner) * p.c_inner_stride + (long long)pos * p.ldc;
            else
                coff = (long long)seq * p.c_seq_stride + (long long)pos * p.ldc;
#pragma unroll
            for (int cb = 0; cb < BN; cb += 32) {
                const int nl = cb + chunk * 4;         // this lane's four columns inside the tile (after the transpose)
                const int n = n0 + nl;
                const bool col_ok = n < p.N;
                const bool full4 = col_ok && (n + 3 < p.N) && p.vec_ok;
                // per-column epilogue operands of this lane (L1 hits after the first tile: same columns every tile)
                float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f), s4 = make_float4(slope1, slope1, slope1, slope1);
                if (full4) {
                    if (p.bias) b4 = __ldg(reinterpret_cast<const float4*>(p.bias + n));
                    if (p.prelu_vec) s4 = __ldg(reinterpret_cast<const float4*>(p.prelu_vec + n));
                }
                __syncwarp();                          // transpose buffer free again
#pragma unroll
                for (int ii = 0; ii < 4; ++ii) {
                    const int i = cb / 8 + ii;
                    const unsigned c = 8u * (unsigned)ii + 2u * (unsigned)(lane & 3);
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const unsigned row = (unsigned)(lane >> 2) + 8u * (unsigned)h;
                        asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(tb + row * 128u + (((c >> 2) ^ (row & 7u)) << 4) + (c & 3u) * 4u),
                                     "f"(acc[4 * i + 2 * h]), "f"(acc[4 * i + 2 * h + 1]) : "memory");
                    }
                }
                __syncwarp();
                if (__all_sync(0xffffffffu, full4 || !col_ok)) {
                    // ---- fast path: whole float4 groups.  Row offsets first (and the residual loads in flight), then math
                    long long co[4];
                    unsigned okm = 0;
#pragma unroll
                    for (int itr = 0; itr < 4; ++itr) {
                        const int row = itr * 4 + rsub;
                        co[itr] = __shfl_sync(0xffffffffu, coff, row) + n;
                        okm |= (unsigned)(__shfl_sync(0xffffffffu, valid, row) & (col_ok ? 1 : 0)) << itr;
                    }
                    float4 rr[4];
                    if (p.R) {
#pragma unroll
                        for (int itr = 0; itr < 4; ++itr)
                            rr[itr] = ((okm >> itr) & 1u) ? *reinterpret_cast<const float4*>(p.R + co[itr]) : make_float4(0.f, 0.f, 0.f, 0.f);
                    }
#pragma unroll
                    for (int itr = 0; itr < 4; ++itr) {
                        const int row = itr * 4 + rsub;
                        float4 o;
                        asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(o.x), "=f"(o.y), "=f"(o.z), "=f"(o.w)
                                     : "r"(tb + (unsigned)row * 128u + (((unsigned)chunk ^ (unsigned)(row & 7)) << 4)));
                        o.x = fmaf(o.x, p.alpha, b4.x); o.y = fmaf(o.y, p.alpha, b4.y); o.z = fmaf(o.z, p.alpha, b4.z); o.w = fmaf(o.w, p.alpha, b4.w);
                        if (has_prelu) {               // max(x,0) + slope * min(x,0)
                            o.x = fmaf(s4.x, fminf(o.x, 0.f), fmaxf(o.x, 0.f)); o.y = fmaf(s4.y, fminf(o.y, 0.f), fmaxf(o.y, 0.f));
                            o.z = fmaf(s4.z, fminf(o.z, 0.f), fmaxf(o.z, 0.f)); o.w = fmaf(s4.w, fminf(o.w, 0.f), fmaxf(o.w, 0.f));
                        }
                        if (p.R) { o.x += rr[itr].x; o.y += rr[itr].y; o.z += rr[itr].z; o.w += rr[itr].w; }
                        if ((okm >> itr) & 1u) *reinterpret_cast<float4*>(p.C + co[itr]) = o;
                    }
                } else {
                    // ---- cold path: ragged N or unaligned rows, element by element
#pragma unroll 1
                    for (int itr = 0; itr < 4; ++itr) {
                        const int row = itr * 4 + rsub;
                        float4 o;
                        asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(o.x), "=f"(o.y), "=f"(o.z), "=f"(o.w)
                                     : "r"(tb + (unsigned)row * 128u + (((unsigned)chunk ^ (unsigned)(row & 7)) << 4)));
                        const long long cor = __shfl_sync(0xffffffffu, coff, row);
                        const int ok = __shfl_sync(0xffffffffu, valid, row);
                        if (!ok || !col_ok) continue;
                        const float ov[4] = {o.x, o.y, o.z, o.w};
                        for (int e = 0; e < 4 && n + e < p.N; ++e) {
                            float x = ov[e] * p.alpha;
                            if (p.bias) x += __ldg(p.bias + n + e);
                            if (p.prelu) x = prelu(x, slope1);
                            if (p.prelu_vec) x = prelu(x, __ldg(p.prelu_vec + n + e));
                            if (p.R) x += p.R[cor + n + e];
                            p.C[cor + n + e] = x;
                        }
                    }
                }
            }
        }
    }
}

}  // namespace umma
}  // namespace l2h
