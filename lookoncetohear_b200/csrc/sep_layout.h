// Shape contract (configs/tsh.json:5-19 of the reference) and HBM layouts of the separation
// engine.  Everything here is compile-time: the kernels are specialised to the one configuration
// the reference ships; l2h_sep_create() rejects anything else.
#pragma once
#include <stdint.h>

namespace l2h {

constexpr int NFFT = 192;      // stft_chunk_size + stft_pad_size
constexpr int HOP = 128;       // stft_chunk_size
constexpr int LOOKAHEAD = 64;  // stft_pad_size
constexpr int NF = 97;         // n_fft/2 + 1
constexpr int NROW = 194;      // filterbank rows (Re | Im)
constexpr int NMIC = 2;
constexpr int NSRC = 2;        // output ears
constexpr int CH = 64;         // D (emb_dim)
constexpr int HID = 64;        // H
constexpr int NHEAD = 4;       // L
constexpr int QE = 6;          // ceil(512/97)
constexpr int VD = 16;         // D / heads
constexpr int ATT = 50;        // local_atten_len
constexpr int RING = 56;       // K/V ring slots per head: the 50-frame window + 6 spare, so that the ring writes of
                               // hops t+1 .. t+6 never touch a row hop t's attention still reads (pipelined streaming;
                               // with 2 spare rows the qkv -> attention -> qkv(t+3) cycle bounds the
                               // pipeline)
constexpr int SPK = 256;
constexpr int QK_DIM = NF * QE;     // 582
constexpr int QK_LD = 584;          // padded to a multiple of 4 floats (16 B rows)
constexpr int V_DIM = NF * VD;      // 1552
constexpr int FC = NF * CH;         // 6208
constexpr int NQKV = 2 * NHEAD * QE + NHEAD * VD;  // 112

// ---- state: one allocation = header + B stream records ---------------------------------------
// header (64 B): the CALL clock of the whole state: int64 pos (frames the calls have covered so
// far), int64 ncalls (calls so far), int64 clip_base (pos at the start of the clip being streamed:
// lets a captured CUDA graph address "chunk pos - clip_base" of a whole-clip buffer without any
// per-launch parameter), int32 done (last-CTA counter of the final kernel).
// Every stream record carries its OWN frame clock (ST_POS, ST_CALLS below): the K/V ring slot of a
// frame and the parity of the double-buffered tails come from it, so streams of one state may start,
// restart and skip hops independently.  Until a stream is reset, copied or skipped, its clock equals
// the header's.
struct StateHeader {
    long long pos;
    long long ncalls;
    long long clip_base;
    int done;
    int pad[9];
};
static_assert(sizeof(StateHeader) == 64, "header");

// per-stream record, offsets in floats
constexpr int64_t ST_EMB = 0;                                   // [256] embedding the gate was built from
constexpr int64_t ST_GEN = ST_EMB + SPK;                        // [4] slot 0: weight generation (int bits) the gate was built with
constexpr int64_t ST_CALLS = ST_GEN + 1;                        // int32: the stream's calls so far (bit 0 = parity of its tails)
constexpr int64_t ST_POS = ST_GEN + 2;                          // int64 (slots 2-3): frames the stream has consumed
constexpr int64_t ST_GATE = ST_GEN + 4;                         // [97][64]  LN(W e + b), (f, c) order
constexpr int64_t ST_CONV = ST_GATE + FC;                       // [2 parity][2 frames][4][97]
constexpr int64_t ST_DECONV = ST_CONV + 2 * 2 * 4 * NF;         // [2][2][97][64]
constexpr int64_t ST_ISTFT = ST_DECONV + 2 * 2 * FC;            // [2][2 ears][194]
constexpr int64_t ST_BLK = ST_ISTFT + 2 * NSRC * NROW;          // blocks start
constexpr int64_t BK_K = 0;                                     // ring [4][RING][584], slot = frame mod RING
constexpr int64_t BK_V = BK_K + (int64_t)NHEAD * RING * QK_LD;  // ring [4][RING][1552]
constexpr int64_t BK_H = BK_V + (int64_t)NHEAD * RING * V_DIM;  // [97][64]
constexpr int64_t BK_C = BK_H + FC;                             // [97][64]
constexpr int64_t BK_STRIDE = BK_C + FC;
static_assert(ST_BLK % 4 == 0 && BK_STRIDE % 4 == 0 && BK_V % 4 == 0, "16 B alignment");
static_assert(ST_POS % 2 == 0, "the int64 stream clock is 8 B aligned (records start 16 B aligned)");

inline int64_t stream_stride(int n_blocks) { return ST_BLK + (int64_t)n_blocks * BK_STRIDE; }

}  // namespace l2h
