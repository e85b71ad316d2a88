// Per-slot enrollment capture: the recent 16 kHz input of each listener, kept on the device so an enrollment can be
// embedded from it in place (l2h_enroll_capture, l2h_embed_forward_slots).  The one statement of the ring's layout, for
// the capture kernel (resample.cu: enroll_capture_kernel) and the enrollment network's ring map (embed_kernels.cuh: XRing).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace l2h {

// A separator chunk of h hops is CHUNK_CARRY samples carried from the previous chunk, then h * CHUNK_HOP new ones: the
// chunks the hop FIFO pops and the capture reads (resample.cu checks them against sep_layout.h's HOP and LOOKAHEAD).
constexpr int CHUNK_HOP = 128, CHUNK_CARRY = 64;

// A slot's row per channel is [EC_HEAD + capacity]: the write position and the samples captured since reset (capped at
// capacity; int32 words stored in the floats' bits), then a ring of `capacity` samples.  The last k <= captured samples
// end just before the write position.  All zeros is an empty capture.
constexpr int EC_HEAD = 2;
constexpr int EC_MIN_CAPACITY = 192;         // the enrollment network's shortest utterance (4 STFT frames)

struct CaptureRow {
    const float* ring;
    int wpos, captured;
};

// the head of the state row st, clamped into the ring: a row that was never written is empty
L2H_DEVINL CaptureRow capture_row(const float* st, int capacity) {
    return {st + EC_HEAD, min(max(__float_as_int(st[0]), 0), capacity - 1), min(max(__float_as_int(st[1]), 0), capacity)};
}

// the head of (slot, ch) of a state of rows of row_floats
L2H_DEVINL CaptureRow capture_row(const float* state, int64_t row_floats, int C, int slot, int ch, int capacity) {
    return capture_row(state + ((int64_t)slot * C + ch) * row_floats, capacity);
}

}  // namespace l2h
