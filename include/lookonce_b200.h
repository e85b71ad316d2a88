/* lookonce_b200.h -- C ABI of the LookOnceToHear inference engine for the H100 (sm_90a).
 *
 * Drop-in boundary for ONE path of vb000/LookOnceToHear: the inference forward of its two
 * networks.  The reference is pure Python; the interface each entry point stands in for is the
 * Python method the reference's evaluation path calls (all paths relative to the reference repository):
 *
 *   l2h_sep_create / l2h_sep_load_weight / l2h_sep_commit_weights
 *        <- Net.__init__ + load_state_dict      src/models/tfgridnet_realtime/net.py:20-49,
 *                                               src/ts_hear_test.py:18-34 (load_model)
 *   l2h_sep_state_bytes / l2h_sep_state_init
 *        <- Net.init_buffers                    net.py:51-52, tfgridnet_causal.py:173-186,408-427
 *   l2h_sep_forward
 *        <- Net.predict / Net.forward           net.py:54-76  -> TFGridNet.forward
 *                                               tfgridnet_causal.py:188-283
 *   l2h_sep_forward_active / l2h_sep_forward_slots
 *        <- one Net.predict hop for some of a state's streams (serving many listeners: INTEGRATION.md)
 *   l2h_sep_forward_slots_frames / l2h_sep_forward_slots_hops
 *        <- several Net.predict hops for a list of a state's streams, the same number for every row or one per row
 *           (Net.advance_slots)
 *   l2h_sep_forward_targets / l2h_sep_forward_targets_groups / l2h_sep_forward_targets_rows
 *        <- Net.predict for several enrolled speakers of each mixture, for a whole state, a list of its listener
 *           groups, or listeners with different numbers of speakers (Net.predict_targets, Net.advance_targets,
 *           Net.advance_target_rows)
 *   l2h_sep_forward_targets_rows_history / l2h_sep_join_targets / l2h_sep_state_move_lead
 *        <- adding a speaker to a running listener, warmed from its recent block-0 output, and dropping one
 *           (Net.advance_target_rows(history=), Net.join_targets, SepState.move_lead)
 *   l2h_sep_stream_host
 *        <- the chunk loop around Net.predict(chunk, embed, state, pad=False)  (SURVEY.md 3.3)
 *           with host buffers: H2D of each chunk and D2H of each result inside the call
 *   l2h_embed_create / l2h_embed_load_weight / l2h_embed_commit_weights / l2h_embed_forward
 *        <- EmbedTFGridNet.__init__/forward     src/models/tfgridnet_orig/tfgridnet.py:88-127
 *   l2h_enroll_capture / l2h_embed_forward_slots
 *        <- EmbedTFGridNet.forward of a listener's own recent stream (EnrollCapture, EmbedTFGridNet.enroll)
 *   l2h_target_mix / l2h_target_mix_set
 *        <- summing each listener's target voices, and a little of its mixture, into one output row with fades
 *           (TargetMixer)
 *   l2h_limiter
 *        <- keeping each listener's output under a ceiling, with one gain for both ears (Limiter)
 *   l2h_leveler
 *        <- bringing each voice a listener hears to one loudness, with one gain for both ears (Leveler)
 *   l2h_band_compressor
 *        <- fitting each listener's output to their hearing: gain per band and per ear, compression per band linked across
 *           the ears (BandCompressor)
 *   l2h_band_compressor_lr
 *        <- the same on a Linkwitz-Riley crossover bank, whose delay is shorter (BandCompressor(bank="lr4" or "lr8"))
 *   l2h_jitter_buffer
 *        <- putting a device's packets back in sequence order and concealing lost ones, over a lossy network
 *           (JitterBuffer)
 *   l2h_jitter_buffer_timed
 *        <- the same, releasing missing packets on the server's clock, so an uplink gap is concealed as it happens
 *           (JitterBuffer(deadline=...))
 *   l2h_jitter_buffer_adaptive
 *        <- the same, with each listener's deadline drawn from the measured lateness of their own packets
 *           (JitterBuffer(deadline=(lo, hi)))
 *
 * Conventions follow the reference's only FFI (src/datasets/motion_simulator.py:30-95): every
 * function returns int (0 = OK, non-zero = error, text via l2h_last_error()), handles are opaque
 * void*, buffers are plain float pointers + sizes, explicit *_destroy.  No torch types.  Device
 * pointers are CUDA device memory of the current device; `stream` is a cudaStream_t passed as
 * void* (NULL = default stream).  Nothing synchronises the stream except where stated.
 * One handle per device; a handle is not thread-safe.
 */
#ifndef LOOKONCE_B200_H
#define LOOKONCE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define L2H_ABI_VERSION 1

/* configs/tsh.json:5-19 -> Net(**model_params) */
typedef struct l2h_sep_config {
    int32_t stft_chunk_size; /* 128 */
    int32_t stft_pad_size;   /* 64  */
    int32_t embed_dim;       /* 256 */
    int32_t num_ch;          /* 2   */
    int32_t D;               /* 64  */
    int32_t L;               /* 4 heads */
    int32_t I;               /* 1   */
    int32_t J;               /* 1   */
    int32_t B;               /* number of GridNet blocks (3) */
    int32_t H;               /* 64  */
    int32_t local_atten_len; /* 50  */
    int32_t use_attn;        /* 1   */
    int32_t lookahead;       /* 1   */
    int32_t chunk_causal;    /* 1   */
    int32_t num_src;         /* 2   */
} l2h_sep_config;

/* flags for l2h_sep_forward */
#define L2H_FLAG_TAPS 1u  /* also copy the activations after every stage into the tap area */
#define L2H_FLAG_GRAPH 2u /* replay the kernel chain from a CUDA graph cached on the exact argument set
                             (pointers, strides, sizes): for callers that reuse fixed staging buffers */

int l2h_abi_version(void);
const char* l2h_last_error(void);

/* ---- separation network -------------------------------------------------------------------- */
int l2h_sep_create(const l2h_sep_config* cfg, void** handle);
int l2h_sep_destroy(void* handle);

/* name = a key of the reference state_dict without the Lightning "model." prefix, e.g.
 * "tfgridnet.blocks.0.intra_rnn.weight_ih_l0"; data = HOST fp32, contiguous, numel elements.
 * Repacks into the engine's layouts in a host staging buffer.  Unknown names -> error 2. */
int l2h_sep_load_weight(void* handle, const char* name, const float* host_data, int64_t numel);
/* number of reference tensors the engine expects / has received so far */
int l2h_sep_weights_expected(void* handle, int32_t* n_expected, int32_t* n_loaded);
/* the index-th expected tensor (0 <= index < n_expected, alphabetical): its reference name (owned by the handle) and
 * element count -- what a host that converts a checkpoint iterates over (examples/stream_clip.cpp) */
int l2h_sep_weight_info(void* handle, int32_t index, const char** name, int64_t* numel);
/* upload the staged weights (one H2D of ~8 MB on `stream`, then synchronises it) */
int l2h_sep_commit_weights(void* handle, void* stream);

int l2h_sep_state_bytes(void* handle, int32_t batch, size_t* bytes);
int l2h_sep_state_init(void* handle, void* state_dev, int32_t batch, void* stream);
/* floats per stream record and header bytes, for host code that builds views of the state */
int l2h_sep_state_layout(void* handle, int64_t* header_bytes, int64_t* stream_stride_floats);
/* The offsets (in floats) inside one stream record, for host code that converts to / from the reference's nested
 * state dict (tfgridnet_causal.py:173-186, :408-427) -- SepState.to_reference() / load_reference().  out[i]:
 * 0 ring slots per head, 1 K row stride, 2 K row length (582), 3 V row length (1552), 4 attention window (50),
 * 5 embedding copy, 6 cached speaker gate, 7 conv tail, 8 deconv tail, 9 iSTFT tail, 10 first block, then inside a
 * block: 11 K ring, 12 V ring, 13 h, 14 c, 15 block stride; then the stream's own clock: 16 its frame count (int64),
 * 17 its call count (int32; bit 0 = which copy of the double-buffered tails is current).  n may be 16 (the first 16
 * values only) or more; at most L2H_STATE_OFFSETS values are written.
 *
 * Every stream of a state has its own clock: the K/V ring slot of a frame and the current tails come from it, not from
 * the state's header (which counts the calls and addresses the clip of l2h_sep_stream_dev).  l2h_sep_state_init sets
 * every clock to 0, and without the three calls below every clock equals the header's. */
#define L2H_STATE_OFFSETS 18
int l2h_sep_state_offsets(void* handle, int64_t* out, int32_t n);

/* Serving many listeners from one state (INTEGRATION.md).  Argument errors (null pointers, batch or n <= 0, a slot outside
 * [0, batch), a slot listed twice) return 1 before anything is enqueued.  Asynchronous on `stream`.
 *
 * l2h_sep_state_reset_streams: records slots_host[0 .. n) of a state of `batch` streams become fresh streams (zero rings,
 * h / c and tails, clock 0, speaker-gate memo invalidated), as in a state just initialised; the other records are not
 * touched.  One kernel launch per 960 slots.
 *
 * l2h_sep_state_copy_streams: record src_slots_host[i] of src_state -> record dst_slots_host[i] of dst_state, the clock
 * included, so the stream continues in its new slot exactly as it would have in the old one.  Both states belong to this
 * handle's configuration and device (they may be the same state; then no slot may be both a source and a destination).
 * The copied records' gate memo is invalidated (it is rebuilt at their next call).  A stream moves to another device by a
 * host copy of its record (SepState views) into an initialised state there. */
int l2h_sep_state_reset_streams(void* handle, void* state_dev, int32_t batch, const int32_t* slots_host, int32_t n, void* stream);
/* l2h_sep_state_move_lead: record new_host[i] takes over as its listener's lead from record old_host[i] (a record of the same
 * listener): the speaker-independent part of old_host[i] -- block 0's K/V rings and (h, c), and the current copy of its conv
 * tails, which goes into the copy new_host[i]'s own parity makes current -- is copied into new_host[i].  Its blocks
 * 1 .. B-1, back tails, embedding, gate memo and clock stay as they are.  The two clocks must be equal: the call waits for
 * `stream`, reads them and refuses the call (1) if any pair differs.  Then old_host[i] may be dropped from the listener's
 * rows.  Errors 1, before anything is enqueued: null pointers, batch or n <= 0, n > batch, a record outside [0, batch) or
 * listed twice in one list, a record in both lists, different clocks. */
int l2h_sep_state_move_lead(void* handle, void* state_dev, int32_t batch, const int32_t* old_host, const int32_t* new_host,
                            int32_t n, void* stream);
int l2h_sep_state_copy_streams(void* handle, void* dst_state_dev, int32_t dst_batch, const int32_t* dst_slots_host,
                               const void* src_state_dev, int32_t src_batch, const int32_t* src_slots_host, int32_t n,
                               void* stream);

int l2h_sep_workspace_bytes(void* handle, int32_t batch, int32_t frames, uint32_t flags, size_t* bytes);

/* One call = `frames` hops of 128 samples for `batch` independent streams.
 *   x_dev   [batch][num_ch][*]  fp32, strides in floats; samples at index >= x_len read as zero
 *           (this is where net.py's mod-pad and look-ahead zero padding happen)
 *   emb_dev [batch][256]
 *   y_dev   [batch][num_src][*] fp32; samples 0 .. min(y_len, 128*frames)-1 are written
 * The state is advanced in place.  Asynchronous on `stream`. */
int l2h_sep_forward(void* handle, const float* x_dev, int64_t x_batch_stride, int64_t x_ch_stride,
                    int32_t x_len, const float* emb_dev, void* state_dev, float* y_dev,
                    int64_t y_batch_stride, int64_t y_ch_stride, int32_t y_len, int32_t batch,
                    int32_t frames, void* workspace_dev, size_t workspace_bytes, uint32_t flags,
                    void* stream);
/* l2h_sep_forward for a one-hop call (frames == 1) in which only some streams advance: stream b advances when
 * active_dev[b] != 0.  For any other stream nothing in its record changes (rings, h / c, tails, clock, gate memo), and its
 * rows of y_dev are not written; it may still be computed.  active_dev is [batch] bytes of DEVICE memory read when the
 * kernels run, so with L2H_FLAG_GRAPH a caller rewrites it in place before every hop and replays the same cached graph.
 * active_dev == NULL is l2h_sep_forward.  Errors 1: a mask with frames != 1 or with L2H_FLAG_TAPS. */
int l2h_sep_forward_active(void* handle, const float* x_dev, int64_t x_batch_stride, int64_t x_ch_stride,
                           int32_t x_len, const float* emb_dev, void* state_dev, float* y_dev,
                           int64_t y_batch_stride, int64_t y_ch_stride, int32_t y_len, int32_t batch,
                           int32_t frames, void* workspace_dev, size_t workspace_bytes, uint32_t flags,
                           void* stream, const uint8_t* active_dev);
/* A one-hop call over a chosen list of a state's records, so a hop costs what its n listed streams need, not what the
 * state's capacity needs.  Call row i reads x / emb row i, writes y row i and advances record slots_dev[i] of a state of
 * state_batch records.  The work, the kernel form and the workspace (l2h_sep_workspace_bytes(handle, n, 1, flags)) are
 * those of a dense call of n streams.  Records not listed are neither read nor written (rings, h / c, tails, gate memo,
 * clock); the header advances as for any call, and so do the clocks of the listed records.
 *   slots_dev  [n] int32 of DEVICE memory read when the kernels run: with L2H_FLAG_GRAPH a caller rewrites the list in place
 *              before every hop and replays the same cached graph (its key holds n, not the list's contents).  An entry
 *              outside [0, state_batch) marks a row that is computed but stores nothing (no record, no y row): a stream
 *              skipping this hop.  A slot listed twice is a caller error the call does not detect.
 * Errors 1, before anything is enqueued: null pointers, n <= 0, n > state_batch, L2H_FLAG_TAPS. */
int l2h_sep_forward_slots(void* handle, const float* x_dev, int64_t x_batch_stride, int64_t x_ch_stride, int32_t x_len,
                          const float* emb_dev, void* state_dev, int32_t state_batch, const int32_t* slots_dev, int32_t n,
                          float* y_dev, int64_t y_batch_stride, int64_t y_ch_stride, int32_t y_len,
                          void* workspace_dev, size_t workspace_bytes, uint32_t flags, void* stream);
/* l2h_sep_forward_slots for `frames` hops: every call row advances its record by `frames` hops in one call, so a listener
 * that fell behind catches up its backlog at once, or listed listeners run at a cadence of several hops.  The T hops of a
 * row run their BiLSTMs side by side as in a dense multi-hop call; only the inter-LSTM cells and the attention run in
 * frame order.  l2h_sep_forward_slots is this call with frames == 1.
 *   x_dev      row i holds 128*frames + 64 samples (x_len); y_dev row i receives 128*frames samples
 *   workspace  l2h_sep_workspace_bytes(handle, n, frames, flags), as for a dense call of n streams and `frames` hops
 *   slots_dev  as for l2h_sep_forward_slots; with L2H_FLAG_GRAPH the cached graph's key holds n and frames.  An entry
 *              outside [0, state_batch) marks a row that is computed from record 0 and stores nothing (no record, no y
 *              row) for all of its frames.
 * Every row advances by the same number of hops; listeners with different backlogs share one call through
 * l2h_sep_forward_slots_hops below, which gives each row its own count.  Records not listed are neither read nor
 * written; the header advances by `frames` as for any call.
 * Errors 1, before anything is enqueued: null pointers, n <= 0, n > state_batch, frames <= 0, L2H_FLAG_TAPS. */
int l2h_sep_forward_slots_frames(void* handle, const float* x_dev, int64_t x_batch_stride, int64_t x_ch_stride,
                                 int32_t x_len, const float* emb_dev, void* state_dev, int32_t state_batch,
                                 const int32_t* slots_dev, int32_t n, int32_t frames, float* y_dev,
                                 int64_t y_batch_stride, int64_t y_ch_stride, int32_t y_len, void* workspace_dev,
                                 size_t workspace_bytes, uint32_t flags, void* stream);
/* l2h_sep_forward_slots_frames in which row i advances its record by its own number of hops h = hops_dev[i], from 0 to
 * `frames` (T, the call's maximum), so listeners with different backlogs catch up in one call, and one graph cached for
 * (n, T) serves every mix of backlogs up to T.  The model is causal in time, so a row's first h hops of a T-hop call are
 * exactly those of an h-hop call; the call computes all T and stores only what h hops leave:
 *   x_dev      x_len = 128*frames + 64 as for l2h_sep_forward_slots_frames, but row i reads only its samples
 *              0 .. 128*h + 63: samples past 128*h + 64 are never read
 *   y_dev      row i receives samples 0 .. 128*h - 1; its later samples are not written
 *   record     its clock advances by h hops and by one call if h > 0; its rings, h / c, tails and gate memo end where h
 *              hops leave them.  h = 0 stores nothing (as a slot outside [0, state_batch) does)
 *   hops_dev   [n] int32 of DEVICE memory read when the kernels run, like slots_dev: with L2H_FLAG_GRAPH a caller rewrites
 *              it in place before every tick and replays the same cached graph (its key holds the pointer, not the
 *              contents).  An entry outside [0, frames] counts as 0.  NULL: every row advances `frames` hops, which is
 *              l2h_sep_forward_slots_frames.
 * The workspace, the argument errors (1, before anything is enqueued) and the header's advance by `frames` are those of
 * l2h_sep_forward_slots_frames. */
int l2h_sep_forward_slots_hops(void* handle, const float* x_dev, int64_t x_batch_stride, int64_t x_ch_stride,
                               int32_t x_len, const float* emb_dev, void* state_dev, int32_t state_batch,
                               const int32_t* slots_dev, const int32_t* hops_dev, int32_t n, int32_t frames,
                               float* y_dev, int64_t y_batch_stride, int64_t y_ch_stride, int32_t y_len,
                               void* workspace_dev, size_t workspace_bytes, uint32_t flags, void* stream);
/* Several enrolled speakers (targets) extracted from one mixture in one call: `batch` mixtures, K = n_targets targets each.
 * The front (STFT, conv encoder) and all of block 0 do not depend on the speaker (the speaker gate applies after block 0,
 * tfgridnet_causal.py:250-251), so they run once per mixture; blocks 1 .. B-1 and the back run once per target.
 *   x_dev      [batch] mixture rows, as for l2h_sep_forward
 *   emb_dev    [batch*K][256]: target row i*K + k is target k of mixture i
 *   y_dev      [batch*K] target rows, same order; y_batch_stride is the stride between consecutive target rows
 *   state_dev  an ordinary state of batch*K records (l2h_sep_state_bytes(handle, batch*K)), in groups of K: record i*K + k
 *              is target k of mixture i.  The group's lead record i*K also holds the mixture's conv tails and block 0's K/V
 *              rings and (h, c); in the group's other records those regions are never read or written.  Every record keeps
 *              its own embedding and gate memo, deconv and iSTFT tails, blocks 1 .. B-1 and clock, and the records of a
 *              group advance together, so their clocks stay equal.  A non-lead record is therefore not a standalone stream:
 *              it continues only inside its group (l2h_sep_state_reset_streams / _copy_streams of whole groups keep working).
 *   workspace  l2h_sep_workspace_bytes(handle, batch*K, frames, flags), as for a dense call of batch*K streams
 * Every kernel form is chosen for the batch*K target rows, and block 0 runs those same forms over the mixtures, so a target
 * row gets the arithmetic of a dense l2h_sep_forward of batch*K streams with each mixture repeated K times; one stage
 * differs: in the fused one-hop form (option "fused_tail") block 1's input projection runs as a separate rows GEMM rather
 * than inside block 0's tail kernel (rounding only).  n_targets == 1 is l2h_sep_forward, bit for bit.  L2H_FLAG_GRAPH works
 * (the cached graph's key holds K).
 * With targets, slot lists and per-row hop counts go through l2h_sep_forward_targets_groups below, which runs listed
 * groups of a larger state.  Not supported with targets: activity masks; the pipelined wavefront graph and
 * l2h_sep_stream_host / _dev; taps.  Non-lead records keep their (unused) block-0 area: there is no compact record.
 * Errors 1, before anything is enqueued: null pointers, batch, n_targets or frames <= 0, batch*n_targets*frames*97 rows
 * beyond the limit of one call, L2H_FLAG_TAPS. */
int l2h_sep_forward_targets(void* handle, const float* x_dev, int64_t x_batch_stride, int64_t x_ch_stride, int32_t x_len,
                            const float* emb_dev, void* state_dev, float* y_dev, int64_t y_batch_stride,
                            int64_t y_ch_stride, int32_t y_len, int32_t batch, int32_t n_targets, int32_t frames,
                            void* workspace_dev, size_t workspace_bytes, uint32_t flags, void* stream);
/* l2h_sep_forward_targets over a chosen list of a state's groups, each group advancing by its own number of hops: the
 * slot-list calls (l2h_sep_forward_slots_hops) for listeners who each want K = n_targets speakers.  The front and block 0
 * still run once per listed group, blocks 1 .. B-1 and the back once per target.
 *   state_dev  a state of state_batch = G*K records in the targets layout: record g*K + k is target k of group g, and g*K is
 *              the group's lead record (the state l2h_sep_forward_targets runs for G mixtures)
 *   groups_dev [n] int32 of DEVICE memory read when the kernels run: call row i is group groups_dev[i].  An entry outside
 *              [0, G) marks a group that is computed but stores nothing (no record, no y row): with a fixed n, a group
 *              missing the tick.  A group listed twice is a caller error the call does not detect.
 *   hops_dev   [n] int32 of DEVICE memory read when the kernels run, or NULL: every group advances `frames` hops.  Otherwise
 *              group i advances h = hops_dev[i] hops, from 0 to `frames` (T), as a row of l2h_sep_forward_slots_hops does:
 *              it reads only x samples 0 .. 128*h + 63 of its row, its K y rows receive samples 0 .. 128*h - 1 only, every
 *              record of the group advances its clock by h (and by one call if h > 0), and h = 0 stores nothing.  An entry
 *              outside [0, frames] counts as 0.
 *   x_dev      [n] mixture rows of 128*frames + 64 samples (x_len); row i is the mixture of group groups_dev[i]
 *   emb_dev    [n*K][256]: row i*K + k is target k of call row i, as for l2h_sep_forward_targets
 *   y_dev      [n*K] target rows, same order; y_batch_stride is the stride between consecutive target rows
 *   workspace  l2h_sep_workspace_bytes(handle, n*K, frames, flags), as for a targets call of n mixtures
 * Groups not listed are neither read nor written; the header advances by `frames` as for any call.  Every kernel form is
 * chosen for the n*K target rows, so a listed group gets the arithmetic of a dense l2h_sep_forward_targets of n groups, bit
 * for bit, in every form.  With L2H_FLAG_GRAPH one graph cached for (n, K, T) serves every tick: its key holds the list
 * pointers, not their contents, so a caller rewrites groups_dev and hops_dev in place before every tick.  n_targets == 1
 * is l2h_sep_forward_slots_hops.
 * Errors 1, before anything is enqueued: null pointers, n, n_targets or frames <= 0, a state_batch that is not a positive
 * multiple of n_targets, n > G, n*n_targets*frames*97 rows beyond the limit of one call, L2H_FLAG_TAPS. */
int l2h_sep_forward_targets_groups(void* handle, const float* x_dev, int64_t x_batch_stride, int64_t x_ch_stride,
                                   int32_t x_len, const float* emb_dev, void* state_dev, int32_t state_batch,
                                   const int32_t* groups_dev, const int32_t* hops_dev, int32_t n, int32_t n_targets,
                                   int32_t frames, float* y_dev, int64_t y_batch_stride, int64_t y_ch_stride,
                                   int32_t y_len, void* workspace_dev, size_t workspace_bytes, uint32_t flags, void* stream);
/* l2h_sep_forward_targets_groups for listeners who enrolled different numbers of speakers: every listener lists its own
 * target rows and their records, so one call, and one cached graph, serves any mix of one-, two- and three-speaker
 * listeners.  The front and block 0 run once per call row (listener), blocks 1 .. B-1 and the back once per target row.
 *   x_dev      [n] call rows of 128*frames + 64 samples (x_len): call row i is one listener's mixture
 *   emb_dev    [R][256], R = n_rows: target row r's embedding
 *   y_dev      [R] target rows; y_batch_stride is the stride between consecutive target rows
 *   records_dev [R] int32 of DEVICE memory: target row r continues record records_dev[r] of the state.  An entry outside
 *              [0, state_batch) marks a row that is computed but stores nothing.  Records need not be adjacent, aligned or
 *              in order, so any free records of a state serve a new listener; a record listed twice is a caller error the
 *              call does not detect.
 *   offsets_dev [n+1] int32 of DEVICE memory: call row i owns target rows offsets_dev[i] .. offsets_dev[i+1]-1.  Rows from
 *              offsets_dev[n] to R-1 belong to no listener and store nothing, so one fixed R carries any number of live
 *              targets.  The offsets are clamped on the device to be non-decreasing and <= R: a bad list gives empty
 *              listeners, never a read out of bounds.
 *   hops_dev   [n] int32 of DEVICE memory, or NULL: every call row advances `frames` hops.  Otherwise call row i advances
 *              h = hops_dev[i] hops, from 0 to `frames`, with the read, write and store rules of
 *              l2h_sep_forward_targets_groups: it reads only x samples 0 .. 128*h + 63, its target rows receive y samples
 *              0 .. 128*h - 1 only, and h = 0 stores nothing; every target row of the listener uses the same count.
 *   state_dev  a state of state_batch records.  A listener's lead record is records_dev[offsets_dev[i]], the record of its
 *              first target row: it also holds the listener's conv tails and block 0's K/V rings and (h, c), as the lead
 *              record g*K of a groups call does; the listener's other records never hold them.  A listener with no target
 *              row, or with a lead record outside the state, stores nothing at all.  The records of a listener advance
 *              together, so their clocks must be equal: start a listener's records together (l2h_sep_state_reset_streams
 *              of all of them), or add a record to a running listener with l2h_sep_join_targets below.  Dropping a
 *              non-lead row is leaving it out of the next call; dropping the lead is l2h_sep_state_move_lead first.
 *   workspace  l2h_sep_workspace_bytes(handle, n_rows, frames, flags)
 * All three lists are read when the kernels run: with L2H_FLAG_GRAPH one graph cached for (n, R, T) serves every tick, and
 * its key holds the list pointers, not their contents, so a caller rewrites records_dev, offsets_dev and hops_dev in place
 * before every tick.  Every kernel form is chosen for the R target rows, and block 0 runs those forms over the n call rows,
 * so with offsets i*K and records g_i*K + k this is l2h_sep_forward_targets_groups, bit for bit.  Not supported: activity
 * masks, the pipelined wavefront graph and l2h_sep_stream_host / _dev, taps.
 * Errors 1, before anything is enqueued: null pointers, n, n_rows or frames <= 0, n_rows > state_batch, n > n_rows,
 * n_rows*frames*97 rows beyond the limit of one call, L2H_FLAG_TAPS. */
int l2h_sep_forward_targets_rows(void* handle, const float* x_dev, int64_t x_batch_stride, int64_t x_ch_stride,
                                 int32_t x_len, const float* emb_dev, void* state_dev, int32_t state_batch,
                                 const int32_t* records_dev, const int32_t* offsets_dev, const int32_t* hops_dev,
                                 int32_t n, int32_t n_rows, int32_t frames, float* y_dev, int64_t y_batch_stride,
                                 int64_t y_ch_stride, int32_t y_len, void* workspace_dev, size_t workspace_bytes,
                                 uint32_t flags, void* stream);
/* Adding and dropping the targets of a running listener (INTEGRATION.md section 1).
 *
 * A block-0 history is hist_dev [state_batch][hist_frames][97*64] fp32 of DEVICE memory (24.8 KB per frame and record),
 * keyed by record: the ring of the last hist_frames frames of block 0's output (before the speaker gate) of a listener's
 * lead record, frame n of the record's own clock in slot n mod hist_frames.  Only leads' rings are written.
 *
 * l2h_sep_forward_targets_rows_history: l2h_sep_forward_targets_rows that also writes, for every listener that stores,
 * its h frames of block 0's output into its lead's ring (its last hist_frames of them when h > hist_frames).  y, the state and every other output are those of
 * l2h_sep_forward_targets_rows, bit for bit; the workspace is the same.  With L2H_FLAG_GRAPH the cached graph's key holds
 * hist_dev and hist_frames.  Errors 1, before anything is enqueued: those of l2h_sep_forward_targets_rows, a null hist_dev,
 * hist_frames < 1. */
int l2h_sep_forward_targets_rows_history(void* handle, const float* x_dev, int64_t x_batch_stride, int64_t x_ch_stride,
                                         int32_t x_len, const float* emb_dev, void* state_dev, int32_t state_batch,
                                         const int32_t* records_dev, const int32_t* offsets_dev, const int32_t* hops_dev,
                                         int32_t n, int32_t n_rows, int32_t frames, float* y_dev, int64_t y_batch_stride,
                                         int64_t y_ch_stride, int32_t y_len, void* workspace_dev, size_t workspace_bytes,
                                         uint32_t flags, void* stream, float* hist_dev, int32_t hist_frames);
/* l2h_sep_join_targets: J new target records, each brought up to the clock of a running listener's lead, so that the next
 * targets-rows call can list it among that listener's rows.  Row j:
 *   records_dev[j]  the record that joins; leads_dev[j] the lead record of the listener it joins.  Both [J] int32 lists of
 *              DEVICE memory, read when the kernels run (with L2H_FLAG_GRAPH the cached graph's key holds the pointers).
 *              A row whose record or lead lies outside [0, state_batch), whose record is another row's record, or whose
 *              record is a listed lead stores nothing (used 0).
 *   W_j        the frames the row replays: min(frames, hist_frames, p), p the lead's clock; 0 without a history.
 *   record     becomes a fresh record (as l2h_sep_state_reset_streams leaves it) with clock p - W_j, its gate memo is built
 *              from emb_dev[j] ([J][256]), and blocks 1 .. B-1 and the back then run over frames p - W_j .. p - 1 of the
 *              lead's history (the gate applied, as a targets call applies it): the record ends at clock p with its K/V
 *              rings, (h, c) and deconv / iSTFT tails warmed.  With a history covering the whole stream it is the record
 *              the target would have had, had it been listed from the start.  W_j = 0 (frames == 0, hist_dev NULL, or a
 *              lead at clock 0) is a cold join: fresh deep state at the lead's clock, nothing computed past the gate memo.
 *              The frames replayed must be in the lead's ring: every call that advanced the lead over them wrote it.
 *   y_dev      [J][num_src][*]: row j receives samples 0 .. 128*W_j - 1 (the replayed frames' output); the rest is not
 *              written.  May be NULL when no frame is replayed.
 *   used_dev   [J] int32 of DEVICE memory receiving W_j (0 for a row that stores nothing), or NULL.
 *   workspace  l2h_sep_workspace_bytes(handle, J, max(1, min(frames, hist_frames)), flags)
 * The lead's record is only read.  The header advances as for any call when frames are replayed.  A join reads its leads'
 * clocks and rings and shares the header's call counter with every call on the state, so it must be ordered with the
 * state's ticks on one stream (or by events), never run beside one.
 * Errors 1, before anything is enqueued: null pointers (y_dev only when frames are replayed), J <= 0, J > state_batch,
 * frames < 0, hist_frames < 1 with a history, J*frames*97 rows beyond the limit of one call, L2H_FLAG_TAPS. */
int l2h_sep_join_targets(void* handle, const int32_t* records_dev, const int32_t* leads_dev, const float* emb_dev, int32_t J,
                         void* state_dev, int32_t state_batch, const float* hist_dev, int32_t hist_frames, int32_t frames,
                         float* y_dev, int64_t y_batch_stride, int64_t y_ch_stride, int32_t* used_dev, void* workspace_dev,
                         size_t workspace_bytes, uint32_t flags, void* stream);

/* Streaming with HOST buffers (the end-to-end path).  Per round: H2D of the round's samples (+64
 * look-ahead) from pinned memory, the kernel chains, D2H of the new samples; one stream synchronise at
 * the end.  A round is one call of chunks_per_call hops -- or, for chunks_per_call == 1 with pipelining
 * enabled, a group of up to l2h_sep_pipeline_frames() one-hop calls that run as one wavefront-pipelined
 * graph (every hop is still its own T=1 chain with the state carried hop to hop).
 * x_host [batch][num_ch][x_len], y_host [batch][num_src][y_len]; x_stage_dev / y_stage_dev must hold
 * [batch][ch][128*G + 64] / [batch][src][128*G] floats with G = max(chunks_per_call, pipeline frames);
 * workspace from l2h_sep_stream_workspace_bytes(). */
int l2h_sep_stream_host(void* handle, const float* x_host, int32_t x_len, const float* emb_dev,
                        void* state_dev, float* y_host, int32_t y_len, int32_t batch,
                        int32_t n_calls, int32_t chunks_per_call, float* x_stage_dev,
                        float* y_stage_dev, void* workspace_dev, size_t workspace_bytes,
                        void* stream);

/* Streaming with DEVICE buffers: x_dev [batch][num_ch][x_len] holds whole clips, y_dev
 * [batch][num_src][y_len]; n_calls chained calls of chunks_per_call frames each, starting at the
 * beginning of x_dev and continuing the state.  Calls are CUDA-graph replays; the chunk a replay
 * works on is derived on the device from the state's frame counter.  With chunks_per_call == 1 the
 * one-hop chains of up to l2h_sep_pipeline_frames() consecutive hops are captured as ONE graph on 8
 * streams with (block, frame) wavefront dependencies, so different blocks work on different hops
 * concurrently (option "pipeline" = 0 runs the hops strictly one after the other).  Asynchronous. */
int l2h_sep_stream_dev(void* handle, const float* x_dev, int32_t x_len, const float* emb_dev,
                       void* state_dev, float* y_dev, int32_t y_len, int32_t batch, int32_t n_calls,
                       int32_t chunks_per_call, void* workspace_dev, size_t workspace_bytes, void* stream);

/* workspace for the two streaming entry points (one slot per in-flight hop when pipelining) and the
 * number of one-hop calls a pipelined graph holds (1 = pipelining off) */
int l2h_sep_stream_workspace_bytes(void* handle, int32_t batch, int32_t chunks_per_call, size_t* bytes);
int l2h_sep_pipeline_frames(void* handle, int32_t* frames);
/* runtime switches (the only way to change them: there are no environment variables).  0 | 1: "pipeline" (wavefront graph for
 * streams of one-hop calls), "pdl", "fused_tail" (one-hop calls of a few streams as 8 launches: front1_kernel, per block
 * the BiLSTM and the 16-CTA tail_kernel; default 1), "back_many" (calls of several frames / many streams through the persistent
 * front_many / back_many kernels; default 1), "fuse_ih" (default 0).  Values: "bf16" (0 = bf16x3 split products, 1 = bf16 weights x
 * split activations, 2 = plain bf16), "tc_lstm_min" (sequence-directions from which the recurrence runs on the tensor cores,
 * default 4096), "tc_pdl" (bit mask, default 7: programmatic launches around the tensor-core GEMMs of many-row chains),
 * "pipeline_gemm_shape" (0 | 1 | 2).  Counts: "pipeline_frames" (hops per graph, <= 500; 0 = as many as the workspace budget
 * holds), "pipeline_midb_hops" (hops per launch of the serial stage, <= 8) and the hops in flight per stage: "pipeline_lanes"
 * (BiLSTM, <= 16), "pipeline_midc_lanes" (<= 3), "pipeline_qkv_lanes" (<= 4), "pipeline_attn_lanes" (<= 4),
 * "pipeline_out_lanes" (<= 4), "pipeline_front_lanes" (<= 8), "pipeline_back_lanes" (<= 6).  "pipeline_pdl": bit mask of the
 * stages launched with programmatic dependent launch (front=1, W_ih gemm=2, bilstm=4, mid_a=8, mid_b=16, mid_c=32, qkv=64,
 * attention=128, attn_out=256, back=512; default 0).  "defaults" restores all pipeline settings.  The pipeline settings never
 * change results (bit-identical, tests/test_sep_gpu.py); "fused_tail", "bf16", "fuse_ih" and "tc_lstm_min" change rounding
 * only (gates in tests/). */
int l2h_sep_set_option(void* handle, const char* name, int32_t value);

/* where the tap area starts inside the workspace (floats) and its stage count; stage s holds
 * [batch*frames*97*64] floats: 0 = encoder out, then per block: after intra, after inter, block out */
int l2h_sep_tap_info(void* handle, int32_t batch, int32_t frames, int64_t* offset_floats,
                     int32_t* n_stages);

/* Measurement aid: run the chain `iters` times (after 2 warm-ups) with a CUDA event between every
 * launch on `stream`; returns, per kernel name (<= 64), the summed device time in ms and the launch
 * count.  Advances the state by (iters+2)*frames.  Synchronises. */
int l2h_sep_profile(void* handle, const float* x_dev, int32_t x_len, const float* emb_dev, void* state_dev,
                    float* y_dev, int32_t batch, int32_t frames, void* workspace_dev, size_t workspace_bytes,
                    int32_t iters, const char** names, float* ms_total, int32_t* counts, int32_t* n_names,
                    void* stream);

/* number of kernels one l2h_sep_forward of `frames` hops launches at a few streams (see l2h_sep_launch_count for the
   exact count of everything a handle launched, pipelined streams included) */
int l2h_sep_launches_per_forward(void* handle, int32_t frames, int32_t* n);

/* kernels this handle has launched so far (a CUDA-graph replay counts its kernel nodes); reset != 0 zeroes the
   counter after reading.  bench.py's gpu_launches is read from here around the timed region. */
int l2h_sep_launch_count(void* handle, int64_t* kernels, int32_t reset);

/* diagnostics: device-side timeline of the separator's kernels.  l2h_sep_trace_start(handle, capacity) allocates a buffer
   of `capacity` records and switches tracing on (capacity 0: off); from then on thread 0 of the first CTA of every
   instrumented kernel stores one 32-byte record {u64 t0_ns, u64 t1_ns (globaltimer at entry / exit), u64 activation
   pointer, u32 kernel id (0 front, 1 W_ih gemm, 2 bilstm, 3 mid_a, 4 mid_b, 5 mid_c, 6 qkv, 7 attention, 8 attn_out,
   9 back, 10 fused mid), u32 SM}.  l2h_sep_trace_read synchronises, copies up to max_records of them to the host and
   restarts the trace.  Used by tools/pipe_trace.py; costs one atomic per kernel while on, one load while off. */
int l2h_sep_trace_start(void* handle, int32_t capacity);
int l2h_sep_trace_read(void* handle, void* records_host, int32_t max_records, int32_t* n_records);

/* ---- enrollment network (EmbedTFGridNet, configs/embed.json:5-10) ---------------------------- */
typedef struct l2h_embed_config {
    int32_t embed_dim;  /* 256 */
    int32_t num_ch;     /* 2   */
    int32_t n_fft;      /* 128 */
    int32_t stride;     /* 64  */
    int32_t num_blocks; /* 3   */
} l2h_embed_config;

int l2h_embed_create(const l2h_embed_config* cfg, void** handle);
int l2h_embed_destroy(void* handle);
/* name = a key of the reference EmbedTFGridNet state_dict (espnet2 naming: "blocks.0.intra_norm.gamma",
 * "blocks.0.attn_conv_Q_0.0.weight", "embed_proj.0.weight", ...); HOST fp32.  The unused deconv.* tensors
 * are accepted and ignored. */
int l2h_embed_load_weight(void* handle, const char* name, const float* host_data, int64_t numel);
int l2h_embed_weights_expected(void* handle, int32_t* n_expected, int32_t* n_loaded);
int l2h_embed_commit_weights(void* handle, void* stream);
/* workspace of one forward call of `batch` utterances padded to n_samples; it includes batch * 4 bytes for the device
 * copy of the lengths of l2h_embed_forward_lengths */
int l2h_embed_workspace_bytes(void* handle, int32_t batch, int32_t n_samples, size_t* bytes);
/* "bf16" (the separator's mapping): 0 (default): every tensor-core product is formed from bf16 hi/lo splits of both fp32
 * operands in three MMA passes (fp32-grade, relative error ~2^-16 per product); 1: bf16 weights x split activations (two
 * passes); 2: plain bf16 operands (one pass).
 * "tc_lstm_min" (default 2048): the sequence-directions of one recurrence from which it runs on the tensor cores
 * (tc_lstm) instead of the CUDA cores (lstm_rec).  The choice is made per call from the padded batch, so a short
 * utterance alone can take the other kernel family than inside a long batch; set it to 1 (always tensor cores) or
 * above any batch (never) to compare results of the same recurrence arithmetic. */
int l2h_embed_set_option(void* handle, const char* name, int32_t value);
/* largest batch one l2h_embed_forward call should be given for utterances of n_samples (workspace bound) */
int l2h_embed_max_batch(void* handle, int32_t n_samples, int32_t* max_batch);
/* x_dev [batch][2][n_samples] fp32 contiguous -> emb_dev [batch][256].  Asynchronous on `stream`.
 * The same as l2h_embed_forward_lengths with lengths_host = NULL. */
int l2h_embed_forward(void* handle, const float* x_dev, float* emb_dev, int32_t batch, int32_t n_samples,
                      void* workspace_dev, size_t workspace_bytes, void* stream);
/* Utterances of different lengths in one call.  x_dev [batch][2][n_max] fp32 contiguous; utterance b is
 * x_dev[b][:][0 .. lengths_host[b]) and row b of emb_dev [batch][256] is its embedding as if it were embedded alone.
 * Samples at index >= lengths_host[b] are never read (they may hold anything, NaN included).  lengths_host is a HOST
 * array of `batch` sample counts, read during the call only; NULL means every utterance is n_max long.  Each length must
 * lie in [192, n_max] (192 samples = the 4 STFT frames of the unfold).  Size the workspace with
 * l2h_embed_workspace_bytes(batch, n_max) and the batch with l2h_embed_max_batch(n_max).  The utterances are computed
 * padded to n_max, so the cost is that of `batch` utterances of n_max samples.
 * Errors, returned before anything is enqueued and before the weights are checked: 1 = a null pointer, batch <= 0, a
 * length outside [192, n_max], or a workspace smaller than the query.  Asynchronous on `stream`. */
int l2h_embed_forward_lengths(void* handle, const float* x_dev, int32_t n_max, const int32_t* lengths_host, int32_t batch,
                              float* emb_dev, void* workspace_dev, size_t workspace_bytes, void* stream);
/* Enrollment from listeners' own streams: row b embeds the last used_b = min(lengths_host[b], captured) samples that slot
 * s = slots[b] of an enrollment capture (l2h_enroll_capture below) holds, read from its ring in place, with no gather copy
 * and nothing read back to the host.  Row b is l2h_embed_forward_lengths of those samples in a batch padded to n_max, bit
 * for bit.
 *   capture_dev  the capture's state [n_slots][2][row_floats] (l2h_enroll_capture_layout(capacity)), written by earlier
 *                work on `stream`
 *   slots_host / slots_dev  exactly one is non-NULL: a HOST array of `batch` distinct slots in [0, n_slots), read during the
 *                call only, or `batch` int32 of DEVICE memory read when the kernels run, where an entry outside [0, n_slots)
 *                marks a row that embeds nothing
 *   lengths_host HOST array of `batch` lengths in [192, n_max], read during the call only
 *   emb_dev      row b goes to emb_dev + b * emb_row_stride (>= 256 floats), so it can land in a row of the separator's
 *                embedding staging buffer.  A row with used_b < 192 (the slot captured too little) is not written: its
 *                listener keeps the embedding it had.
 *   used_dev     [batch] int32 of DEVICE memory: used_b, or 0 for a row that was not written
 *   workspace    l2h_embed_workspace_bytes(batch, n_max), as for l2h_embed_forward_lengths; n_max <= capacity
 * Errors, returned before anything is enqueued and before the weights are checked: 1 = a null pointer, both or neither slot
 * list, batch or n_slots <= 0, batch > n_slots, capacity < 192, n_max outside [192, capacity], emb_row_stride < 256, a length
 * outside [192, n_max], a host slot outside [0, n_slots) or listed twice, or a workspace smaller than the query.
 * Asynchronous on `stream`. */
int l2h_embed_forward_slots(void* handle, const float* capture_dev, int32_t n_slots, int32_t capacity, const int32_t* slots_host,
                            const int32_t* slots_dev, const int32_t* lengths_host, int32_t batch, int32_t n_max, float* emb_dev,
                            int64_t emb_row_stride, int32_t* used_dev, void* workspace_dev, size_t workspace_bytes, void* stream);
/* Enrollment from a capture in slices: l2h_embed_forward_slots cut into an ordered plan of units, each one stage of one or
 * a few kernel launches, so a service can put a bounded amount of enrollment work between its ticks.  *units receives the
 * number of units of the plan for (batch, n_max, window): 2 + num_blocks * (8 + w), where w = ceil((1 + n_max / 64 - 3) /
 * window) windows of the inter-frame recurrence, or w = 1 for window = 0 or a window at least that long.  Error 1: a null
 * pointer, batch <= 0, n_max < 192 or window < 0. */
int l2h_embed_slots_units(void* handle, int32_t batch, int32_t n_max, int32_t window, int32_t* units);
/* Enqueues units [first_unit, first_unit + n_units) of that plan on `stream`.  The other arguments are those of
 * l2h_embed_forward_slots, and all units run in one call equal it, bit for bit, for every window.
 *   - Every unit runs exactly once, in order; every call passes the same arguments and the same workspace.
 *   - Between calls the stream may run any work that does not touch that workspace, emb_dev rows or used_dev: ticks that
 *     keep writing the capture and ticks that read the staging rows emb_dev points into included.  The embedding is that
 *     of the samples the capture held when unit 0 ran.
 *   - used_dev is final after unit 0.  emb_dev rows are written by the last unit only: until then a listener keeps the
 *     embedding it had.
 *   - The workspace is l2h_embed_workspace_bytes(batch, n_max), as for l2h_embed_forward_slots: the (h, c) the windows of
 *     the recurrence carry live in it.
 * Errors, returned before anything is enqueued: every error of l2h_embed_forward_slots (host slot lists are checked on
 * every call), and 1 = window < 0, n_units < 1, or a unit range outside the plan.  Asynchronous on `stream`. */
int l2h_embed_forward_slots_units(void* handle, const float* capture_dev, int32_t n_slots, int32_t capacity,
                                  const int32_t* slots_host, const int32_t* slots_dev, const int32_t* lengths_host, int32_t batch,
                                  int32_t n_max, float* emb_dev, int64_t emb_row_stride, int32_t* used_dev, void* workspace_dev,
                                  size_t workspace_bytes, int32_t window, int32_t first_unit, int32_t n_units, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Evaluation epilogue on the device (replaces the CPU metric code after `outputs.cpu()` in
 * src/ts_hear_test.py:139-146): per mixture b, out_dev[b] = { output_sisnr, si_snr_i, embedding_sim }
 *   output_sisnr  = mean over channels of SI-SNR(est, target)                 (torchmetrics definition, zero-mean)
 *   si_snr_i      = mean over channels of SI-SNR(est, target) - SI-SNR(mixture, target)   (0 if mixture_dev is NULL)
 *   embedding_sim = cosine similarity of emb and emb_gt                        (0 if either is NULL)
 * SI-SNR is computed in double in torchmetrics' order: the means, then the centred sums and alpha, then the residual
 * energy |alpha t~ - p~|^2 directly (three passes over each row), so a DC offset on the signals costs no precision.
 * The cosine clamps each norm to 1e-8 separately, as F.cosine_similarity does.
 * est / target / mixture: [batch][channels][n_samples] fp32 contiguous on the device (est = the separator's output
 * buffer); emb / emb_gt: [batch][emb_dim].  Asynchronous on `stream`; the caller copies 3 floats per mixture back. */
int l2h_eval_metrics(const float* est_dev, const float* target_dev, const float* mixture_dev, int32_t batch, int32_t channels,
                     int32_t n_samples, const float* emb_dev, const float* emb_gt_dev, int32_t emb_dim, float* out_dev,
                     void* stream);

/* ------------------------------------------------------------------------------------------------
 * Binaural rendering of mono events on the device (the data-side arithmetic of the reference's simulators):
 *   events[b][s][ear] = convolve(src[b][s], rir[b][s][ear])[:n_samples]      src/datasets/multi_ch_simulator.py:56-58
 *   noise scaled by noise_scale[b]; norm = max|sum(events) + noise|; if norm > 1 events and noise are divided by it;
 *   mixture = sum(events) + noise                                   src/datasets/MixLibriSpeechNoisyEnrollNorm.py:179-202
 * src_dev [batch][n_src][n_samples] mono; rir_dev [batch][n_src][2][rir_len] (already at the sampling rate of src:
 * l2h_resample brings responses stored at another rate there); noise_dev [batch][2][n_samples] or NULL; noise_scale_dev
 * [batch] or NULL (= 1); events_dev [batch][n_src][2][n_samples]; mixture_dev [batch][2][n_samples]; norm_dev [batch] or
 * NULL; scratch_dev: batch * 4 bytes.  Asynchronous on `stream`. */
int l2h_render_binaural(const float* src_dev, const float* rir_dev, const float* noise_dev, const float* noise_scale_dev,
                        int32_t batch, int32_t n_src, int32_t n_samples, int32_t rir_len, float* events_dev,
                        float* mixture_dev, float* norm_dev, void* scratch_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Band-limited resampling of many rows in one call: torchaudio.functional.resample(row, orig_freq[r], new_freq) at its
 * defaults (Hann-windowed sinc, lowpass_filter_width 6, rolloff 0.99) -- impulse responses from the rate of their file
 * to the dataset rate (src/datasets/multi_ch_simulator.py:49) and the dataset's resample_rate step
 * (MixLibriSpeechNoisyEnrollNorm.py:69-75).  Other methods or parameters are not implemented.
 *   x_dev       [n_rows] rows of n_in fp32 samples, x_row_stride floats apart (>= n_in)
 *   orig_freq   HOST array of n_rows rates in Hz, one per row; new_freq the rate of every output row
 *   y_dev       [n_rows] rows of y_capacity fp32 samples, y_row_stride floats apart (>= y_capacity); must not overlap x
 * Row r gets n_out(r) = ceil(new_freq * n_in / orig_freq[r]) resampled samples (computed exactly in integers; a row
 * with orig_freq[r] == new_freq is copied bit for bit), then zeros up to y_capacity -- rows of different rates come out
 * zero-padded to a common length.  Errors, returned before anything is enqueued: 1 = null pointer, bad size or stride,
 * a rate <= 0, or some n_out(r) > y_capacity; 2 = a reduced rate ratio orig/new too large for the kernel's input
 * window (downsampling by more than about 45x).  Asynchronous on `stream`; orig_freq is read during the call only. */
int l2h_resample(const float* x_dev, int64_t x_row_stride, int32_t n_in, int32_t n_rows, const int32_t* orig_freq,
                 int32_t new_freq, float* y_dev, int64_t y_row_stride, int32_t y_capacity, void* stream);

/* Streaming resampling for a list of a state's slots: devices at 48, 32, 24 or 8 kHz into and out of the 16 kHz
 * separator, one push of `block` input samples per 8 ms tick.  With the rates reduced by their gcd to o and q and
 * w = ceil(6 o / (0.99 min(o, q))) taps per side (as in l2h_resample), `block` must be a positive multiple of o, and each
 * push yields out_block = block * q / o samples.  A stream's output is z, the l2h_resample output of everything it has
 * been pushed as one signal, delayed by delay = D = floor(w q / o) samples, with zeros before z's start: after k pushes
 * it has returned k * out_block samples, and every one of them is bit for bit the matching sample of z (the ones of z
 * whose taps have all arrived).  Equal rates, and rates whose 8 ms is not a whole number of samples (44.1 kHz family),
 * are refused.
 *
 * The state is [n_slots][channels][hist + keep] fp32 of DEVICE memory: per channel the trailing input samples the next
 * push reads, then the last `keep` outputs.  All zeros is a fresh stream (zero samples before its start), so a slot is
 * reset by zeroing its rows and moved by copying them.
 *
 * l2h_resample_stream_layout: hist (H), delay (D) and out_block of a stream.  Errors: 1 = null pointer, a rate <= 0, equal
 * rates, a block that is not a positive multiple of o, keep < 0; 2 = the staged window of one push (hist + block + keep +
 * out_block samples) exceeds the kernel's shared memory.
 *
 * l2h_resample_stream: row i of a call pushes h = hops_dev[i] blocks (`blocks` = T, the call's maximum, when hops_dev is
 * NULL) into slot slots_dev[i] of the state:
 *   x_dev      [n][channels][blocks * block] fp32, strides in floats; row i reads only its first h * block samples
 *   y_dev      [n][channels][keep + blocks * out_block] fp32; row i receives y[i][c][0 .. keep + h * out_block): the last
 *              keep + h * out_block samples of its stream's delayed output (the keep window, then the h new pushes' samples;
 *              what precedes the stream's start reads as 0).  Its later samples are not written.  Must not overlap x or
 *              the state.
 *   slots_dev  [n] int32 of DEVICE memory read when the kernel runs, like l2h_sep_forward_slots_hops's list: an entry
 *              outside [0, n_slots) marks a row that stores nothing (neither its y row nor any state row).  A slot listed
 *              twice is a caller error the call does not detect.
 *   hops_dev   [n] int32 of DEVICE memory read when the kernel runs, or NULL (every row pushes `blocks`).  h = 0, or an entry
 *              outside [0, blocks], stores nothing.
 * So a service passes the same slot and hop tensors to the resampler and the separator, and a call captured in a CUDA graph
 * serves any list of the same n rewritten in place.  One launch; nothing on the host is read from the device.
 * Errors, returned before anything is enqueued: 1 = null pointers, n, channels, blocks or n_slots <= 0, n > n_slots,
 * channel or row strides under the lengths above, and the layout's errors 1; 2 = the staged window of one row (hist +
 * blocks * block + keep + blocks * out_block samples) exceeds the kernel's shared memory.  Asynchronous on `stream`. */
int l2h_resample_stream_layout(int32_t orig_freq, int32_t new_freq, int32_t block, int32_t keep, int32_t* hist,
                               int32_t* delay, int32_t* out_block);
int l2h_resample_stream(const float* x_dev, int64_t x_row_stride, int64_t x_ch_stride, float* y_dev, int64_t y_row_stride,
                        int64_t y_ch_stride, int32_t n, int32_t channels, int32_t blocks, const int32_t* slots_dev,
                        const int32_t* hops_dev, float* state_dev, int32_t n_slots, int32_t orig_freq, int32_t new_freq,
                        int32_t block, int32_t keep, void* stream);

/* Streaming resampling of pushes of any length, for a list of a state's slots: devices at 44.1, 22.05 or 11.025 kHz (whose
 * 8 ms is no whole number of samples), and clients that send 10 ms packets, at any rate, into and out of the 16 kHz
 * separator.  With o, q and w as in l2h_resample_stream and D = floor(w q / o), a stream that has been pushed N samples
 * in all has returned exactly floor(N q / o) samples, and they are bit for bit the first floor(N q / o) samples of z
 * delayed by D (z the l2h_resample output of everything it was pushed as one signal, zeros before z's start): the same
 * output and delay as l2h_resample_stream with keep 0, whose pushes of whole periods give the same bits.
 *
 * The state is [n_slots][channels][row_floats] fp32 of DEVICE memory: per channel the count of outputs made (capped at D)
 * and the input count modulo o, both exact in a float, then the last ceil((D + 1) o / q) + w + 1 input samples.  All
 * zeros is a fresh stream, so a slot is reset by zeroing its rows and moved by copying them.
 *
 * l2h_resample_packets_layout: row_floats, delay (D) and max_out = ceil(max_in q / o), the most samples one push of up to
 * max_in samples returns.  Errors: 1 = null pointer, a rate <= 0, equal rates, max_in <= 0; 2 = the staged window of one
 * push (the history and max_in samples) exceeds the kernel's shared memory.
 *
 * l2h_resample_packets: row i of a call pushes c_i * unit samples, c_i = counts_dev[i], into slot slots_dev[i]:
 *   x_dev           [n][channels][max_in] fp32, strides in floats; row i reads only its first c_i * unit samples
 *   y_dev           [n][channels][max_out] fp32; row i receives y[i][c][0 .. m_i), the m_i samples its push makes final.
 *                   Its later samples are not written.  Must not overlap x or the state.
 *   counts_dev      [n] int32 of DEVICE memory read when the kernel runs; c_i * unit outside [0, max_in] counts as 0.
 *                   unit = 1 counts samples; unit = 128 takes the separator's hop counts (l2h_hop_fifo's hops_dev) as they
 *                   are, for the way back out of it.
 *   out_counts_dev  [n] int32 of DEVICE memory: m_i, 0 for a row that stores nothing.
 *   slots_dev       [n] int32 of DEVICE memory read when the kernel runs, like l2h_resample_stream's: an entry outside
 *                   [0, n_slots) marks a row that stores nothing (no y sample, no state row).  So does a push of 0 samples.
 * One launch; nothing on the host is read from the device, and a call captured in a CUDA graph serves any lists of the
 * same n rewritten in place.  Errors, returned before anything is enqueued: 1 = null pointers, n, channels, unit or n_slots
 * <= 0, n > n_slots, channel or row strides under the lengths above, and the layout's errors 1; 2 = as for the layout.
 * Asynchronous on `stream`. */
int l2h_resample_packets_layout(int32_t orig_freq, int32_t new_freq, int32_t max_in, int32_t* row_floats, int32_t* delay,
                                int32_t* max_out);
int l2h_resample_packets(const float* x_dev, int64_t x_row_stride, int64_t x_ch_stride, float* y_dev, int64_t y_row_stride,
                         int64_t y_ch_stride, int32_t n, int32_t channels, int32_t max_in, const int32_t* counts_dev,
                         int32_t unit, int32_t* out_counts_dev, const int32_t* slots_dev, float* state_dev, int32_t n_slots,
                         int32_t orig_freq, int32_t new_freq, void* stream);

/* A per-slot hop FIFO: 16 kHz pieces of any length in, the separator's chunks and per-row hop counts out, so one tick runs
 * from device memory (packets in, l2h_resample_packets, l2h_hop_fifo, l2h_sep_forward_slots_hops, l2h_resample_packets
 * with unit 128) with no count read back to the host.  A slot's signal is 64 zeros, then every sample appended since it
 * was reset; p is its read position (0 when fresh), and the slot holds the samples past p + 64.
 *
 * l2h_hop_fifo: row i appends c_i * unit samples of x row i to slot slots_dev[i] (c_i = counts_dev[i], the count and slot
 * rules of l2h_resample_packets), then pops h_i = min(frames, floor(held / 128)) hops, held counted after the append:
 *   chunk_dev   [n][channels][128 * frames + 64] fp32; row i receives chunk[i][c][0 .. 128 h_i + 64), samples
 *               [p, p + 128 h_i + 64) of its slot's signal (the l2h_sep_forward_slots_hops chunk of h_i hops), and p
 *               advances by 128 h_i: the last 64 samples stay as the next chunk's start.  Its later samples are not written.
 *   hops_dev    [n] int32 of DEVICE memory: h_i, 0 for a row whose slot lies outside [0, n_slots) (it stores nothing).
 * So the same slot list and hops_dev go straight to l2h_sep_forward_slots_hops, and a row with count 0 still drains the
 * whole hops its slot holds.  Samples past the slot's `capacity` are dropped (the held ones stay intact) and added to the
 * slot's dropped-sample counter, which shows a client that sends faster than it is served; nothing is read or written out
 * of bounds.
 *
 * The state is [n_slots][channels][row_floats] fp32 of DEVICE memory: per channel three int32 words stored in the floats'
 * bits (p modulo the ring, the samples held, the samples dropped, saturating at 2^31 - 1), then a ring of 64 + capacity
 * samples.  All zeros is an empty FIFO, so a slot is reset by zeroing its rows and moved by copying them.
 * l2h_hop_fifo_layout: row_floats = 3 + 64 + capacity.  Errors: 1 = null pointer, capacity < 128 (one hop).
 *
 * One launch.  Errors, returned before anything is enqueued: 1 = null pointers, n, channels, max_in, unit, frames or
 * n_slots <= 0, n > n_slots, channel or row strides under the lengths above, and the layout's errors.  Asynchronous on
 * `stream`. */
int l2h_hop_fifo_layout(int32_t capacity, int32_t* row_floats);
int l2h_hop_fifo(const float* x_dev, int64_t x_row_stride, int64_t x_ch_stride, int32_t max_in, const int32_t* counts_dev,
                 int32_t unit, float* chunk_dev, int64_t chunk_row_stride, int64_t chunk_ch_stride, int32_t* hops_dev,
                 int32_t n, int32_t channels, int32_t frames, const int32_t* slots_dev, float* state_dev, int32_t n_slots,
                 int32_t capacity, void* stream);

/* A per-slot enrollment capture: the recent 16 kHz input of each listener, kept on the device as it streams, so an
 * enrollment (l2h_embed_forward_slots) needs no copy of the audio on the host.
 *
 * l2h_enroll_capture: row i appends samples 64 .. 64 + 128 h - 1 of its chunk, h = hops_dev[i], to slot slots_dev[i]: the
 * hops' new samples, without the look-ahead that the next chunk repeats.  It takes the chunk, slot and hop tensors that
 * l2h_hop_fifo gives l2h_sep_forward_slots_hops:
 *   chunk_dev   [n][channels][128 * frames + 64] fp32, strides in floats; row i reads only samples 64 .. 128 h + 63
 *   slots_dev   [n] int32 of DEVICE memory read when the kernel runs: an entry outside [0, n_slots) marks a row that stores
 *               nothing.  A slot listed twice is a caller error the call does not detect.
 *   hops_dev    [n] int32 of DEVICE memory read when the kernel runs: h = 0, or an entry outside [0, frames], stores nothing.
 * So a call captured in a CUDA graph with l2h_hop_fifo and l2h_sep_forward_slots_hops serves any lists of the same n
 * rewritten in place.  A slot keeps its last `capacity` samples.
 *
 * The state is [n_slots][channels][row_floats] fp32 of DEVICE memory: per channel two int32 words stored in the floats' bits
 * (the write position in the ring, the samples captured since reset, capped at capacity), then a ring of capacity samples.
 * All zeros is an empty capture, so a slot is reset by zeroing its rows and moved by copying them.
 * l2h_enroll_capture_layout: row_floats = 2 + capacity.  Errors: 1 = null pointer, capacity < 192 (the shortest enrollment).
 *
 * One launch.  Errors, returned before anything is enqueued: 1 = null pointers, n, channels, frames or n_slots <= 0,
 * n > n_slots, channel or row strides under the chunk's length, and the layout's errors.  Asynchronous on `stream`. */
int l2h_enroll_capture_layout(int32_t capacity, int32_t* row_floats);
int l2h_enroll_capture(const float* chunk_dev, int64_t chunk_row_stride, int64_t chunk_ch_stride, int32_t n, int32_t channels,
                       int32_t frames, const int32_t* slots_dev, const int32_t* hops_dev, float* state_dev, int32_t n_slots,
                       int32_t capacity, void* stream);

/* A per-listener target mixer: the separated voices of each listener (the target rows of l2h_sep_forward_targets_rows) and,
 * optionally, a little of its unprocessed mixture ("transparency") summed into one row per listener, each term scaled by
 * a gain that ramps smoothly when it changes, so a voice that joins or drops fades in or out instead of clicking.
 *
 * The state is [n_records + n_slots][channels][row_floats] fp32 of DEVICE memory: one ramp per separator record and
 * channel, then one per listener slot and channel for the ambient term.  A ramp (g0, g1, F, p) goes from g0 to g1 over F
 * samples, p of them mixed already (words 2 and 3 are int32 words stored in the floats' bits: F + 1, 0 for a row never
 * set, and p).  The sample at ramp position q (q = p for the next one mixed) is mixed at
 *     G(q) = g1                                              if q + 1 >= F   (F = 0: an immediate change)
 *          = g0 + (g1 - g0) (1 - cos(pi (q + 1) / F)) / 2     otherwise       (a raised cosine, fp32, cospif)
 * so a ramp ends exactly at g1, and a sample's gain depends only on its position in the ramp.  All
 * zeros is a fresh row: a record settled at gain 1, a slot settled at ambient gain 0.  So a row is reset by zeroing it and
 * moved by copying it.  A record's or slot's channels are written only by the CTAs of that channel.
 * l2h_target_mix_layout: row_floats = 4.  Errors: 1 = null pointer.
 *
 * l2h_target_mix: listener row i (h = hops_dev[i], or frames without hops) writes, for s < 128 h,
 *     out[i][c][s] = sum over its target rows r, in row order, of G_r(s) y[r][c][s]  +  A_i(s) chunk[i][c][s]
 *   y_dev        [R][channels][128 * frames] fp32, strides in floats: the y of l2h_sep_forward_targets_rows
 *   chunk_dev    [n][channels][128 * frames + 64] fp32, the separator's input of the same call, or NULL: no ambient term.
 *                chunk[i][c][0 .. 128 h) is exactly the stretch of the mixture that y[r][c][0 .. 128 h) estimates, with
 *                the same 64-sample look-ahead delay, so the ambient term is time-aligned with no buffer of its own.
 *   out_dev      [n][channels][128 * frames] fp32: row i receives out[i][c][0 .. 128 h); its later samples are not
 *                written.  Must not overlap y or the chunk.
 *   records_dev  [R] int32 of DEVICE memory: target row r's gain is record records[r]'s ramp; a record outside
 *                [0, n_records) marks a row that is skipped.  A record listed twice is a caller error the call does not
 *                detect.
 *   offsets_dev  [n + 1] int32 of DEVICE memory: row i owns target rows offsets[i] .. offsets[i+1]-1, the offsets clamped
 *                as l2h_sep_forward_targets_rows clamps them (non-decreasing, at most R); rows from offsets[n] on belong to
 *                nobody and are not read.
 *   hops_dev     [n] int32 of DEVICE memory, or NULL (every row mixes frames hops)
 *   slots_dev    [n] int32 of DEVICE memory: row i's ambient gain is slot slots[i]'s ramp.
 * G_r(s) and A_i(s) are the ramps' G at positions p + s; the call advances every ramp it mixes by 128 h (the ambient ramp
 * too when chunk_dev is NULL: it keeps the listener's clock).  Each sample's sum starts at -0 and takes, with fmaf in the
 * order above, every term whose gain at that sample is nonzero.  fmaf(g, x, -0) is g x exactly, so the first such term
 * starts the sum with nothing added to a zero: one target at unity gain gives y itself, and several at unity with no
 * ambient give their fp32 sum in row order, bit for bit.  A sample that no term enters is -0, so a row that stores but
 * has no live term writes zeros.  A term at gain 0 never reaches a sample, not even as the sign of a zero or a NaN in its
 * input, and a term whose gain is 0 for every sample of the call is not read at all.  So the output depends only on the
 * samples' gains, and cutting the hops differently changes no bit of it.  A row whose slot lies outside [0, n_slots), or whose h lies outside [1, frames], stores nothing and
 * advances no ramp.  The output of l2h_sep_forward_targets_groups (K targets per group) is served as y [n K][channels]
 * [128 frames] with offsets i K and records g_i K + k.  All lists are read when the kernel runs, so a call captured in a
 * CUDA graph with l2h_hop_fifo, l2h_sep_forward_targets_rows and l2h_resample_packets serves any lists of the same n and R
 * rewritten in place.  One launch.  Errors, returned before anything is enqueued: 1 = null pointers (chunk_dev may be
 * NULL), n, R, channels, frames, n_records or n_slots <= 0, n > R, n > n_slots, channel or row strides under the lengths
 * above, out overlapping y or the chunk.  y and the chunk share the one `channels` count, so a chunk whose channels differ
 * from y's cannot be passed here (TargetMixer refuses it by shape).  Asynchronous on `stream`.
 *
 * l2h_target_mix_set: entry e sets the ramp of state row rows_dev[e] (a record b as row b, a slot s as row n_records + s) in
 * every channel to (g0, gains_dev[e], fades_dev[e], 0): a fade to gains_dev[e] over fades_dev[e] samples, starting at
 * starts_dev[e], or, with starts_dev NULL, at the gain of the last sample mixed (a fresh row: its rest gain), so changing a
 * ramp halfway never jumps.  rows_dev, gains_dev, starts_dev and fades_dev are [n] arrays of DEVICE memory read when the
 * kernel runs, so a set can run from a CUDA graph; a row outside [0, n_records + n_slots), or a fade outside
 * [0, 2^31 - 2], marks an entry that stores nothing.  A row listed twice is a caller error the call does not detect.
 * Enqueue a set on the stream of the mixer's calls, between them: a set that runs while a mix call reads the same ramps
 * races with it.  One launch.  Errors, returned before anything is enqueued: 1 = null pointers (starts_dev may be NULL),
 * n_records, n_slots, channels or n <= 0.  The fades live in device memory and are read when the kernel runs, so a
 * negative fade is no argument error: it marks an entry that stores nothing (TargetMixer refuses it in host lists).
 * Asynchronous on `stream`. */
int l2h_target_mix_layout(int32_t* row_floats);
int l2h_target_mix(const float* y_dev, int64_t y_row_stride, int64_t y_ch_stride, const float* chunk_dev,
                   int64_t chunk_row_stride, int64_t chunk_ch_stride, float* out_dev, int64_t out_row_stride,
                   int64_t out_ch_stride, int32_t n, int32_t R, int32_t channels, int32_t frames, const int32_t* records_dev,
                   const int32_t* offsets_dev, const int32_t* hops_dev, const int32_t* slots_dev, float* state_dev,
                   int32_t n_records, int32_t n_slots, void* stream);
int l2h_target_mix_set(float* state_dev, int32_t n_records, int32_t n_slots, int32_t channels, const int32_t* rows_dev,
                       int32_t n, const float* gains_dev, const float* starts_dev, const int32_t* fades_dev, void* stream);

/* A per-slot look-ahead peak limiter: each listener's output kept under a ceiling, with one gain for all channels at each
 * sample, so interaural level ratios are preserved.  Put it after the up-resampler, on the samples the device plays:
 * band-limited upsampling of a limited 16 kHz signal can overshoot the ceiling between its samples.
 *
 * Gains live in an integer log domain of Q = 65536 quanta per octave of amplitude.  At input sample k of a slot,
 * La = lookahead samples and `release_step` quanta of recovery per sample:
 *     p[k] = max over channels of |x[c][k]|;   q[k] = 0 if p <= ceiling, else ceil(Q log2(p / ceiling)) + 1,
 *            and 150 Q (a gain of exactly 0) when a channel's sample is not finite
 *     s[k] = max q[k - La .. k]          r[k] = max(s[k], r[k - 1] - release_step)          a[k] = sum r[k - La .. k]
 *     y[c][k] = 2^(-a[k] / (Q (La + 1))) x[c][k - La]        (0 where x[c][k - La] is not finite)
 * The fp32 gain is exp2f of the fraction times an exact power of two, the same for every channel.
 * So every written sample has |y| <= ceiling exactly, whatever the input; while no reduction is pending (a = 0) the gain
 * is exactly 1 and y is x delayed by La samples, bit for bit; and, the recurrence being exact integer arithmetic, cutting
 * a stream into other pushes changes no bit of the output or the state.  A non-finite sample mutes the output around it,
 * and the gain then recovers at the release rate from 150 octaves (about 900 dB): zeroing the slot's rows ends it at once.
 *
 * The state is [n_slots][channels][row_floats] fp32 of DEVICE memory.  Per channel: four head words, the channel's last La
 * input samples, then the last La q and the last La r (int32 words stored in the floats' bits).  The head words and the q
 * and r histories are channel 0's only: r of the last sample (int32), the slot's ceiling (float; 0: the call's), the
 * samples written with a > 0 since the slot was fresh (int32, saturating at 2^31 - 1) and the gain reduction in dB at the
 * last sample written (float).  A ceiling written into word 1 (a positive normal float; anything else means the call's)
 * applies to samples pushed after it.  All zeros is a fresh
 * slot, whose delay line starts with La zeros, so a slot is reset by zeroing its rows and moved by copying them.
 * l2h_limiter_layout: row_floats = 4 + 3 La.  Errors: 1 = null pointer, channels <= 0, lookahead < 0; 2 = the staging of
 * a one-sample push ((channels + 2) (La + 1) words) exceeds the kernel's shared memory.
 *
 * l2h_limiter: row i pushes m_i = counts_dev[i] * unit samples of x row i into slot slots_dev[i]:
 *   x_dev       [n][channels][max_in] fp32, strides in floats; row i reads only its first m_i samples
 *   y_dev       [n][channels][max_in] fp32; row i receives y[i][c][0 .. m_i), its slot's next m_i output samples.  Its later
 *               samples are not written.  Must not overlap x or the state.
 *   counts_dev  [n] int32 of DEVICE memory read when the kernel runs; m_i outside [0, max_in] counts as 0.  unit = 1 takes
 *               l2h_resample_packets' out counts, unit = 128 the separator's hop counts (l2h_hop_fifo's hops_dev).
 *   slots_dev   [n] int32 of DEVICE memory read when the kernel runs: an entry outside [0, n_slots) marks a row that stores
 *               nothing (no y sample, no state row).  So does a push of 0 samples.  A slot listed twice is a caller error
 *               the call does not detect.
 * One launch, one CTA per row over all its channels; nothing on the host is read from the device, and a call captured in
 * a CUDA graph serves any lists of the same n rewritten in place.  Errors, returned before anything is enqueued:
 * 1 = null pointers, n, channels, max_in, unit or n_slots <= 0, n > n_slots, a ceiling that is not a positive normal float,
 * release_step outside [1, 150 Q], lookahead < 0, channel or row strides under max_in, y overlapping x; 2 = the staging of
 * a row ((channels + 2) (La + max_in) words) exceeds the kernel's shared memory.  Asynchronous on `stream`. */
int l2h_limiter_layout(int32_t channels, int32_t lookahead, int32_t* row_floats);
int l2h_limiter(const float* x_dev, int64_t x_row_stride, int64_t x_ch_stride, int32_t max_in, const int32_t* counts_dev,
                int32_t unit, float* y_dev, int64_t y_row_stride, int64_t y_ch_stride, int32_t n, int32_t channels,
                const int32_t* slots_dev, float* state_dev, int32_t n_slots, float ceiling, int32_t lookahead,
                int32_t release_step, void* stream);

/* A per-row loudness leveler: brings each voice a listener hears to one loudness, with one gain for all channels, so
 * interaural level ratios are preserved.  A row is a separator record (the target rows of l2h_sep_forward_targets_rows,
 * before the mixer) or a listener slot (the mixer's sum).  It works on the separator's 16 kHz grid of 128-sample hops,
 * with no look-ahead and no added delay.  Per hop of a row, over its channels:
 *     each channel passes the two BS.1770 pre-filters ("K-weighting") for 16 kHz, derived from the analog prototypes as
 *       libebur128 derives them: a high shelf (f0 = 1681.974450955533 Hz, G = 3.999843853973347 dB, Q = 0.7071752369554196,
 *       Vb = Vh^0.4996667741545416), then a high-pass (f0 = 38.13547087602444 Hz, Q = 0.5003270373238773), K = tan(pi f0 / fs);
 *     P = the mean square of the weighted samples over the hop, summed over the channels; its loudness -0.691 + 10 log10 P
 *       LUFS;
 *     gate: a hop updates the estimate only when its loudness is at least `gate` and, once the row has an estimate, at
 *       least the estimate's loudness + `relative` (so pauses and a silent target's residual never pull the gain up);
 *     estimate: E <- E + w (P - E), w = max(alpha, 1 / (n + 1)) with n the gated hops before: the plain mean of the first
 *       hops, then an exponential average;
 *     gain (dB, one per row): 0 until the row has settle_hops gated hops; in the hop that reaches them,
 *       d = clamp(target - L(E), min_gain, max_gain); after that it moves toward d by at most rise_step dB up and
 *       fall_step dB down per hop (a hop that fails the gate still moves it toward the d of the held estimate);
 *     apply: sample k = 1 .. 128 of the hop is multiplied, in every channel, by 10^(g_k / 20) with
 *       g_k = g_prev + (g_new - g_prev) k / 128; a g_k of 0 dB is exactly 1.0f.
 * With min_gain = max_gain = 0 every written sample is its input bit for bit.  A hop with a sample that is not finite,
 * or whose magnitude is 2^32 or more, is not measured: its filters, estimate, count and gain keep their values (its samples
 * are written as x times the held gain, and a limiter downstream mutes a non-finite one), so the state stays finite.  A
 * hop's result depends only on the state at its start and its samples, so cutting hops into other calls changes no bit.
 *
 * The state is [n_rows][channels][row_floats] fp32 of DEVICE memory.  Per channel: three head words, then the channel's
 * shelf and high-pass states (two each).  The head words are channel 0's only: the estimate E (mean-square power), the
 * gated hops n (an int32 word stored in the float's bits, saturating at 2^31 - 1) and the gain in dB at the last sample
 * written.  All zeros is a fresh row, so a row is reset by zeroing it and moved by copying it.
 * l2h_leveler_layout: row_floats = 7.  Errors: 1 = null pointer, channels <= 0.
 *
 * l2h_leveler: call row r (one CTA each, over all its channels) levels y[r][c][0 .. 128 h) into out[r][c][0 .. 128 h):
 *   y_dev        [R][channels][128 * frames] fp32, strides in floats
 *   out_dev      the same shape; its rows' later samples, and the rows that store nothing, are not written.  out may be
 *                y itself (the same pointer and strides), which levels in place; any other overlap is refused.
 *   records_dev  [R] int32 of DEVICE memory: row r keeps its state in row records[r]; a record outside [0, n_rows) marks
 *                a row that stores nothing and advances nothing.  A record listed twice is a caller error the call does
 *                not detect.
 *   offsets_dev  [n + 1] int32 of DEVICE memory: listener i owns rows offsets[i] .. offsets[i+1]-1, the offsets clamped as
 *                l2h_sep_forward_targets_rows and l2h_target_mix clamp them; rows from offsets[n] on belong to nobody and
 *                store nothing.  NULL: listener i owns row i alone (rows from n on store nothing), the placement on the
 *                mixer's sum with records = slots.
 *   hops_dev     [n] int32 of DEVICE memory, or NULL (frames hops): listener i's rows level h = hops[i] hops; h outside
 *                [1, frames] stores nothing.
 *   alpha        1 - exp(-128 / (window * 16000)) for an averaging window in seconds; rise_step and fall_step in dB per
 *                hop (dB/s * 128 / 16000); settle_hops in hops.
 * All lists are read when the kernel runs, so a call captured in a CUDA graph with the FIFO, the rows call and the mixer
 * serves any lists of the same n and R rewritten in place.  One launch; nothing is read back to the host.  Errors,
 * returned before anything is enqueued: 1 = null pointers (offsets_dev and hops_dev may be NULL), n, R, channels, frames
 * or n_rows <= 0, n > R, n > n_rows, 128 frames above 2^31 - 1, a target, gate, relative, min_gain or max_gain that is
 * not finite, relative > 0, alpha outside (0, 1], min_gain > max_gain or a gain outside [-40, 40] dB, rise_step or
 * fall_step negative or not finite, settle_hops < 1, channel or row strides under 128 frames, out overlapping y other than
 * as y itself.  Asynchronous on `stream`. */
int l2h_leveler_layout(int32_t channels, int32_t* row_floats);
int l2h_leveler(const float* y_dev, int64_t y_row_stride, int64_t y_ch_stride, float* out_dev, int64_t out_row_stride,
                int64_t out_ch_stride, int32_t n, int32_t R, int32_t channels, int32_t frames, const int32_t* records_dev,
                const int32_t* offsets_dev, const int32_t* hops_dev, float* state_dev, int32_t n_rows, float target,
                float gate, float relative, float alpha, int32_t settle_hops, float min_gain, float max_gain,
                float rise_step, float fall_step, void* stream);

/* A per-slot multiband compressor: fits each listener's output to their hearing with a gain per band and per ear, and
 * compression per band that is the same for every channel, so the dynamics keep the interaural level differences.  It
 * works on the separator's 16 kHz grid of 128-sample hops, on the mixer's sum (one row per slot).
 *
 * The bank (l2h_band_compressor_design) has K bands, 1 <= K <= 16, cut at K - 1 edges that rise strictly inside
 * (0, 8000) Hz; each band is a linear-phase FIR of L taps, L odd in [33, 255], with a delay of D = (L - 1) / 2 samples.
 * With LP_j = scipy.signal.firwin(L, edge_j, fs=16000) (a Hamming-windowed sinc scaled to a DC gain of 1), band 0 is
 * LP_1, band j is LP_{j+1} - LP_j and band K - 1 is delta[n - D] - LP_{K-1}, all computed in float64, so the bands sum to
 * delta[n - D].  Per hop of a slot, over its channels:
 *     stage: the hop's 128 samples of each channel follow the slot's last L - 1 staged samples; a sample that is not
 *       finite, or whose magnitude is 2^32 or more, enters as 0, and the hop is then not measured;
 *     filter: band[c][b][k] = sum_j h_b[j] x_c[k - j];
 *     measure: P_b = the mean square of band b over the hop's samples, averaged over the channels; the detector
 *       S_b <- S_b + a (P_b - S_b), a = attack if P_b > S_b, else release; L_b = 10 log10 S_b dBFS (a full-scale sine
 *       reads -3.01);
 *     gain: R_b = slope_b max(0, L_b - knee_b) dB, shared by the channels; channel c's band b ends the hop at
 *       g_cb = clamp(gain_cb - R_b, -40, 40) dB;
 *     apply: sample k = 1 .. 128 is sum_b 10^(g_k / 20) band[c][b][k], summed in band order, with g_k = g_prev + (g_cb -
 *       g_prev) k / 128 from the gain at the previous hop's end; a g_k of 0 dB is exactly 1.0f;
 *     bypass: when every g of the slot is exactly 0 dB at the hop's start and end, the output is the staged input delayed
 *       by D samples, bit for bit.
 * A hop's result depends only on the state at its start and its samples, so cutting hops into other calls changes no bit.
 *
 * The state is [n_slots][channels][row_floats] fp32 of DEVICE memory.  Per channel: the channel's K profile gains (dB),
 * its K current gains (dB, at the last sample written), then K words of channel 0's only: S_b (mean square), then K more:
 * knee_b (dBFS), then K more: slope_b = 1 - 1 / ratio_b, then the channel's last L - 1 staged samples.  All zeros is a
 * fresh slot with a flat 0 dB profile and no compression, so a slot is reset by zeroing its rows and moved by copying
 * them; a profile is set by writing its words, and takes effect from the next hop, across one hop's dB ramp.
 *
 * l2h_band_compressor_design: writes the bank, out [bands][taps] fp32 of HOST memory, from edges_hz [bands - 1] (HOST
 * memory; may be NULL when bands = 1).  Uploads nothing.  Errors: 1 = null pointer, bands outside [1, 16], taps not odd
 * in [33, 255], edges that do not rise strictly inside (0, 8000).
 * l2h_band_compressor_layout: row_floats = 5 bands + taps - 1.  Errors: 1 = null pointer, channels <= 0, bands outside
 * [1, 16], taps not odd in [33, 255]; 2 = the staging of a row (taps 4 ceil(bands / 4) + channels (taps + 127) +
 * channels bands 130 words) exceeds the kernel's shared memory.
 *
 * l2h_band_compressor: call row i (one CTA each, over all its channels) compresses y[i][c][0 .. 128 h) into
 * out[i][c][0 .. 128 h) with the state of slot slots[i]:
 *   y_dev        [n][channels][128 * frames] fp32, strides in floats
 *   out_dev      the same shape; its rows' later samples, and the rows that store nothing, are not written.  out may be y
 *                itself (the same pointer and strides): each hop is staged before anything of it is written.  Any other
 *                overlap is refused.
 *   slots_dev    [n] int32 of DEVICE memory: an entry outside [0, n_slots) marks a row that stores nothing and advances
 *                nothing.  A slot listed twice is a caller error the call does not detect.
 *   hops_dev     [n] int32 of DEVICE memory, or NULL (frames hops): row i compresses h = hops[i] hops; h outside
 *                [1, frames] stores nothing.
 *   taps_dev     [bands][taps] fp32 of DEVICE memory: the bank, read when the kernel runs.
 *   attack, release  the detector's coefficients per hop, 1 - exp(-0.008 / tau) for a time constant tau in seconds.
 * All lists are read when the kernel runs, so a call captured in a CUDA graph with the FIFO, the rows call and the mixer
 * serves any lists of the same n rewritten in place.  One launch; nothing is read back to the host.  Errors, returned
 * before anything is enqueued: 1 = null pointers (hops_dev may be NULL), n, channels, frames or n_slots <= 0,
 * n > n_slots, 128 frames above 2^31 - 1, attack or release outside (0, 1], bands outside [1, 16], taps not odd in
 * [33, 255], channel or row strides under 128 frames, out overlapping y other than as y itself; 2 = the staging of a
 * row exceeds the kernel's shared memory (as in the layout).  Asynchronous on `stream`. */
int l2h_band_compressor_design(int32_t bands, const float* edges_hz, int32_t taps, float* out);
int l2h_band_compressor_layout(int32_t channels, int32_t bands, int32_t taps, int32_t* row_floats);
int l2h_band_compressor(const float* y_dev, int64_t y_row_stride, int64_t y_ch_stride, float* out_dev,
                        int64_t out_row_stride, int64_t out_ch_stride, int32_t n, int32_t channels, int32_t frames,
                        const int32_t* slots_dev, const int32_t* hops_dev, const float* taps_dev, int32_t bands,
                        int32_t taps, float* state_dev, int32_t n_slots, float attack, float release, void* stream);

/* The band compressor on a Linkwitz-Riley crossover bank: the same per-slot compressor as l2h_band_compressor, with a bank
 * of IIR crossovers in place of the linear-phase FIRs, so the delay it adds is short and falls with frequency (with the
 * default edges 500, 1000, 2000 and 4000 Hz at order 4: 1.83 ms at 250 Hz, 1.09 ms at 1 kHz, 0.41 ms at 2.8 kHz, 0.19 ms at
 * 6 kHz, against the FIR bank's 4 ms at every frequency), for weaker band separation and a non-linear phase.
 *
 * The bank (l2h_band_compressor_lr_design) has K bands, 1 <= K <= 16, cut at K - 1 edges that rise strictly inside
 * (0, 8000) Hz, with crossovers of order N = 4 or 8.  At edge e, LP_e = (Butterworth low-pass of order N / 2)^2, HP_e =
 * (Butterworth high-pass of order N / 2)^2 and AP_e is the allpass on the same poles, each by the bilinear transform
 * prewarped at the edge, as scipy.signal.butter(N / 2, edge, fs=16000) designs it, so LP_e + HP_e = AP_e.  Band b (from 0)
 * is HP_1 .. HP_b, then LP_{b+1} for every band but the last, then AP_{b+2} .. AP_{K-1} (edges counted from 1), so the
 * bands sum to the allpass cascade AP_1 .. AP_{K-1}: magnitude 1 at every frequency, no pure delay.  Every coefficient is
 * derived in float64 and rounded to fp32 at the end.  Each band is a cascade of S = N / 2 (K - 1) second-order sections
 * (b0, b1, b2, a1, a2; y = b0 x + s1, s1 <- b1 x - a1 y + s2, s2 <- b2 x - a2 y, transposed direct form II with fp32
 * states), the shorter cascades ending in identity sections (1, 0, 0, 0, 0).  K = 1 has no sections: its band is the input.
 * Per hop of a slot, over its channels, as l2h_band_compressor:
 *     stage: a sample that is not finite, or whose magnitude is 2^32 or more, enters as 0, and the hop is then not measured;
 *     filter: band[c][b] = channel c's staged samples through band b's sections, sample by sample;
 *     measure, gain: as l2h_band_compressor, P_b, S_b, R_b and g_cb;
 *     apply: sample k = 1 .. 128 is sum_b 10^(g_k / 20) band[c][b][k], summed in band order from -0, with g_k ramped as
 *       there; a g_k of 0 dB is exactly 1.0f.  There is no bypass: at 0 dB everywhere the output is the bands' sum, the
 *       allpass cascade of the input, not the input; with K = 1 it is the input bit for bit.
 * A hop's result depends only on the state at its start and its samples, so cutting hops into other calls changes no bit.
 *
 * The state is [n_slots][channels][row_floats] fp32 of DEVICE memory.  Per channel the first 5 K words are those of
 * l2h_band_compressor (profile gains, current gains, then channel 0's S_b, knee_b and slope_b), then the two states of
 * each section of each band, [K][S][2].  All zeros is a fresh slot with a flat 0 dB profile and no compression; a slot is
 * reset by zeroing its rows, moved by copying them, and fitted by writing the same words as for l2h_band_compressor.
 *
 * l2h_band_compressor_lr_design: writes the bank, out [bands][S][5] fp32 of HOST memory, S = order / 2 (bands - 1), from
 * edges_hz [bands - 1] (HOST memory; may be NULL when bands = 1).  Uploads nothing.  Errors: 1 = null pointer, bands
 * outside [1, 16], order not 4 or 8, edges that do not rise strictly inside (0, 8000).
 * l2h_band_compressor_lr_layout: row_floats = 5 bands + 2 bands S.  Errors: 1 = null pointer, channels <= 0, bands outside
 * [1, 16], order not 4 or 8; 2 = the staging of a row (5 bands S + channels 128 + channels bands 130 words) exceeds the
 * kernel's shared memory.
 *
 * l2h_band_compressor_lr: the arguments of l2h_band_compressor, with sos_dev [bands][S][5] fp32 of DEVICE memory (the
 * bank, read when the kernel runs) and order in place of taps_dev and taps.  The same list rules: a slot outside
 * [0, n_slots), or a hop count outside [1, frames], stores nothing and advances nothing; out may be y itself.  All lists
 * are read when the kernel runs, so a call captured in a CUDA graph serves any lists of the same n rewritten in place.
 * One launch; nothing is read back to the host.  Errors, returned before anything is enqueued: those of
 * l2h_band_compressor, with order not 4 or 8 in place of the taps; 2 = the staging of a row exceeds the kernel's shared
 * memory (as in the layout).  Asynchronous on `stream`. */
int l2h_band_compressor_lr_design(int32_t bands, const float* edges_hz, int32_t order, float* out);
int l2h_band_compressor_lr_layout(int32_t channels, int32_t bands, int32_t order, int32_t* row_floats);
int l2h_band_compressor_lr(const float* y_dev, int64_t y_row_stride, int64_t y_ch_stride, float* out_dev,
                           int64_t out_row_stride, int64_t out_ch_stride, int32_t n, int32_t channels, int32_t frames,
                           const int32_t* slots_dev, const int32_t* hops_dev, const float* sos_dev, int32_t bands,
                           int32_t order, float* state_dev, int32_t n_slots, float attack, float release, void* stream);

/* A per-slot jitter buffer: the first stage of a tick for devices that send packets of P samples with RTP's 16-bit
 * sequence numbers over a lossy network (UDP over Wi-Fi or BLE).  It puts packets back in sequence order, drops late and
 * duplicate ones and conceals lost ones, so every later stage sees one continuous stream at the device's rate.  A tick:
 *     l2h_jitter_buffer(x, seqs, counts -> y, out_counts)                     device rate, in order, losses concealed
 *     l2h_resample_packets(y, counts = out_counts, unit = P -> y16, n16)      (a 16 kHz device skips this)
 *     l2h_hop_fifo(y16, counts = n16, unit = 1 -> chunk, hops)
 *     l2h_sep_forward_slots_hops(chunk, slots, hops)
 * all from device memory and capturable in one CUDA graph.
 *
 * Sequence numbers are compared in serial-number arithmetic (RFC 1982): with `next` the number of the next packet to
 * decide, a packet s lies d = (s - next) mod 2^16, taken in [-2^15, 2^15), ahead of it, so a stream that wraps from 65535 to
 * 0 passes unchanged.  A row's packets are processed one at a time, in row order:
 *   - the first packet of a fresh slot sets next := s;
 *   - d < 0: late, dropped and counted in `late`;
 *   - a packet already held: a duplicate, dropped and counted in `duplicate`;
 *   - 0 <= d < window: held;
 *   - d >= window: a restart (a device reboot, a long outage): the held packets are discarded and counted in `dropped`,
 *     next := s, the packet is held, the restart is counted in `restarts`, and the packet fades in as after a loss run.
 * Then, while next is held it is released and next advances; while next is missing and a packet at least next + depth + 1
 * is held, next is declared lost (counted in `lost`), released as concealment, and next advances.  So depth = 0
 * conceals a gap as soon as any later packet arrives, and each step up waits one more packet for a late arrival.
 * In-order traffic is released on arrival: with no loss, duplicate or reordering the output is the input bit for bit,
 * with no added delay.  The window counts from next: the decided packets a call does not write (at most max_out per row
 * per call) wait in a backlog of up to `window` more, which the slot's next call writes first (also with count 0).  So
 * every decision is a function of the arrival sequence alone, and cutting the same arrivals into other calls, or another
 * max_out, changes only where the output is cut, bit for bit.  A release that finds the backlog full discards its oldest
 * packet and counts it in `dropped`; a service that writes what it decides every tick never reaches that.
 *
 * Concealment (after ITU-T G.711 Appendix I: pitch-period repetition with fading), one decision per slot for all channels,
 * so the repeated period keeps its interaural time and level differences.  Lags tau_min = round(0.0025 rate) ..
 * tau_max = round(0.015 rate) (66-400 Hz), correlation window Wc = round(0.020 rate), round(v) = floor(v + 0.5):
 *   - at the first lost packet of a run, with s the fp32 channel sum (channels in order) of the last Wc + tau_max written
 *     samples (concealment included), tau is the first maximiser over the lags of
 *         sum_k s[N - Wc + k] s[N - Wc + k - tau] / sqrt(max(sum_k s[N - Wc + k - tau]^2, FLT_MIN)),  k = 0 .. Wc - 1
 *     over the lags whose numerator is positive (each lag's sums in fp32, k ascending, fmaf), tau_max when none is;
 *   - channel c plays e_c[k] = g(k) x_c[N - tau + (k mod tau)], the last period looped, with g = 1 for k < round(0.010
 *     rate), (B - k) / (B - A) in fp32 from A = round(0.010 rate) to B = round(0.060 rate), and exactly 0 from B on;
 *   - the first real packet after a run, or after a restart (which searches a period first when no run is going), starts
 *     with a raised-cosine crossfade over Lr = min(round(0.004 rate), P) samples from the continuing concealment e (with
 *     its gain) to the packet r: v = e + w (r - e), w = 0.5 - 0.5 cospif((i + 1) / (Lr + 1)), i < Lr (fmaf);
 *   - a sample that is not finite, or whose magnitude is 2^32 or more, enters as 0.
 *
 * The state is [n_slots][channels][row_floats] fp32 of DEVICE memory, row_floats = 16 + R + R P + H + tau_max with
 * R = 2 window and H = Wc + tau_max: per channel sixteen head words and R ring tags (channel 0's only), a ring of R
 * packets, the last H samples written and the period being repeated.  The head words are int32 words in the floats' bits:
 * 0 started, 1 next, 2 the ring position of the oldest packet not written, 3 the packets decided and not written,
 * 4 the concealed samples into the current run (capped at B), 5 the run's lag (0: no run), 6 lost, 7 late, 8 duplicate,
 * 9 dropped, 10 restarts (saturating at 2^31 - 1; a negative one counts as 0), 11 the packets held, 12 the lag of the
 * last run (`pitch`).  A tag is 0 (empty), s + 1 for a stored packet s (with bit 17 set for a released one that fades
 * in) or -1 (a released loss); a released entry plays its packet whatever its number (a restart may lie between it and
 * next, and its packets still play), and a released entry with any other tag is concealed.  All zeros is a fresh
 * slot, so a slot is reset by zeroing its rows and moved by copying them.
 *
 * l2h_jitter_buffer_layout: row_floats.  Errors: 1 = null pointer, channels <= 0, rate outside [8000, 384000], packet < 1,
 * window outside [1, 4096], depth outside [0, window - 1], max_out < 1, a slot row of more than 2^31 - 1 floats; 2 = the
 * staging of a row (channels (H + max_out P) + H + channels tau_max + R + 1 + max_out words) exceeds the kernel's shared
 * memory.
 *
 * l2h_jitter_buffer: row i pushes packets j < c_i = counts_dev[i] of x row i into slot slots_dev[i]:
 *   x_dev           [n][channels][max_in P] fp32, strides in floats; packet j of row i is x[i][c][j P .. (j + 1) P)
 *   seqs_dev        [n][max_in] int32 of DEVICE memory read when the kernel runs: packet j's sequence number; an entry
 *                   outside [0, 65535] marks a packet that is skipped
 *   counts_dev      [n] int32 of DEVICE memory read when the kernel runs: c_i in packets
 *   y_dev           [n][channels][max_out P] fp32; row i receives y[i][c][0 .. m_i P), its slot's next m_i packets.  Its
 *                   later samples are not written.  Must not overlap x or the state.
 *   out_counts_dev  [n] int32 of DEVICE memory: m_i, in packets
 *   slots_dev       [n] int32 of DEVICE memory read when the kernel runs: an entry outside [0, n_slots), or a count outside
 *                   [0, max_in], marks a row that stores nothing and gets out count 0.  A slot listed twice is a caller
 *                   error the call does not detect.
 * One launch, one CTA per row over all its channels; nothing on the host is read from the device, and a call captured in
 * a CUDA graph serves any lists of the same n rewritten in place.  Errors, returned before anything is enqueued:
 * 1 = null pointers, n, channels, max_in or n_slots <= 0, n > n_slots, the layout's errors 1, channel or row strides under
 * the lengths above, y overlapping x; 2 = the staging of a row (as in the layout, with max_in in place of 1) exceeds the
 * kernel's shared memory.  Asynchronous on `stream`. */
int l2h_jitter_buffer_layout(int32_t channels, int32_t rate, int32_t packet, int32_t depth, int32_t window, int32_t max_out,
                             int32_t* row_floats);
int l2h_jitter_buffer(const float* x_dev, int64_t x_row_stride, int64_t x_ch_stride, int32_t max_in, const int32_t* seqs_dev,
                      const int32_t* counts_dev, float* y_dev, int64_t y_row_stride, int64_t y_ch_stride,
                      int32_t* out_counts_dev, int32_t n, int32_t channels, const int32_t* slots_dev, float* state_dev,
                      int32_t n_slots, int32_t rate, int32_t packet, int32_t depth, int32_t window, int32_t max_out,
                      void* stream);

/* The jitter buffer released on time: l2h_jitter_buffer with wall-clock deadlines, so a gap in a device's uplink is
 * concealed as it happens instead of when the uplink recovers, and a long outage ends in a restart with no added
 * latency.  A missing packet is declared lost by the arrival rule above or by its deadline on the server's clock,
 * whichever comes first.
 *
 * Clock.  now = *now_dev, read when the kernel runs, is the server's clock at the call in microseconds, an int32 that
 * wraps; clocks are compared in serial arithmetic (mod 2^32, only differences under 2^31 us matter).  Every packet pushed
 * in a call is taken to have arrived at that call's now.
 * Anchor.  A slot keeps the highest-numbered packet ever placed in its window, the anchor (a_s, a_t): its sequence
 * number and the now of the call it arrived in.  The first packet of a fresh slot sets it, and so does a restart; late and duplicate
 * packets never move it.
 * Deadline.  Packet s is expected at a_t + (s - a_s) period, with period = round(1e6 P / rate) us and s - a_s taken in
 * [-2^15, 2^15) (products mod 2^32).  Packet next expires once now - expected(next) >= deadline_us.
 * A row's work: first its arrivals run exactly as in l2h_jitter_buffer (except for a stalled slot, below).  Then the
 * release rule runs once more at now, with a third way to release next: next has expired and the slot has not stalled.
 * That release is a loss, counted in `lost` and in `expired`, and concealed as any loss is; held packets that follow it
 * are released too.  So a deadline <= e period declares a gap lost as soon as a packet e past it arrives, as depth does.
 * Stall.  Deadline releases stop once the concealment has gone silent: once next - a_s - 1 >= S, S = ceil(B / P)
 * packets (60 ms; 6 at 44.1 kHz / 441 and at 16 kHz / 160).  From then on the slot releases nothing, and its next arrival
 * with s - next >= 0 restarts the slot at s through the restart rule (counted in `restarts`, faded in), so no silent
 * backlog is released and a long outage adds no latency.  A packet behind next is still late.
 * With a deadline that no call reaches the output, the out counts and head words 0-12 equal l2h_jitter_buffer's, bit for
 * bit.  Over one sequence of (arrivals, now) calls another max_out changes only where the output is cut; splitting one
 * call's arrivals into two calls at the same now can change decisions (the deadline rule runs after each call).
 * A slot's deadlines are checked only in calls that list it: a service that runs deadlines lists every live slot in
 * every tick, with count 0 when the slot sent nothing.
 *
 * State: the layout of l2h_jitter_buffer_layout, with channel 0's head words 13 a_s, 14 a_t and 15 expired (saturating
 * at 2^31 - 1), which l2h_jitter_buffer leaves as they are.  One slot's state is meant for one of the two entries.
 *
 * l2h_jitter_buffer_timed: the arguments of l2h_jitter_buffer, plus
 *   now_dev         [1] int32 of DEVICE memory read when the kernel runs: the clock, so a call captured in a CUDA graph
 *                   serves any clock rewritten in place
 *   deadline_us     >= 0, in microseconds
 * Errors: those of l2h_jitter_buffer, and 1 = now_dev null, deadline_us < 0.  Asynchronous on `stream`. */
int l2h_jitter_buffer_timed(const float* x_dev, int64_t x_row_stride, int64_t x_ch_stride, int32_t max_in,
                            const int32_t* seqs_dev, const int32_t* counts_dev, float* y_dev, int64_t y_row_stride,
                            int64_t y_ch_stride, int32_t* out_counts_dev, int32_t n, int32_t channels,
                            const int32_t* slots_dev, float* state_dev, int32_t n_slots, int32_t rate, int32_t packet,
                            int32_t depth, int32_t window, int32_t max_out, const int32_t* now_dev, int32_t deadline_us,
                            void* stream);

/* The jitter buffer with adaptive deadlines: l2h_jitter_buffer_timed whose deadline each slot draws from the measured
 * lateness of its own packets, between lo_us and hi_us, so a listener on a clean link waits little for a loss and one
 * on a jittery link loses few packets to `late`.
 *
 * Arrivals.  arrivals_dev [n][max_in] int32 (may be null) holds each packet's arrival time on the server's clock in
 * us, with the clock's wrap and serial arithmetic.  Without it every arrival is the call's now; an arrival after now
 * (serial) is taken as now.  The anchor (a_s, a_t) is kept as in l2h_jitter_buffer_timed, except that a_t is the
 * arrival time of the packet that set it, not the now of its call.
 * Lateness.  With the anchor in force before packet s is placed, its lateness is
 *     l = arrival - (a_t + (s - a_s) period)   us, s - a_s in [-2^15, 2^15), in serial int32,
 * the quantity the release rule compares with the deadline.  It is measured for every packet placed in the window and
 * for every late packet (d < 0; late packets are the evidence that the deadline is too short), except that nothing is
 * measured for a slot's first packet, a duplicate, a packet that restarts the slot, or a packet that arrives while the
 * slot is stalled (an outage is not jitter).
 * Statistics, in exact integer arithmetic, so that the same timestamped arrivals cut into other calls give the same
 * statistics.  A slot keeps 64 int32 bins h_0 .. h_63 of width w = max(1, ceil(hi_us / 64)) us (a bin read outside
 * [0, 2^30] is clamped to it) and k, the packets measured (saturating at 2^31 - 1).  Lateness l falls in bin
 * b = clamp(floor(l / w), 0, 63): early packets land in bin 0, lateness of hi_us or more in bin 63.  With the memory
 * N = max(1, round(5e6 / period)) packets (about 5 s) each measured packet, in arrival order, with m = min(k + 1, N):
 *     h_i -= floor(h_i / m) for every i;  h_b += floor(2^24 / m);  k += 1
 * so the first packets are weighted as a plain mean and later ones forget exponentially; the bins sum to about 2^24.
 * Deadline.  Once per call, after its arrivals and before the release at now, each listed slot that has started
 * recomputes its deadline: with the tail T_b = sum_{i > b} h_i, the total T = sum_i h_i (int64) and
 * r = round(late_rate 2^16), b is the smallest bin with T_b 2^16 <= r T, and the deadline is clamp((b + 1) w, lo_us,
 * hi_us).  While k < ceil(1 / late_rate) it is hi_us: a (1 - late_rate) quantile needs that many samples.
 * The release at now is then l2h_jitter_buffer_timed's rule with the slot's deadline; the stall S, restarts,
 * concealment, backlog and max_out are unchanged.  With lo_us == hi_us == D and no arrivals_dev (or every arrival the
 * now of its call) the output, the out counts and head words 0-15 equal l2h_jitter_buffer_timed's at deadline D, bit
 * for bit.  A slot's deadlines are checked only in calls that list it: a service lists every live slot in every tick.
 *
 * State: [n_slots][channels][row_floats] with row_floats from l2h_jitter_buffer_adaptive_layout, 66 words more than
 * l2h_jitter_buffer_layout's.  The first row_floats - 66 words of each channel's row are laid out as in
 * l2h_jitter_buffer_timed; channel 0's last 66 words are the statistics block: 64 bins, k, and the deadline of the last
 * call (0 until the slot has started; the other channels leave these words unused).  All zeros is a fresh slot, so a
 * slot is reset by zeroing its rows and moved by copying them.
 *
 * l2h_jitter_buffer_adaptive_layout: the arguments and errors of l2h_jitter_buffer_layout.
 *
 * l2h_jitter_buffer_adaptive: the arguments of l2h_jitter_buffer_timed with deadline_us replaced by
 *   arrivals_dev    [n][max_in] int32 of DEVICE memory read when the kernel runs, or null: packet j's arrival time, so a
 *                   call captured in a CUDA graph serves any arrival times rewritten in place
 *   lo_us, hi_us    0 <= lo_us <= hi_us, the bounds of every slot's deadline, in microseconds
 *   late_rate       in (0, 0.5]: the fraction of measured packets the deadline may leave late
 * Errors: those of l2h_jitter_buffer (the staging of a row also holds max_in more words), and 1 = now_dev null,
 * lo_us < 0, hi_us < lo_us, late_rate outside (0, 0.5].  Asynchronous on `stream`. */
int l2h_jitter_buffer_adaptive_layout(int32_t channels, int32_t rate, int32_t packet, int32_t depth, int32_t window,
                                      int32_t max_out, int32_t* row_floats);
int l2h_jitter_buffer_adaptive(const float* x_dev, int64_t x_row_stride, int64_t x_ch_stride, int32_t max_in,
                               const int32_t* seqs_dev, const int32_t* counts_dev, float* y_dev, int64_t y_row_stride,
                               int64_t y_ch_stride, int32_t* out_counts_dev, int32_t n, int32_t channels,
                               const int32_t* slots_dev, float* state_dev, int32_t n_slots, int32_t rate, int32_t packet,
                               int32_t depth, int32_t window, int32_t max_out, const int32_t* now_dev,
                               const int32_t* arrivals_dev, int32_t lo_us, int32_t hi_us, double late_rate, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* LOOKONCE_B200_H */
