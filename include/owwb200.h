/*
 * owwb200.h - C ABI of libowwb200.so: the H100 (sm_90a) replacement for the three
 * inference sessions on openWakeWord's streaming hot path, plus the device-resident
 * stream state that sits between them.
 *
 * What each entry point replaces in the reference (paths in the original openWakeWord project):
 *   oww_melspectrogram   -> AudioFeatures.melspec_model_predict   openwakeword/utils.py:84-87,202
 *                           (melspectrogram.onnx; graph spec notebooks/converting_google_speech_embedding_model.ipynb:426-477)
 *   oww_embed_windows    -> AudioFeatures.embedding_model_predict openwakeword/utils.py:90-93,235,443
 *                           (embedding_model.onnx; graph spec same notebook :871-951)
 *   oww_head_predict     -> Model.model_prediction_function[name] openwakeword/model.py:137-138,158-159
 *                           (<head>.onnx; family openwakeword/train.py:56-83,144-165)
 *   oww_set_streams / oww_reset / oww_step / oww_step_host
 *                        -> AudioFeatures buffers + _streaming_features + the per-head window reads of
 *                           Model.predict                         openwakeword/utils.py:163-178,387-460; model.py:282-302
 *   oww_embed_clips      -> AudioFeatures.embed_clips             openwakeword/utils.py:358-385
 *   oww_predict_clips / oww_predict_clips_ragged
 *                        -> Model.predict_clip over many clips (bulk_predict's inner loop)
 *                                                                 openwakeword/model.py:388-426; utils.py:467-539
 *   oww_get_features / oww_get_mel
 *                        -> AudioFeatures.get_features / .melspectrogram_buffer   openwakeword/utils.py:454-460,165
 *
 * Conventions: every function returns 0 (OWW_OK) or a negative code; oww_last_error() gives the
 * message of the last failure on that handle (or, with NULL, of the last failed oww_create).
 * No exceptions cross the boundary.  Pointers named d_* are CUDA device addresses on the handle's
 * device (e.g. torch.Tensor.data_ptr()); h_* are host addresses.  `stream` is a cudaStream_t
 * passed as void* (NULL = the legacy default stream); all device work of a call is enqueued on it
 * and the call does not synchronise unless stated.  The caller owns every buffer it passes; the
 * library owns weights, rings and scratch inside the handle.  A handle is single-producer: one
 * host thread at a time.
 */
#ifndef OWWB200_H
#define OWWB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OWW_OK            0
#define OWW_EINVAL      (-1)   /* bad argument / wrong call order            */
#define OWW_ECUDA       (-2)   /* a CUDA runtime call failed                 */
#define OWW_ENOMEM      (-3)   /* host or device allocation failed           */
#define OWW_EUNSUPPORTED (-4)  /* graph shape outside what the kernels cover */

#define OWW_SAMPLES_PER_CHUNK 1280   /* 80 ms @ 16 kHz                         */
#define OWW_MEL_BINS            32
#define OWW_WINDOW_ROWS         76   /* mel rows per embedding window          */
#define OWW_EMBEDDING_DIM       96
#define OWW_INIT_FEATURE_ROWS   41   /* rows AudioFeatures seeds the ring with */
#define OWW_MAX_HEAD_LAYERS      8

/* embedding-CNN execution modes */
#define OWW_CNN_FP32_WINDOW       0  /* CUDA-core fp32, full 76-row window per frame (reference-shaped)  */
#define OWW_CNN_TC_WINDOW         2  /* wgmma fp16-operand/fp32-accumulate implicit GEMM, full window    */
#define OWW_CNN_TC_INCREMENTAL    3  /* wgmma, fused 20-layer kernel on the 8 new mel rows per stream
                                        (per-stream activation tails in HBM); first step after a reset and
                                        the stateless/batch calls use the full-window wgmma kernels        */

typedef struct oww_ctx oww_ctx;

/* Largest max_chunks oww_create accepts (a larger one fails with OWW_EINVAL before anything is allocated): the mel ring
 * of next_pow2(76 + 8 * max_chunks) rows stays within 2^20 rows, which the rebase of the row counts past 2^30 needs
 * (oww_get_counts). */
#define OWW_MAX_CHUNKS 131062

typedef struct oww_config {
    int32_t device;        /* CUDA device ordinal                                               */
    int32_t max_chunks;    /* largest n_chunks a single oww_step may carry (1..OWW_MAX_CHUNKS)  */
    int32_t cnn_mode;      /* OWW_CNN_*                                                         */
    int32_t window_batch;  /* windows per CNN sub-batch in the window modes (0 = default)       */
    int32_t reserved[4];   /* reserved[0] bit 0: 1 = keep mode 3's steady-state step as separate launches
                              (mel, CNN, append, heads) instead of the single fused step kernel;
                              bit 1: 1 = heads on CUDA cores (heads.cu) even in the tensor-core modes;
                              bit 2: 1 = tensor-core heads with plain fp16 operands (1 MMA term instead of the
                              fp32-grade 3-term hi/lo split);
                              bit 3: 1 = one tensor-core heads CTA per (128 streams, head) reading the fp32 rings
                              (heads_tc.cu) instead of one CTA per 128 streams for all heads that share a window,
                              fed from the fp16 mirror of the rings (heads_grp.cu);
                              bit 5: 1 = no programmatic dependent launches inside the late chain;
                              bit 4 and bits 6 and up are ignored.
                              reserved[1]: first conv layer that takes fp16 hi/lo split operands in the
                              tensor-core modes (0 = default 11; 20 = plain fp16 everywhere): 2..20 in
                              OWW_CNN_TC_WINDOW; OWW_CNN_TC_INCREMENTAL accepts only 3, 7, 11, 15 and 20 (the
                              split must start at a (1,3) layer behind a pool); with any other value
                              oww_set_streams fails with OWW_EUNSUPPORTED                                       */
} oww_config;

typedef struct oww_head_desc {
    int32_t n_in;                              /* embedding frames read per prediction (model_inputs)  */
    int32_t n_layers;                          /* Linear layers (>=1, <= OWW_MAX_HEAD_LAYERS)          */
    int32_t dims[OWW_MAX_HEAD_LAYERS + 1];     /* dims[0] = n_in*96, dims[n_layers] = n_out            */
    int32_t layernorm;                         /* 1: LayerNorm(eps 1e-5) after every hidden Linear     */
    int32_t final_act;                         /* 0 none, 1 sigmoid, 2 softmax, 3 relu then softmax,
                                                  4 relu (train.py's multi-class Net before the softmax wrapper) */
} oww_head_desc;

/* ---- lifetime ---------------------------------------------------------------------------- */
int  oww_create(const oww_config* cfg, oww_ctx** out);
void oww_destroy(oww_ctx* ctx);
const char* oww_last_error(const oww_ctx* ctx);
const char* oww_version(void);

/* ---- weights (host pointers; copied) ------------------------------------------------------ */
/* window512: the 512-tap analysis window (periodic Hann(400) centred); mel_fb: [257][32] filterbank.
 * Either may be NULL to use the built-in constants computed in double precision.                */
int oww_load_mel(oww_ctx* ctx, const float* h_window512, const float* h_mel_fb);
/* blob layout: openwakeword_b200/weights.py:pack_embedding_blob (20 x {HWIO kernel, scale, bias}). */
int oww_load_embedding(oww_ctx* ctx, const float* h_blob, size_t n_floats);
/* blob layout: weights.py:pack_head_blob.  *head_id receives the index; score columns are
 * appended in head order (head 0's n_out columns first).                                        */
int oww_add_head(oww_ctx* ctx, const oww_head_desc* desc, const float* h_blob, size_t n_floats, int* head_id);
/* Conditional verifier pair (the released hey_jarvis graph, docs/models/hey_jarvis.md:9,38: "the second network ...
 * only predicting on audio frames that have a score > 0.5 from the first"): wherever the score of single-output head
 * `main_head` exceeds `threshold` it is replaced by the score of single-output head `verifier_head`, per chunk, before
 * the max over a multi-chunk call.  Both columns stay in d_scores (the verifier's holds its raw score).          */
int oww_add_gate(oww_ctx* ctx, int main_head, int verifier_head, float threshold);

/* ---- custom verifier models (openwakeword/model.py:175-195,319-328; custom_verifier_model.py:91-113;
 *      docs/custom_verifier_models.md) ------------------------------------------------------------------------------
 * A verifier is the speaker-specific pipeline train_verifier_model pickles, FunctionTransformer(flatten_features) ->
 * StandardScaler -> binary LogisticRegression, restated on the D = n_in*96 newest feature rows x of its parent head:
 *     p = 1 / (1 + exp(-(bias + sum_j (x_j - mean_j) * weight_j)))   mean = scaler.mean_, weight = coef_ / scaler.scale_
 * (host-computed in float64, stored as fp32; fp32 accumulation in a fixed order).  After the heads, the verifier gates
 * and the max over the chunk windows of a step, every score column of the parent that is >= threshold (compared in
 * fp32) is replaced by p of the stream's verifier on the newest window; columns below it keep their value.
 *   oww_add_verifier_bank      - slots for up to `capacity` verifiers of head `head_id` (of a gated pair: the main head);
 *                                every stream starts without a verifier (slot -1).  8*D bytes per slot.
 *   oww_add_bank_verifier_bank - the same for the per-stream head bank `head_bank` (below): its score columns, its n_in.
 *                                A stream (or bulk row) whose head-bank slot is -1 has no model and is never verified: its
 *                                columns stay 0.0 whatever the threshold.  Every other call here takes either kind of bank.
 *   oww_load_verifier          - copy one verifier into a slot; h_mean and h_weight hold D floats each.  Synchronises
 *                                the device first, so steps already in flight use the old contents.
 *   oww_assign_verifier        - stream-ordered, allocation-free: stream h_stream_ids[i] (NULL = all streams, then n is
 *                                the stream count) uses slot h_slots[i] (-1 = none) from the next step enqueued on `stream`
 *                                or submitted with oww_step_host / oww_step_host_submit
 *   oww_set_verifier_clip_slot - the slot oww_predict_clips applies to every clip (-1 = none, the default; a bank of a
 *                                head bank verifies clips only while that bank's clip slot is not -1)
 *   oww_set_verifier_threshold - new threshold for the steps and clip calls enqueued from now on
 *   oww_enable_verifiers       - 0: steps and clip calls enqueued from now on skip every bank (their scores are the
 *                                heads' max over the chunk windows), 1 (default): they apply them.  For a caller that
 *                                splits one long call into several steps and verifies the max itself.
 *   oww_verifier_predict       - stateless and ungated: d_feats [n][n_in][96] -> d_out[n] = predict_proba(...)[:, -1]
 * At most one bank per head or head bank, 16 banks of heads and 16 of head banks per handle (OWW_EUNSUPPORTED past
 * that).  Every bank of both kinds runs in one launch per step, after everything else.  oww_set_streams resets every
 * assignment to -1; oww_reset / oww_reset_async leave them as they are (which user owns a stream is the caller's
 * business).  A handle without banks launches nothing for verifiers.                                                  */
int oww_add_verifier_bank(oww_ctx* ctx, int head_id, int capacity, float threshold, int* bank_id);
int oww_add_bank_verifier_bank(oww_ctx* ctx, int head_bank, int capacity, float threshold, int* bank_id);
int oww_load_verifier(oww_ctx* ctx, int bank, int slot, const float* h_mean, const float* h_weight, float bias);
int oww_assign_verifier(oww_ctx* ctx, int bank, const int32_t* h_stream_ids, int n, const int32_t* h_slots, void* stream);
int oww_set_verifier_clip_slot(oww_ctx* ctx, int bank, int slot);
int oww_set_verifier_threshold(oww_ctx* ctx, int bank, float threshold);
int oww_enable_verifiers(oww_ctx* ctx, int enabled);
int oww_verifier_predict(oww_ctx* ctx, int bank, int slot, const float* d_feats, int n, float* d_out, void* stream);
/* Training verifiers (custom_verifier_model.py:95-113, train_verifier_model), many users in one launch.
 *   oww_fit_verifiers  - user u's samples are i in [h_sample_offsets[u], h_sample_offsets[u+1]) (host int64, n_users+1
 *                        entries, non-decreasing, first >= 0); sample i is the window of n_in consecutive rows of
 *                        d_rows [n_rows][96] (fp32, 16-byte aligned) starting at row d_first_row[i] (device int64), with
 *                        label d_labels[i] (device uint8; nonzero = positive).  Windows may overlap; a plain [N][n_in][96]
 *                        array is the case first_row[i] = i*n_in.  Per user, in float64: StandardScaler's mean_ and
 *                        var_ (ddof 0; scale_ = sqrt(var_), 1 for the features scikit-learn treats as constant) ->
 *                        d_mean, d_var [n_users][D]; the unique minimiser of 1/2 |w|^2 + C sum_i log(1 + exp(-s_i (w.z_i
 *                        + b))), z = (x - mean_)/scale_, s_i = +-1, intercept unpenalised -> d_coef [n_users][D] (coef_,
 *                        standardized space), d_intercept [n_users]; Newton iterations -> d_iters; d_status:
 *                          0 converged: max |gradient| <= tol * C * n_u (scikit-learn's scaling of its tol)
 *                          1 max_iter Newton iterations reached, or no further descent: the outputs are the last iterate
 *                          2 n_u = 0 or one class only      3 a non-finite value, or a window not inside [0, n_rows)
 *                        (statuses 2 and 3 zero the user's outputs).  A user's outputs are the same bits whatever the
 *                        other users of the call.  Stream-ordered; allocation-free after the first call at a given size
 *                        (the scratch is the handle's: do not overlap two fits of one handle on different streams).
 *                        OWW_EINVAL before anything is enqueued for C <= 0 or non-finite, n_in outside [1, 120], max_iter
 *                        < 1, tol < 0 or non-finite, decreasing offsets, or a misaligned d_rows.
 *   oww_load_verifiers - slot h_slots[i] (distinct, host) of bank `bank` <- d_mean[i], d_weight[i] (device, [n][D] fp32;
 *                        weight = coef_ / scale_) and d_bias[i] (device fp32 [n]).  Stream-ordered on `stream` and ordered
 *                        against the handle's own stream, like oww_assign_verifier; no synchronisation.  Load slots no
 *                        stream is assigned to, then assign them: steps in flight never see a half-written slot.     */
int oww_fit_verifiers(oww_ctx* ctx, const float* d_rows, int64_t n_rows, int n_in, const int64_t* d_first_row,
                      const int64_t* h_sample_offsets, const uint8_t* d_labels, int n_users, double C, int max_iter,
                      double tol, double* d_mean, double* d_var, double* d_coef, double* d_intercept, int32_t* d_iters,
                      int32_t* d_status, void* stream);
int oww_load_verifiers(oww_ctx* ctx, int bank, const int32_t* h_slots, int n, const float* d_mean,
                       const float* d_weight, const float* d_bias, void* stream);

/* ---- per-stream head banks (a different wake-word model on every stream; each slot replaces one <head>.onnx session
 *      of Model.model_prediction_function, openwakeword/model.py:137-138,158-159, for the streams assigned to it) -------
 * A bank holds `capacity` slots, each a head of the one graph shape `desc` (the train.py family, openwakeword/train.py:
 * 56-83).  Its n_out = desc->dims[n_layers] score columns are appended when the bank is added, in call order with
 * oww_add_head (oww_n_outputs counts them; banks do not count against the 16 heads of a handle).  In every step, a stream
 * assigned slot k gets in those columns what head k would give as an ordinary head on that stream (per chunk window,
 * the max over the windows of a multi-chunk call; held streams of a ragged step are not written); a stream on slot -1
 * gets 0.0.  A slot runs the tensor-core heads kernel with the operand split, term count and accumulation order of
 * oww_head_predict, so it equals an ordinary head of the same weights bit for bit where that head runs that kernel
 * (oww_head_predict in cnn_modes 2/3, and streaming with reserved[0] bit 3).  Gates apply to ordinary heads only;
 * custom verifiers attach to a bank with oww_add_bank_verifier_bank.  reserved[0] bit 2 (plain fp16 operands) applies
 * to banks; bits 1 and 3 do not.
 *   oww_add_head_bank        - capacity slots of shape desc, allocated here: per slot the fp16 hi/lo packing of every
 *                              layer plus the fp32 biases and LayerNorm parameters (415 672 B at 16x96 -> 64 -> 64
 *                              -> 1, 863 672 B at 16x96 -> 128 -> 128 -> 1, descriptor included).  Every stream starts on slot -1.
 *                              OWW_EUNSUPPORTED in cnn_mode 0 and for any layer wider than 128.
 *   oww_load_bank_head       - copy a head (pack_head_blob layout of the bank's shape) into a slot.  Synchronises the
 *                              device first, so steps already in flight keep the old weights.
 *   oww_assign_bank_head     - stream-ordered, allocation-free: stream h_stream_ids[i] (NULL = all streams, then n is the
 *                              stream count) uses slot h_slots[i] (-1 = none; a slot must hold a head) from the next step
 *                              enqueued on `stream` or submitted with oww_step_host*.  The host sorts the streams by slot
 *                              and stages the work table through pinned memory (it waits for the copy of the previous
 *                              assignment of the bank).
 *   oww_set_head_bank_clip_slot - the slot oww_predict_clips / _ragged apply to every clip (-1, the default: zeros;
 *                              oww_predict_clips_streams uses each clip's stream instead)
 *   oww_bank_head_predict    - stateless: d_feats [n][n_in][96] -> d_out [n][n_out] with the head of `slot`
 * oww_set_streams resets every assignment to -1; oww_reset / oww_reset_async leave them as they are.  A bad bank,
 * slot or stream id fails with OWW_EINVAL.  A handle without banks launches nothing for them.                        */
int oww_add_head_bank(oww_ctx* ctx, const oww_head_desc* desc, int capacity, int* bank_id);
int oww_load_bank_head(oww_ctx* ctx, int bank, int slot, const float* h_blob, size_t n_floats);
int oww_assign_bank_head(oww_ctx* ctx, int bank, const int32_t* h_stream_ids, int n, const int32_t* h_slots, void* stream);
int oww_set_head_bank_clip_slot(oww_ctx* ctx, int bank, int slot);
int oww_bank_head_predict(oww_ctx* ctx, int bank, int slot, const float* d_feats, int n, float* d_out, void* stream);

int oww_n_heads(const oww_ctx* ctx);
int oww_n_outputs(const oww_ctx* ctx);          /* total score columns over all heads and head banks */

/* ---- stateless graph calls (drop-in for the three ORT sessions) --------------------------- */
/* d_pcm [n_clips][n_samples] int16 -> d_mel [n_clips][T][32], T = (n_samples-512)/160+1.
 * The -80 dB clamp is per clip (the reference's CPU path runs the graph one clip per call).
 * affine != 0 applies AudioFeatures' x/10+2 (utils.py:180,206).                                 */
int oww_melspectrogram(oww_ctx* ctx, const int16_t* d_pcm, int n_clips, int n_samples,
                       float* d_mel, int affine, void* stream);
/* d_windows [n][76][32] float32 -> d_emb [n][96] */
int oww_embed_windows(oww_ctx* ctx, const float* d_windows, int n, float* d_emb, void* stream);
/* d_feats [n][n_in][96] -> d_out [n][n_out] */
int oww_head_predict(oww_ctx* ctx, int head_id, const float* d_feats, int n, float* d_out, void* stream);

/* ---- streaming state ----------------------------------------------------------------------- */
int oww_set_streams(oww_ctx* ctx, int n_streams);    /* (re)allocates rings; implies reset of all */
int oww_n_streams(const oww_ctx* ctx);
/* Reset streams to AudioFeatures.__init__/reset() state: empty PCM history, mel ring = ones(76,32),
 * feature ring = h_feature_init[n_rows][96] (NULL -> zeros(41,96); the reference fills it with
 * embeddings of unseeded noise, SURVEY.md F6 - pass the same rows to both sides for parity).
 * h_stream_ids NULL = all streams.  Synchronises.                                              */
int oww_reset(oww_ctx* ctx, const int32_t* h_stream_ids, int n, const float* h_feature_init, int n_rows);
/* Same, stream-ordered: no allocation, no synchronisation.  Enqueue it on the stream the steps run on (the one passed
 * to oww_step).  Streams that were reset re-prime from a full 76-row window at their next step (their first chunk
 * yields 5 mel rows, utils.py:393-398) on a side stream while every other stream keeps the incremental fused kernel. */
int oww_reset_async(oww_ctx* ctx, const int32_t* h_stream_ids, int n, const float* h_feature_init, int n_rows, void* stream);
/* One predict() worth of work for every stream: n_chunks*1280 new samples per stream.
 * d_pcm row b starts at d_pcm + b*pcm_stride (samples); any stride >= n_chunks*1280 and any 2-byte aligned
 * d_pcm are accepted, a shorter stride fails with OWW_EINVAL before anything is enqueued (so does it in
 * oww_step_host and oww_step_host_submit).  d_scores [n_streams][oww_n_outputs]:
 * per head the element-wise max over the n_chunks window positions (model.py:287-298).          */
int oww_step(oww_ctx* ctx, const int16_t* d_pcm, int64_t pcm_stride, int n_chunks,
             float* d_scores, void* stream);
/* Same, host buffers: H2D of the PCM and D2H of the scores through pinned staging inside the handle;
 * returns after the scores have landed in h_scores (= submit + collect).                          */
int oww_step_host(oww_ctx* ctx, const int16_t* h_pcm, int64_t pcm_stride, int n_chunks, float* h_scores);
/* Pipelined form for serving loops: submit copies the PCM to pinned memory, enqueues H2D (copy stream),
 * the step (compute stream, in submission order) and the D2H of the scores, and returns a ticket (0/1)
 * without waiting; at most two tickets may be in flight, so the H2D of step k+1 overlaps the kernels
 * of step k.  collect blocks until that step's scores are in h_scores.                          */
int oww_step_host_submit(oww_ctx* ctx, const int16_t* h_pcm, int64_t pcm_stride, int n_chunks, int* ticket);
int oww_step_host_collect(oww_ctx* ctx, int ticket, float* h_scores);
/* Ragged step: streams advance at their own pace.  Stream b steps h_chunks[b] chunks (host memory, 0..max_chunks),
 * the first h_chunks[b]*1280 samples of row b; pcm_stride >= max(h_chunks)*1280.  Afterwards stream b is exactly a
 * stream that was given those samples by oww_step(h_chunks[b]): its row of d_scores is what that call returns for it
 * (per head the max over its own chunk windows, gates per chunk, custom verifiers after the max) and its -80 dB clamp
 * spans its own chunks.  A stream with h_chunks[b] == 0 is held: its state (PCM tail, mel and feature rings, conv
 * tails) does not change, bit for bit, a fresh stream stays fresh, and its row of d_scores is not written.
 * All counts equal to n >= 1: the call is oww_step(n).  All 0: nothing is enqueued.  A count outside 0..max_chunks
 * or a short stride fails with OWW_EINVAL before anything is enqueued.  Stream-ordered; no device allocation after
 * the first call.  The counts are staged through a ring of four pinned buffers of the handle: a call waits (host
 * side) for the count copy of the call four staging uses back - backpressure once the host runs that far ahead of
 * the device (a multi-chunk call whose one-chunk streams take the fused launch on their own uses two).  The host
 * side sorts the counts in small heap buffers.                                                                     */
int oww_step_ragged(oww_ctx* ctx, const int16_t* d_pcm, int64_t pcm_stride, const int32_t* h_chunks, float* d_scores,
                    void* stream);
/* Same, host buffers (submit + collect, or the pipelined submit completed by oww_step_host_collect).  The collect
 * leaves the rows of held streams in h_scores as the caller had them.                                               */
int oww_step_host_ragged(oww_ctx* ctx, const int16_t* h_pcm, int64_t pcm_stride, const int32_t* h_chunks, float* h_scores);
int oww_step_host_ragged_submit(oww_ctx* ctx, const int16_t* h_pcm, int64_t pcm_stride, const int32_t* h_chunks, int* ticket);
/* last n rows of one stream's feature ring, ending `back` rows before the newest -> h_out[n][96];
 * rows older than the ring holds come back as zeros.  Synchronises.                             */
int oww_get_features(oww_ctx* ctx, int stream_id, int n, int back, float* h_out);
int oww_get_mel(oww_ctx* ctx, int stream_id, int n_rows, float* h_out);   /* last n_rows<=76 mel rows */
/* rows written to the stream's mel / feature buffer since its last reset, initial rows included (76 ones / the
 * feature_init rows) - len(melspectrogram_buffer) / len(feature_buffer) of the reference before its 970 / 120 caps
 * (utils.py:400-401,449-450).  A count that reaches 2^30 is lowered by 2^30 - 2^20 (a multiple of every ring size) by
 * the step that reaches it, so past 2^30 rows it is that number minus a multiple of 2^30 - 2^20, never below 2^20;
 * it always exceeds 120 there.  Either pointer may be NULL.  Synchronises.                                     */
int oww_get_counts(oww_ctx* ctx, int stream_id, int* mel_rows, int* feature_rows);

/* ---- moving live streams: stream records ----------------------------------------------------------------------------
 * A stream record is one stream's complete state - PCM tail, counters, the newest 76 mel rows and 120 feature rows, and
 * in cnn_mode 3 the conv tails of the fused kernel and the late layers as stored - in a layout that depends only on the
 * cnn_mode, split_from and the loaded weights, not on the stream count, max_chunks, the heads or the other reserved
 * flags.  It starts with a header (format version, record size, configuration key); the size is a multiple of 16 bytes.
 *   oww_stream_state_info   - the record size of this handle and its configuration key (a hash of the format version,
 *                             cnn_mode, split_from in mode 3, the mel constants and the embedding blob).  Needs
 *                             oww_set_streams first.
 *   oww_export_streams      - stream h_stream_ids[i] -> record i of d_records [n][record_bytes] (device memory of the
 *                             handle's device).  Duplicate ids are allowed.
 *   oww_import_streams      - record i -> stream h_stream_ids[i] (no duplicates).  Afterwards that stream is exactly the
 *                             stream the record was taken from: its next steps of any kind give the same scores and leave
 *                             the same rings and counts, bit for bit wherever both handles run the same arithmetic.  The
 *                             fp16 feature mirror of the targets is resynced as after a reset.  No other stream changes,
 *                             and no stream's verifier or head-bank assignment changes (targets included).  A row
 *                             count at or past 2^30 in a record is rebased as a step rebases it (oww_get_counts).
 *   oww_stream_state_status - records the imports since the last call skipped (*n_rejected); synchronises; clears.
 * Export and import are stream-ordered and allocation-free after the first call, like oww_reset_async, and ordered
 * against oww_step_host / oww_step_host_submit on the handle's own stream: an export enqueued between two steps
 * captures exactly the state between them.  No oww_set_streams yet, an id out of range, n greater than the stream
 * count or a duplicate id in an import fails with OWW_EINVAL before anything is enqueued.  A record whose header does
 * not match this handle's size and key is skipped on the device: its stream is left unchanged and the rejection is
 * counted for oww_stream_state_status.                                                                                 */
int oww_stream_state_info(const oww_ctx* ctx, size_t* record_bytes, uint64_t* config_key);
int oww_export_streams(oww_ctx* ctx, const int32_t* h_stream_ids, int n, void* d_records, void* stream);
int oww_import_streams(oww_ctx* ctx, const int32_t* h_stream_ids, int n, const void* d_records, void* stream);
int oww_stream_state_status(oww_ctx* ctx, int* n_rejected);

/* ---- detections on the device (openwakeword/model.py:303-363: the prediction history, the zeroing of the first five
 *      predictions, patience, debounce_time, the repeat of the previous prediction below 1280 samples, the threshold) ---
 * A detector turns the score matrix of a step into detections, per stream, with the history on the device.  It has
 * n_labels labels (<= 256); label j reads score column `column` (-1: always 0.0, a class mapped past its head's outputs)
 * and has `repeats` (1: a label of a single-output head, which repeats its previous prediction when fewer than 1280
 * samples were prepared; 0: a class of a multi-output head, which reads 0.0 then), `threshold` (NaN = none) and `patience`
 * (0 = none, else 1..30); debounce_time (seconds, 0 = off) is one per handle (oww_set_stream_detection, below, gives
 * streams their own).  Per stream the handle keeps the last 30
 * final predictions of every label and one count of predictions appended since the stream's reset (11 labels: 1324 B).
 *   oww_set_detector  - configure, reconfigure or (n_labels 0) remove the detector.  Synchronises the device.  The same
 *                       columns and repeats as before keep the histories (the reference takes thresholds, patience and
 *                       debounce per predict call); another label set starts every stream with an empty history.  Before
 *                       oww_set_streams the state is allocated by that call.  OWW_EINVAL: a column outside
 *                       -1..oww_n_outputs-1, a patience outside 0..30, a patience without a threshold, a patience together
 *                       with a debounce_time, n_labels > 256.
 *   oww_detect        - one prediction for every stream from d_scores [n_streams][oww_n_outputs] (what oww_step* wrote).
 *                       Stream b prepared p = h_prepared[b] samples in this call (host int32 [n_streams]; NULL: p =
 *                       prepared_all for every stream) - what AudioFeatures.__call__ returns:
 *                         p < 0:      the stream is skipped: nothing is read, appended or reported (a stream held with 0
 *                                     chunks in oww_step_ragged), and its row of d_final is not written;
 *                         p >= 1280:  prediction = d_scores[b][column] (0.0 for column -1);
 *                         0 <= p < 1280: the newest history entry of a `repeats` label (0.0 when the history is empty),
 *                                     0.0 for any other label; the row of d_scores is not read.
 *                       Then, with count = predictions appended so far and the history = the last min(count, 30) of them:
 *                       (1) count < 5 -> 0; (2) patience: the prediction is nonzero and fewer than `patience` of the last
 *                       min(patience, count) entries are >= threshold -> 0; (3) else debounce: the label has a threshold,
 *                       the prediction is nonzero and >= threshold, and one of the last n entries is >= threshold -> 0,
 *                       n = ceil(debounce_time / (p / 16000)) in double (the whole history for p == 0), capped by the
 *                       entries present; (4) the prediction is appended, count += 1.  Comparisons are in fp32.
 *                       d_final [n_streams][n_labels] (may be NULL) receives the predictions.  d_n_events (may be NULL,
 *                       then so is d_events) receives the number of (stream, label) pairs whose label has a threshold and
 *                       whose prediction is >= it; d_events (may be NULL with max_events 0) receives the first
 *                       min(that number, max_events) of them in ascending (stream, label) order - the order never
 *                       depends on scheduling - with `index` = the stream's count before the append, in the count's
 *                       frame after this call's rebase (the count after the call minus 1: 63, not 2^30 - 1, on the call
 *                       that reaches 2^30).  Memory past those is not written.  Stream-ordered, no allocation, no synchronisation: one launch, two with
 *                       d_n_events.  h_prepared is staged through a ring of four pinned buffers: a call waits (host
 *                       side) for the copy of the call four staging uses back.  OWW_EINVAL before anything is enqueued:
 *                       no detector (or no streams), d_scores NULL, max_events < 0 or > 0 without d_events, d_events
 *                       without d_n_events, d_final and d_n_events both NULL.
 *   oww_detector_export / _import - the history of streams h_stream_ids[i] <-> d_hist [n][n_labels][30] (oldest first:
 *                       entry k was appended 30 - k predictions ago; zeros where the stream has fewer) and d_counts [n];
 *                       stream-ordered on `stream`.  Duplicate ids fail an import with OWW_EINVAL.  Stream records
 *                       (oww_export_streams) do not carry this history: move it with these two calls.
 * oww_reset / oww_reset_async clear the history of the streams they reset (one more launch), oww_set_streams that of
 * all.  The count is rebased by a multiple of 30 past 2^30, like the ring counters.  A handle without a detector
 * launches nothing for it.                                                                                             */
typedef struct oww_detect_label { int32_t column; int32_t repeats; float threshold; int32_t patience; } oww_detect_label;
typedef struct oww_event { int32_t stream; int32_t label; float score; int32_t index; } oww_event;
int oww_set_detector(oww_ctx* ctx, const oww_detect_label* h_labels, int n_labels, double debounce_time);
int oww_detect(oww_ctx* ctx, const float* d_scores, int prepared_all, const int32_t* h_prepared, float* d_final,
               oww_event* d_events, int max_events, int32_t* d_n_events, void* stream);
int oww_detector_export(oww_ctx* ctx, const int32_t* h_stream_ids, int n, float* d_hist, int32_t* d_counts, void* stream);
int oww_detector_import(oww_ctx* ctx, const int32_t* h_stream_ids, int n, const float* d_hist, const int32_t* d_counts,
                        void* stream);
/* ---- per-stream detection settings: every stream at its own sensitivity ----------------------------------------------
 * A stream may override, per label, the threshold and patience of oww_set_detector, and the debounce_time.  oww_detect
 * applies its rules, unchanged, with the stream's values; a stream without an override detects with the handle's values,
 * bit for bit as without this call.  One record per (stream, label), oww_stream_detect:
 *   threshold - NaN: the handle's threshold of the label; else this stream's;
 *   patience  - -1: the handle's patience of the label; else this stream's, 0..30;
 *   flags     - OWW_DETECT_NO_THRESHOLD: the label has no threshold on this stream (it never fires there and is not
 *               debounced; `threshold` is ignored).  Other bits must be 0.
 * and one debounce per stream (seconds; NaN: the handle's debounce_time).
 *   oww_set_stream_detection - streams h_stream_ids[i] (NULL: every stream, n = the stream count) take the records
 *                       h_overrides [n][n_labels] and the debounce h_debounce [n] (NULL: the handle's for all of them);
 *                       h_overrides NULL returns the streams to the handle's settings (h_debounce is then ignored).  A
 *                       record set equal to "the handle's values" (NaN, -1, 0 and NaN) is no override.  Each stream's
 *                       resulting values are checked as oww_set_detector checks the handle's: patience 0..30, a debounce
 *                       finite and >= 0, a patience needs a threshold and excludes a debounce.  Stream-ordered: oww_detect
 *                       calls enqueued on `stream` afterwards use the new settings.  The host keeps the whole table and
 *                       uploads it ([n_streams][n_labels] records and [n_streams] doubles, pageable: staged before the
 *                       call returns) while any stream has an override; no device allocation.
 *   oww_get_stream_detection - the settings of streams h_stream_ids[i] -> h_overrides [n][n_labels] and h_debounce [n]
 *                       (either may be NULL); a stream without an override reads NaN, -1, 0 and NaN.  Host only.
 * Both fail with OWW_EINVAL before anything changes for no detector (or no streams), an id out of range or a duplicate id,
 * n outside [0, n_streams], a record or debounce the checks refuse (a getter may repeat ids).  oww_set_detector clears every override (the checks
 * were made against the values it replaces); oww_set_streams keeps those of the streams below the new count and gives
 * the new streams none; oww_reset / oww_reset_async keep them.  oww_detector_export / _import move histories only:
 * move the settings with these two calls.  While no stream has an override oww_detect reads no record.                */
typedef struct oww_stream_detect { float threshold; int32_t patience; int32_t flags; } oww_stream_detect;
#define OWW_DETECT_NO_THRESHOLD 1
#ifdef __cplusplus
static_assert(sizeof(oww_stream_detect) == 12, "oww_stream_detect is 12 bytes");
#else
_Static_assert(sizeof(oww_stream_detect) == 12, "oww_stream_detect is 12 bytes");
#endif
int oww_set_stream_detection(oww_ctx* ctx, const int32_t* h_stream_ids, int n, const oww_stream_detect* h_overrides,
                             const double* h_debounce, void* stream);
int oww_get_stream_detection(oww_ctx* ctx, const int32_t* h_stream_ids, int n, oww_stream_detect* h_overrides,
                             double* h_debounce);
/* The same rules over the calls of the bulk clip path (oww_predict_clips_ragged / _streams, oww_predict_clips): what
 * predict_clip(clip, padding, chunk_size, patience=..., threshold=..., debounce_time=...) returns after a reset, for
 * every clip at once.  Stateless: it uses neither the handle's detector nor its streams.
 *   h_labels, n_labels (1..256), debounce_time: as oww_set_detector, checked the same way.
 *   d_scores [rows][oww_n_outputs]: the raw rows of the clip call; only rows of calls that step a chunk are read.
 *   h_row_offsets (host int64 [n_clips + 1], 0 first, non-decreasing): clip i's calls are rows [off[i], off[i+1]), in call
 *     order, each clip from an empty history.  chunk_size: samples per call (>= 1).  Call j of a clip steps k = floor((j+1)
 *     c / 1280) - floor(j c / 1280) chunks (oww_clip_schedule; d_stepped of the clip call is 1 exactly there), has count
 *     j and prepared 1280 k samples, or ((j+1) c) mod 1280 when k = 0 - what AudioFeatures._streaming_features returns.
 *   d_verified (may be NULL) [rows][n_labels]: on a call with k = 0, a label whose entry is not NaN and whose prediction
 *     (the repeat, or 0.0) is >= verifier_threshold takes that entry instead, before the zeroing of the first five -
 *     Model.predict re-verifies a repeated prediction on the clip's newest window.
 *   d_final [rows][n_labels] (may be NULL): the predictions.  d_n_events / d_events / max_events as oww_detect, with the
 *     events in ascending (clip, label, call) order: `stream` = clip, `index` = call.
 * Stream-ordered, no synchronisation; two launches, one without d_n_events, none for n_clips 0 (d_n_events is then
 * set to 0).  The row offsets are staged before the call returns.  OWW_EINVAL before anything is enqueued: the
 * label checks, null pointers, offsets that do not start at 0 or decrease, chunk_size < 1, and the output checks of
 * oww_detect.                                                                                                       */
int oww_detect_clips(oww_ctx* ctx, const oww_detect_label* h_labels, int n_labels, double debounce_time,
                     const float* d_scores, const float* d_verified, float verifier_threshold, const int64_t* h_row_offsets,
                     int n_clips, int chunk_size, float* d_final, oww_event* d_events, int max_events, int32_t* d_n_events,
                     void* stream);

/* ---- stream audio on the device (openwakeword/utils.py:164,403-430: AudioFeatures.raw_data_buffer) ------------------
 * With an audio history of H samples the handle keeps, per stream, the last H samples it stepped (int16 ring) and pos =
 * the samples it has stepped since its reset; the ring holds samples [max(0, pos - H), pos).  Every step appends exactly
 * the samples it steps, in stream order, in one launch per call before the frontend: oww_step, oww_step_host and
 * oww_step_host_submit n_chunks*1280 per stream, the ragged calls cnt[b]*1280 for stream b (a held stream is untouched).
 * Memory: 2*H + 8 bytes per stream (8192 streams x 10 s: 2.6 GB).  Samples a caller holds back (less than a chunk) are
 * not in the ring until a step consumes them.
 *   oww_set_audio_history - n_samples 0: off (frees); else a multiple of 1280, <= 960000 (60 s).  Synchronises the
 *                       device; every stream starts with an empty history.  Before oww_set_streams the state is
 *                       allocated by that call.  OWW_ENOMEM (or OWW_ECUDA) on a failed allocation, with history off.
 *   oww_get_audio     - row i of d_out [n][n_samples] <- samples [e - n_samples, e) of stream h_stream_ids[i], e =
 *                       h_end[i] (h_end NULL or h_end[i] < 0: the stream's pos).  An e beyond pos asks for audio after
 *                       an event once the stream has advanced far enough (post-roll).  d_pos [n] (may be NULL) receives
 *                       the stream's pos at that point in stream order.  Duplicate ids are allowed; 1 <= n_samples <= H.
 *   oww_capture_events - for the event list of oww_detect, read from device memory (enqueue it right after oww_detect,
 *                       before the host has read the count): row i < min(*d_n_events, max_events) of d_out
 *                       [max_events][n_samples] <- the last n_samples samples of stream d_events[i].stream, ending at its
 *                       pos; d_pos[i] (may be NULL) <- that pos.  Rows past the count are not written.  One CTA per
 *                       possible event; those past the count exit at once.
 *   oww_audio_export / _import - the history of streams h_stream_ids[i] <-> d_audio [n][H] oldest first (entry k is
 *                       sample pos - H + k; zeros before sample 0) and d_pos [n].  Import takes records of the same H
 *                       (a negative pos is taken as 0); duplicate ids fail with OWW_EINVAL.  Stream records
 *                       (oww_export_streams) do not carry the audio: move it with these two calls.
 * Samples outside [max(0, pos - H), pos) come out as zeros.  Every call is stream-ordered, ordered with the host-buffer
 * steps of oww_step_host_submit (the handle's own stream), and allocates nothing after the first (oww_get_audio grows
 * its id staging once when n exceeds the stream count).  OWW_EINVAL before anything is enqueued: no history, n_samples
 * outside its range (or, for oww_set_audio_history, not a multiple of 1280), a stream id out of range, a NULL output.
 * oww_reset / oww_reset_async empty the history of the streams they reset (one more launch), oww_set_streams that of
 * all.  A handle without history launches nothing for it.                                                              */
int oww_set_audio_history(oww_ctx* ctx, int n_samples);
int oww_get_audio(oww_ctx* ctx, const int32_t* h_stream_ids, const int64_t* h_end, int n, int n_samples, int16_t* d_out,
                  int64_t* d_pos, void* stream);
int oww_capture_events(oww_ctx* ctx, const oww_event* d_events, const int32_t* d_n_events, int max_events, int n_samples,
                       int16_t* d_out, int64_t* d_pos, void* stream);
int oww_audio_export(oww_ctx* ctx, const int32_t* h_stream_ids, int n, int16_t* d_audio, int64_t* d_pos, void* stream);
int oww_audio_import(oww_ctx* ctx, const int32_t* h_stream_ids, int n, const int16_t* d_audio, const int64_t* d_pos,
                     void* stream);

/* ---- ingest: every stream's packets at its own sample rate (the reference's server example resamples each packet on
 *      the host before Model.predict, examples/web/streaming_server.py:54-60, and AudioFeatures keeps the remainder
 *      below a chunk on the host, openwakeword/utils.py:409-430) -------------------------------------------------------
 * Rates: r in {8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000}; with g = gcd(16000, r), up = 16000/g and
 * down = r/g.  16000 is the identity (a copy).  For the other rates the filter is scipy's resample_poly design: mr =
 * max(up, down), half = 10*mr, N = 2*half + 1, h[k] = sinc((k - half)/mr) * kaiser(N, beta 5)[k] for k < N, normalised to
 * sum 1 and multiplied by up; computed in double on the host and rounded once to fp32.  A phase has at most 61 taps.
 * Stream b's 16 kHz output is y = upfirdn(h, x, up, down) of its input x since its restart (causal: 0.6 - 1.3 ms of
 * delay).  After S input samples the first A(S) = ceil(S*up/down) outputs depend on no later input: those are final and
 * are staged.  An 80 ms packet at any rate of the table therefore yields exactly 1280 samples.  Each output is one fp32
 * sum over its phase's taps in a fixed order (newest input sample first), so the 16 kHz samples are the same bits whatever the
 * packet split; it is converted to int16 by round-half-even with saturation (sum |h| of a phase reaches 2.24, so
 * full-scale input can overshoot).
 * Per stream the handle keeps the rate, the last 128 input samples (the filter history), and a staging row of the 16 kHz
 * samples not yet stepped; its capacity is C = max_chunks*1280 + 1279 samples (8192 streams at max_chunks 2: 63 MB).
 * The input count S, the staged count and the rate live on the host, so no call reads the device.  Nothing is allocated
 * and nothing is launched for ingest until the first oww_set_input_rates.
 *   oww_set_input_rates - stream h_stream_ids[i] (NULL: all streams, n = the stream count) takes input at h_rates[i]
 *                       from the next oww_ingest on; its resampler restarts (history zero, S = 0), its staged samples are
 *                       kept.  The first call allocates the state (every other stream at 16000) and synchronises the
 *                       device; later calls enqueue nothing.  OWW_EINVAL: a rate outside the table, an id out of range.
 *   oww_ingest        - stream b's new samples are d_in[h_offsets[b] .. h_offsets[b+1]) (int16 at its rate; host int64
 *                       offsets, n_streams + 1 entries, non-decreasing, first >= 0; a stream may get none).  One launch
 *                       resamples every stream and writes its new final samples behind its staged ones; then the
 *                       staged samples step as oww_step_ragged steps them: stream b steps chunks[b] = floor(staged / 1280)
 *                       chunks, d_scores rows as oww_step_ragged writes them (held rows are not written), with the audio
 *                       history, detector inputs, verifiers and head banks of that call.  The rest (< 1280 samples) stays
 *                       staged.  h_chunks_out[b] (may be NULL) <- chunks[b]; h_prepared_out[b] (may be NULL) <- what
 *                       AudioFeatures.__call__ returns: chunks[b]*1280, or the staged count when the stream stepped
 *                       nothing - oww_detect's h_prepared.  Both are filled on the host before the call returns, with no
 *                       synchronisation.  The per-stream table is staged through a ring of four pinned buffers (a call
 *                       waits, host side, for the copy of the call four back).  OWW_EINVAL before anything is enqueued:
 *                       no ingest state, bad offsets, a NULL d_in with samples or a NULL d_scores, or a stream whose
 *                       staged plus new samples would exceed C (oww_ingest_capacity gives the limit).
 *   oww_ingest_capacity - pure host: h_max_in[b] (int64 [n_streams]) <- the most input samples stream b's next
 *                       oww_ingest may take.  A caller splits longer packets with it.
 *   oww_ingest_plan   - pure host, no handle or GPU: for a stream at `rate` on a handle of max_chunks, that has taken
 *                       n_before input samples since its restart and holds `staged` samples, an oww_ingest of n_in more
 *                       samples makes *n_out (may be NULL) new final samples, steps *chunks chunks and leaves *staged_after;
 *                       *max_in (may be NULL) <- oww_ingest_capacity's limit.  OWW_EINVAL: a rate outside the table, or
 *                       n_in over that limit (only *max_in is written then).
 *   oww_resampler_taps - pure host, no handle or GPU: the fp32 taps h (N of them; the first min(N, max) go to h_taps, which
 *                       may be NULL) and *up, *down the library uses for `rate`.  Returns N (0 at 16000), or OWW_EINVAL
 *                       outside the table.
 *   oww_ingest_export / _import - stream h_stream_ids[i] <-> h_rates[i], h_consumed[i] (S, int64), h_staged[i] (host), its
 *                       staged samples in row i of d_staged [n][staged_stride] int16 (the rest of the row zero on export),
 *                       and its history in d_hist [n][128] int16 (oldest first; zeros at 16000 Hz, which keeps none, and
 *                       before the first input).  Export fills the host arrays before it returns; with d_staged and d_hist
 *                       NULL it enqueues nothing (a query of the staged counts), else staged_stride must hold every
 *                       exported row.  Import takes rates from the table, h_staged[i] in
 *                       [0, C], distinct ids; a moved stream continues bit for bit.  Stream-ordered on `stream`.
 * oww_reset / oww_reset_async clear the staged samples and the history of the streams they reset and keep their rates;
 * oww_set_streams sets every stream to 16000 with nothing staged.  The steps of oww_step* do not touch the ingest state
 * (a caller that mixes them on one stream feeds that stream at one place only).                                          */
int oww_set_input_rates(oww_ctx* ctx, const int32_t* h_stream_ids, int n, const int32_t* h_rates, void* stream);
int oww_ingest(oww_ctx* ctx, const int16_t* d_in, const int64_t* h_offsets, int32_t* h_chunks_out, int32_t* h_prepared_out,
               float* d_scores, void* stream);
int oww_ingest_capacity(oww_ctx* ctx, int64_t* h_max_in);
int oww_ingest_plan(int rate, int max_chunks, int64_t n_before, int staged, int64_t n_in, int64_t* n_out, int32_t* chunks,
                    int32_t* staged_after, int64_t* max_in);
int oww_resampler_taps(int rate, float* h_taps, int max, int* up, int* down);
int oww_ingest_export(oww_ctx* ctx, const int32_t* h_stream_ids, int n, int32_t* h_rates, int64_t* h_consumed,
                      int32_t* h_staged, int16_t* d_staged, int64_t staged_stride, int16_t* d_hist, void* stream);
int oww_ingest_import(oww_ctx* ctx, const int32_t* h_stream_ids, int n, const int32_t* h_rates, const int64_t* h_consumed,
                      const int32_t* h_staged, const int16_t* d_staged, int64_t staged_stride, const int16_t* d_hist,
                      void* stream);

/* ---- pipelined detection from host audio: a serving loop's whole call (the reference's server example runs it per
 *      packet on the host, examples/web/streaming_server.py:40-68; examples/capture_activations.py keeps the audio of
 *      each activation) with nothing in between that waits for the device ------------------------------------------------
 *   oww_detect_host_submit - exactly oww_ingest(packets, h_offsets) followed by oww_detect(h_prepared = what that ingest
 *                       returned) and, with capture_samples > 0, oww_capture_events(capture_samples): stream b's packet is
 *                       h_packets[h_offsets[b] .. h_offsets[b+1]) (host int16 at the stream's rate; host int64 offsets,
 *                       n_streams + 1 entries, as oww_ingest).  Returns a ticket (0/1) without waiting; at most two are in
 *                       flight.  The packets [h_offsets[0], h_offsets[n_streams]) are staged through one of two pinned
 *                       slots of the handle, or, when that span is page-locked (cudaMallocHost, cudaHostRegister, torch
 *                       pin_memory), DMA'd straight from it: then it must stay untouched until the ticket is collected.
 *                       The copy runs on a copy stream, the work on the handle's own stream behind an event, so the copy
 *                       of one call overlaps the kernels of the other.  After the detect a delivery kernel reads the event
 *                       count on the device and writes it, the first min(count, max_events) events and with capture their
 *                       clip rows and ends into the slot's mapped host buffer: only the events found cross PCIe.  With
 *                       want_final the final predictions [n_streams][n_labels] follow as one copy.  No device allocation
 *                       once the slots have grown to the largest call (samples, max_events, capture_samples) so far.
 *   oww_detect_host_collect - waits for the ticket and copies its results out of the slot: *h_n_events <- the event count;
 *                       h_events <- the first min(count, max_events) events in oww_detect's (stream, label) order; with
 *                       capture, h_clips [that many][capture_samples] and h_ends (each clip's end, its stream's position);
 *                       h_chunks / h_prepared [n_streams] <- what oww_ingest returned; with want_final h_final [n_streams]
 *                       [n_labels].  Every output may be NULL (not delivered).  These are what the synchronous sequence
 *                       gives, bit for bit.  A ticket that is not in flight, or one collected before an older ticket, fails
 *                       with OWW_EINVAL.
 * Preconditions: ingest state (oww_set_input_rates; a 16 kHz stream takes the identity rate) and a detector; with capture
 * an audio history.  OWW_EINVAL before anything is enqueued, every stream unchanged: a third ticket while two are in
 * flight, no ingest state or weights, no detector, capture_samples < 0 or above the history (or any without one),
 * max_events < 0, offsets that are negative or decrease, a packet over its stream's capacity.  The host keeps each
 * stream's input and staged counts at submit time, so oww_ingest_capacity stays exact while calls are in flight and the
 * capacity check counts what earlier submits staged.
 * Ordering: a call made between two submits applies to the later one and not to the earlier one, as in the synchronous
 * loop - oww_reset / oww_reset_async, oww_set_stream_detection, oww_set_input_rates, oww_assign_*, and the export and
 * import of streams, detector histories, ingest state and audio are ordered against the handle's own stream, on
 * whichever stream they are enqueued.  Steps of oww_step_host_submit may be pending beside detect tickets: all their work
 * is ordered on the handle's own stream.  A stream must still be fed at one place only (ingest, above).               */
int oww_detect_host_submit(oww_ctx* ctx, const int16_t* h_packets, const int64_t* h_offsets, int max_events,
                           int capture_samples, int want_final, int* ticket);
int oww_detect_host_collect(oww_ctx* ctx, int ticket, oww_event* h_events, int32_t* h_n_events, int16_t* h_clips,
                            int64_t* h_ends, int32_t* h_chunks, int32_t* h_prepared, float* h_final);

/* ---- batch paths --------------------------------------------------------------------------- */
/* d_pcm [n_clips][n_samples] -> d_emb [n_clips][W][96], W = (T-76)/8+1 (utils.py:322).           */
int oww_embed_clips(oww_ctx* ctx, const int16_t* d_pcm, int n_clips, int n_samples, float* d_emb, void* stream);
/* predict_clip for n_clips equal-length clips, each from a FRESH state seeded with h_feature_init
 * (SURVEY.md F9): pad_samples zeros each side, 1280-sample steps, steps = len(range(0, L-1280, 1280)).
 * d_scores [n_clips][steps][oww_n_outputs].  Raw head outputs (the first-5-zeroing of
 * model.py:330-333 is label bookkeeping done by the host wrapper).  Equals streaming the padded clips through
 * fresh streams of this handle's configuration; uses none of the handle's streams.  No heads: returns at once.
 * The equal-length, chunk_size 1280 case of oww_predict_clips_ragged (every call steps one chunk).               */
int oww_predict_clips(oww_ctx* ctx, const int16_t* d_pcm, int n_clips, int n_samples, int pad_samples,
                      const float* h_feature_init, int n_rows, float* d_scores, void* stream);
/* Call schedule of predict_clip(clip, padding, chunk_size): on n_padded_samples = len + 2*pad samples it makes
 * len(range(0, L - chunk_size, chunk_size)) predict calls; AudioFeatures._streaming_features steps whole 1280-sample
 * chunks and keeps the remainder for the next call, so call j steps floor((j+1) c / 1280) - floor(j c / 1280) chunks
 * (0: the call only accumulated samples).  Writes that count for the first min(calls, max) calls (h_chunks_per_call may
 * be NULL) and returns the number of calls.  Pure host computation, usable without a GPU; the bulk path uses the same
 * arithmetic (csrc/oww_internal.h).                                                                                 */
int oww_clip_schedule(int chunk_size, int64_t n_padded_samples, int32_t* h_chunks_per_call, int max);
/* predict_clip over clips of any lengths, in one call, each from a FRESH state (as oww_predict_clips).  Clip i is
 * d_pcm[h_offsets[i] .. h_offsets[i+1]) (host int64 sample offsets, monotone; any lengths, 0 included); pad_samples
 * zeros each side; chunk_size samples per predict call, 1 .. max_chunks*1280.  Score rows are the clips' calls in input
 * order (clip i's rows start at the total call count of clips 0..i-1; oww_clip_schedule gives the counts):
 *   d_scores [rows][oww_n_outputs]: for a call that steps, per head the max over its chunk windows (verifier gates per
 *            chunk before the max, custom verifiers after it on the call's newest window: what oww_step returns for
 *            the same call).  Rows of calls that step no chunk are not written.
 *   d_stepped [rows] (may be NULL): set to 1 on the rows of calls that step; other bytes are not written.
 *   d_emb (may be NULL) [sum of the clips' steps][96]: the embedding rows each clip's steps appended, clip by clip.
 * Clips are sorted by length into slabs of neighbours; a shorter clip of a slab runs on over virtual zeros, which leaves
 * its own calls' rows unchanged (oww_clip_slab_plan reports the steps this computes).  No heads: returns at once.   */
int oww_predict_clips_ragged(oww_ctx* ctx, const int16_t* d_pcm, const int64_t* h_offsets, int n_clips, int pad_samples,
                             int chunk_size, const float* h_feature_init, int n_rows, float* d_scores, uint8_t* d_stepped,
                             float* d_emb, void* stream);
/* Same, but clip i is scored as stream h_clip_streams[i] (host, in [0, n_streams); repeats allowed) would score it: the
 * head-bank slots and verifier slots that stream is assigned when the call is enqueued, instead of the clip slots, for
 * the banks of ordinary heads and of head banks alike.  Needs oww_set_streams; the handle's streams are not touched.
 * An id out of range, or h_clip_streams NULL with n_clips > 0, fails with OWW_EINVAL before anything is enqueued.    */
int oww_predict_clips_streams(oww_ctx* ctx, const int16_t* d_pcm, const int64_t* h_offsets, int n_clips, int pad_samples,
                              int chunk_size, const float* h_feature_init, int n_rows, float* d_scores, uint8_t* d_stepped,
                              float* d_emb, const int32_t* h_clip_streams, void* stream);
/* The slabs oww_predict_clips_ragged would run for clips of h_steps[i] chunks each (ctx may be NULL: the default
 * configuration): returns the slab count, and the steps the slabs compute and the steps the clips need.  Pure host. */
int oww_clip_slab_plan(oww_ctx* ctx, const int32_t* h_steps, int n_clips, int64_t* h_steps_computed, int64_t* h_steps_needed);
/* Whole clips at any rate of the ingest table, resampled to 16 kHz without state (the reference converts a corpus to
 * 16 kHz with ffmpeg / sox first, openwakeword/data.py:convert_clips).  A clip x of S samples at rate r, with pad_samples
 * = pad 16 kHz samples of padding, becomes the first A(S) + 2*pad outputs of upfirdn(h, zeros(pad*down/up) ++ x ++
 * zeros(pad*down/up), up, down), with h, up, down and A of the ingest section above and each output computed exactly as
 * oww_ingest computes it (the same fp32 FMA chain and int16 rounding).  So the first pad outputs are 0, the next A(S) are
 * the samples oww_ingest makes final for x on a fresh stream, bit for bit, and the last pad hold the filter's tail (at
 * most 39 nonzero samples), then zeros: the whole is what a fresh stream makes of the padded clip.  At 16000 a clip is
 * copied between pad zeros.
 *   oww_resample_clip_plan - pure host, no handle or GPU: *n_out (may be NULL) <- A(n_in) + 2*pad_samples.  OWW_EINVAL:
 *                       a rate outside the table, a negative n_in or pad_samples, or a pad_samples the rate's up factor
 *                       does not divide (every up of the table divides 640, so whole seconds always work).
 *   oww_resample_clips - clip i is d_in[h_in_offsets[i] .. h_in_offsets[i+1]) at h_rates[i] Hz (host arrays, n_clips + 1
 *                       offsets, non-decreasing, first >= 0; rates may differ between clips; lengths 0 and 1 are legal);
 *                       its outputs go to d_out[h_out_offsets[i] .. h_out_offsets[i+1]), pads included, and
 *                       h_out_offsets[i+1] - h_out_offsets[i] must equal oww_resample_clip_plan's count.  One launch
 *                       over tiles of 2048 outputs; the pads are never read from memory.  The first call uploads the
 *                       filter tables (a synchronous copy); a call waits, host side, until the previous call's launch has
 *                       read its tables.  The handle's streams and ingest state are not touched, and a handle that never
 *                       calls it allocates nothing for it.  OWW_EINVAL before anything is enqueued: bad offsets or rates,
 *                       a pad the up factor does not divide, output offsets that do not match the plan, NULL buffers. */
int oww_resample_clip_plan(int rate, int64_t n_in, int pad_samples, int64_t* n_out);
int oww_resample_clips(oww_ctx* ctx, const int16_t* d_in, const int64_t* h_in_offsets, const int32_t* h_rates, int n_clips,
                       int pad_samples, int16_t* d_out, const int64_t* h_out_offsets, void* stream);

/* ---- mixing clips with background noise and room impulse responses (openwakeword/data.py:294-527: mix_clips_batch,
 * mix_clip, truncate_clip and speechbrain's reverberate), the test clips of a false-reject evaluation ----------------
 * Foreground and background clips are packed int16 (clip i is d_x[h_x_off[i] .. h_x_off[i+1]), host int64 offsets,
 * non-decreasing, first >= 0), RIRs packed float32 the same way.  A sample s is read as s / 32768.  Mixture i, with the
 * record p = h_params[i] and N = n_samples for every mixture of the call, is computed as (real arithmetic):
 *   1. f[k] = fg clip p.fg at p.fg_start + k, k < p.fg_len (the window is the host's truncation of the clip)
 *   2. b[n] = bg clip p.bg at (p.bg_offset + n) mod len_bg, n < N (tiling of a short background, crop of a long one)
 *   3. g = 10^(p.snr_db / 20) * |b|_2 / |f|_2;  m = b;  m[p.start + k] += g f[k];  m /= 2        (data.py:491-496)
 *   4. p.rir >= 0, h the RIR of L taps: d = first index of max |h[k]|, a0 = mean |m|,
 *      y[n] = sum_{k<L} h[k] m[(n - k + d) mod N]  (circular, aligned on the direct path), y *= a0 / (mean |y| + 1e-14)
 *      (speechbrain's reverberate(x, h, rescale_amp="avg") as its published source reads; not compared against it);
 *      p.rir < 0: y = m
 *   5. p.volume >= 0: y *= p.volume / max_n y[n] (the signed maximum, data.py:454); else y /= max(max_n |y[n]|, 1)
 *   6. out[i][n] = clamp(trunc(32767 y[n]), -32768, 32767).  The reference's astype(int16) wraps instead; saturation
 *      is deliberate (a negative peak can exceed full scale under the signed-maximum rule).
 * d_valid[i] = 0 when |f|_2 = 0, |b|_2 = 0 or (with a volume) max y <= 0: such a row is written as zeros; and when the
 * row's largest int16 sample is 0 (what data.py:466 means to drop).  Otherwise 1.
 * Device arithmetic: norms and the mixture in float64, m stored as float32; the reverb as a banded circulant GEMM on the
 * tensor cores with fp16 hi/lo split operands (three products) and fp32 accumulation, the taps scaled by a power of two
 * so that the largest is in [0.5, 1); the rescale and level in float64.  Launches per call: two without any reverb, three
 * with, whatever n_mix.  Stream-ordered: the call returns once its tables are enqueued; it waits, host side,
 * until the previous call's launches have read their tables, and it may (re)allocate its scratch (n_mix * N floats,
 * plus as many for the reverberated rows) with cudaMalloc, which synchronises the device.
 *   OWW_EINVAL before anything is enqueued: N <= 0, negative counts, bad offsets, an index out of range, a foreground
 *   window outside its clip, an empty background, bg_offset outside [0, len_bg), start < 0 or start + fg_len > N,
 *   an empty RIR or one longer than N, a non-finite snr_db or volume, NULL buffers.  n_mix = 0 enqueues nothing. */
typedef struct oww_mix_params {
    int32_t fg, bg, rir;       /* clip indices; rir = -1: no reverb */
    int32_t reserved;          /* 0 */
    int64_t fg_start, fg_len;  /* foreground window */
    int64_t bg_offset;         /* background sample at output 0, in [0, len_bg) */
    int64_t start;             /* output sample of the foreground's first sample */
    double snr_db;
    double volume;             /* < 0: no volume, normalise to [-1, 1] only where needed */
} oww_mix_params;
int oww_mix_clips(oww_ctx* ctx, const int16_t* d_fg, const int64_t* h_fg_off, int n_fg,
                  const int16_t* d_bg, const int64_t* h_bg_off, int n_bg,
                  const float* d_rir, const int64_t* h_rir_off, int n_rir,
                  const oww_mix_params* h_params, int n_mix, int64_t n_samples,
                  int16_t* d_out, uint8_t* d_valid, void* stream);

/* ---- score metrics on the device (openwakeword/metrics.py:24-100) --------------------------------
 * d_scores holds n_series score sequences of n_frames float32 (or float64) each, series i at d_scores + i*series_stride.
 * oww_metrics_false_positives: h_counts[i][j] = get_false_positives(series i, h_thresholds[j], grouping_window)
 * with the reference's grouping rule (restated in oracle/metrics.py); generate_roc_curve_fprs is this count at
 * np.linspace(0.01, 0.99, n_points) divided by the hours the series spans.
 * oww_metrics_count_ge: h_counts[j] = number of the n scores >= h_thresholds[j] (generate_roc_curve_tprs * len).
 * The _f64 forms take float64 scores and are otherwise the same.
 * Every comparison is (double)score >= h_thresholds[j].  To reproduce NumPy's `scores >= threshold` in the dtype D it
 * promotes to, round the threshold to D before passing it (openwakeword_b200.metrics does): widening the scores and
 * a D-rounded threshold to double is exact, so the double comparison is exactly the comparison in D.
 * 1..4096 thresholds per false-positive call, 1..64 per count call, n_series >= 1, n_frames >= 0, n >= 0; anything
 * else, or a NULL pointer, is OWW_EINVAL with nothing launched.  Both synchronise. */
int oww_metrics_false_positives(oww_ctx* ctx, const float* d_scores, int64_t series_stride, int n_series, int n_frames,
                                const double* h_thresholds, int n_thresholds, int grouping_window, int32_t* h_counts, void* stream);
int oww_metrics_false_positives_f64(oww_ctx* ctx, const double* d_scores, int64_t series_stride, int n_series, int n_frames,
                                    const double* h_thresholds, int n_thresholds, int grouping_window, int32_t* h_counts,
                                    void* stream);
int oww_metrics_count_ge(oww_ctx* ctx, const float* d_scores, int64_t n, const double* h_thresholds, int n_thresholds,
                         uint64_t* h_counts, void* stream);
int oww_metrics_count_ge_f64(oww_ctx* ctx, const double* d_scores, int64_t n, const double* h_thresholds, int n_thresholds,
                             uint64_t* h_counts, void* stream);

/* ---- parity instrumentation --------------------------------------------------------------- */
/* Runs the embedding CNN on d_windows [n][76][32] (n <= window_batch) up to and including conv
 * layer `layer` (0..18) and its max-pool, and writes that activation as NHWC float32
 * [n][T][F][C] to d_out - used by the tests to localise a mismatch layer by layer.             */
int oww_debug_layer(oww_ctx* ctx, const float* d_windows, int n, int layer, float* d_out, void* stream);

/* Geometry plan of the fused incremental CNN kernel for groups of `group` streams, as raw int32
 * (struct IncPlan of csrc/oww_internal.h); returns the number of ints written (> 0) or an error.
 * oww_debug_inc_plan: the full 20-layer plan.  oww_debug_inc_cut_plan: n_layers conv layers inside
 * the kernel - 0 or 20 for the full plan, split_from for the cut plan of cnn_mode 3 (the fused kernel
 * stops after the pooled layer split_from - 1).  group 0 with a handle: the plan that handle's fused kernel runs,
 * whose first int is the group size the library chose for its stream count (n_streams, n_layers ignored).
 * Pure host computation (usable without a GPU): tests/test_inc_plan.py replays it in NumPy.          */
int oww_debug_inc_plan(oww_ctx* ctx, int group, int n_streams, int32_t* out, int max_ints);
int oww_debug_inc_cut_plan(oww_ctx* ctx, int group, int n_streams, int n_layers, int32_t* out, int max_ints);

/* cnn_mode 3 only, instrumentation: oww_debug_inc_clocks arms a clock buffer; the next step then records clock64()
 * stamps taken by CTA 0 on its first group; oww_debug_inc_clocks_read synchronises and returns 104 values:
 * [0..19] start of each layer phase, [20] end of layer 19, per layer l [61+l] phase start -> first accumulator ready,
 * [81+l] phase start -> last tile stored, [92..97] frontend phases of warp 0, [101] group start (before the fused
 * frontend), [102] end of the fused heads phase (0 when the step was not fused); other entries stay 0. */
int oww_debug_inc_clocks(oww_ctx* ctx, int64_t* h_unused);
int oww_debug_inc_clocks_read(oww_ctx* ctx, int64_t* h_out104);
/* Instrumentation of the mirror-path heads kernel (heads_grp.cu): the first call arms the stamps, later calls synchronise
 * and return 8 clock64() values per head (CTA 0 of its launch): [0] start, [1] producer done, [2] first-layer
 * accumulators complete, [4] scores stored; the other entries stay 0. */
int oww_debug_heads_clocks(oww_ctx* ctx, int64_t* h_out64);

/* ---- multi-GPU gather over peer memory (one process per GPU) ---------------------------------
 * The reference has no multi-device path; SURVEY.md section 8e defines the only exchange of the sharded hot path: the
 * per-step scores float32[B/G][n_labels] of every rank gathered on one rank.  Instead of a collective call after the
 * step, a rank moves its finished score block into the gathering rank's memory (a buffer opened with oww_peer_open)
 * with oww_peer_copy - one DMA over NVLink; d_scores of oww_step may also point into the mapping directly, at the
 * price of scattered 4-byte remote stores - then publishes a step counter with oww_peer_signal; the gathering rank
 * orders its consumer behind oww_peer_wait.  openwakeword_b200.distributed.PeerGather drives the protocol
 * (double-buffered slots, acknowledgement counters); checked by tests/test_gpu_multi.py on two GPUs.
 *   oww_peer_alloc  - cudaMalloc'd, zero-filled buffer on this handle's device + its 64-byte CUDA IPC handle
 *   oww_peer_open   - map another process's buffer (peer access is enabled lazily); oww_peer_close unmaps it
 *   oww_peer_signal - stream-ordered: after all earlier work of `stream`, *d_flag = value (system-scope release;
 *                     d_flag may be local or peer-mapped)
 *   oww_peer_wait   - stream-ordered: later work of `stream` starts once d_flags[i*stride] >= value for all i < n
 *                     (n <= 1024).  If that takes longer than timeout_s (<= 0: 10 s) the kernel gives up, the stream
 *                     goes on and oww_peer_status reports the timeout - a dead peer can neither hang the GPU nor
 *                     poison the CUDA context.                                                                    */
int oww_peer_alloc(oww_ctx* ctx, size_t bytes, void** d_ptr, unsigned char handle_out[64]);
int oww_peer_free(oww_ctx* ctx, void* d_ptr);
int oww_peer_open(oww_ctx* ctx, const unsigned char handle[64], void** d_ptr);
int oww_peer_close(oww_ctx* ctx, void* d_ptr);
/* stream-ordered block copy into (or out of) a peer mapping (4-byte words, a copy kernel with coalesced 16-byte stores:
 * full lines over NVLink instead of the step kernels' scattered 4-byte stores) - the way
 * openwakeword_b200.distributed moves a rank's [rows x columns] score block */
int oww_peer_copy(oww_ctx* ctx, void* d_dst, const void* d_src, size_t bytes, void* stream);
int oww_peer_signal(oww_ctx* ctx, uint64_t* d_flag, uint64_t value, void* stream);
int oww_peer_wait(oww_ctx* ctx, const uint64_t* d_flags, int n, int stride, uint64_t value, double timeout_s, void* stream);
/* a wait that ran into its timeout lets the stream continue and raises a flag on the handle: *timed_out = 1 (the flag is
 * cleared by the read).  Synchronises the device. */
int oww_peer_status(oww_ctx* ctx, int* timed_out);

/* ---- introspection ------------------------------------------------------------------------- */
uint64_t oww_launch_count(const oww_ctx* ctx);       /* kernels launched by this handle so far   */
/* n_slots > 0: every following oww_step / oww_step_host brackets its three stages (mel, embedding
 * CNN + ring append, heads) with CUDA events on the launching stream, step k in slot k % n_slots;
 * 0 disables.  oww_stage_ms synchronises on the recorded events and returns the per-step AVERAGE
 * {mel, cnn, heads} milliseconds over the steps recorded since enabling (at most n_slots).      */
int oww_enable_stage_timing(oww_ctx* ctx, int n_slots);
int oww_stage_ms(oww_ctx* ctx, float out_ms[3]);

#ifdef __cplusplus
}
#endif
#endif /* OWWB200_H */
