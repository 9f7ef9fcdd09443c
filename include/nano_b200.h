/*
 * nano_b200.h -- C-ABI of the H100 (sm_90a) batch-1 decode engine for bd4sur/Nano model files.
 *
 * This is the "thin C-ABI" under the reference's own host API (infer/infer.h, infer/tensor.h): the
 * reference-facing shim (include/nano_infer_abi.h, nano_b200/csrc/infer_b200.c) implements
 * llm_context_init / generate_next_token / llm_session_step / ... on top of these entry points, and
 * tests / bench.py bind them with ctypes.  Plain pointers and sizes only; no torch types.
 *
 * Every entry point returns 0 on success or a negative NB200_E* code; nb200_last_error() gives the
 * message.  There is no CPU fallback: without a CUDA device every compute entry point fails.
 *
 * Reference interfaces replaced (paths relative to the reference repo):
 *   nb200_engine_create   <- load_llm_from_buffer   infer/infer.c:323-326 (parse_model_file :220-320,
 *                            memory_map_params :100-217, malloc_fwd_buffer :15-85)
 *   nb200_engine_destroy  <- free_llm               infer/infer.c:369-404
 *   nb200_forward         <- llm_forward            infer/infer.c:971-1018
 *   nb200_read_logits     <- FwdBuffer.logits       infer/infer.h:139 (host float* in the reference)
 *   nb200_next_greedy     <- generate_next_token    infer/infer.c:1135-1193 (temperature == 0 branch:
 *                            repetition penalty :1156-1167 + sample_argmax :1026-1037)
 *   nb200_next_sampled    <- generate_next_token    infer/infer.c:1156-1189 (temperature > 0: softmax :616-634,
 *                            sample_top_p :1062-1109 with the caller's xorshift coin utils.c:959-970)
 *   nb200_decode_greedy   <- the llm_session_step loop of infer/infer.c:1243-1310 with the token fed back
 *                            on the device (no host round trip per token)
 *   nb200_op_*            <- rmsnorm :601, matmul :637, matmul_quant :654 (infer/infer.c); quantize tensor.c:21,
 *                            quantize_tensor_q4k_in_situ tensor.c:281, matmul_q4k tensor.c:438.  (softmax :616, rope :681 and
 *                            rope_qwen3 :692 have no stand-alone entry point: they exist only fused inside the attention kernels
 *                            and are pinned through the exact-mode K-row / logits tests.)
 */
#ifndef NANO_B200_H
#define NANO_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NB200_OK 0
#define NB200_EINVAL (-1)   /* bad argument / unsupported model shape */
#define NB200_ECUDA (-2)    /* CUDA runtime error (message in nb200_last_error) */
#define NB200_ENODEV (-3)   /* no CUDA device: the engine has no CPU path */
#define NB200_ENOMEM (-4)

/* engine creation flags */
#define NB200_FLAG_EXACT 0x1u      /* exact mode: reference-order fp32 reductions (validation, slower) */
#define NB200_FLAG_NO_GRAPH 0x2u   /* launch kernels directly instead of replaying a CUDA graph */
#define NB200_FLAG_NO_PDL 0x4u     /* disable programmatic dependent launch */
#define NB200_FLAG_NO_STREAM 0x10u /* do not use the grid-wide streaming kernel (per-CTA TMA weight ring, one launch per run of tokens) */

/* quantisation / architecture ids: identical to infer/tensor.h:72-76 and infer/infer.h:45-47 */
#define NB200_QUANT_F32 0x00u
#define NB200_QUANT_Q80 0x80u
#define NB200_QUANT_Q4K 0x42u
#define NB200_ARCH_NANO 0u
#define NB200_ARCH_QWEN2 2u
#define NB200_ARCH_QWEN3 3u

typedef struct nb200_engine nb200_engine;

/* mirrors LLM_Config + LLM.arch/quant_type/group_size (infer/infer.h:89-99,159-166) plus derived dims */
typedef struct nb200_config {
    uint32_t arch, quant, group_size;
    uint32_t block_size, vocab_size, n_layer, n_embd, n_head, n_kv_head, n_hidden, tied, head_dim;
    uint32_t q_dim, kv_dim, max_seq_len;
    uint32_t tp_rank, tp_size;
    uint32_t reserved[7];   /* [0] execution path: 4 | CTAs << 8 | C << 24 streaming kernel on a grid of that many CTAs, launched in clusters of C CTAs (0: plain launch), 1 CUDA graph, 0 direct launches; [1], [2] creation-time calibration:
                               us per token of the streaming kernel / of the multi-kernel graph (0 = the choice was not measured);
                               multi-kernel path, recorded when a kernel is launched or captured into the graph:
                               [3] matvec variants used since creation, bit 3 * epilogue + {0: RB 1, 1: RB 2, 2: RB 4} with the
                                   epilogues store 0, qkv 1, residual 2, swiglu 3, classifier 4 (the exact-mode F32 kernel sets none);
                               [4] attention kernel of the last layer run: 0 none yet, 1 exact, 2 generic split-KV,
                                   3 | kv_mul << 8 the split-KV kernel specialised for that kv_mul;
                               nb200_prefill and nb200_verify_greedy: [5] positions per chunk M (0 until the first call), [6] the
                                   attention kernel of the last prefill or verify pass, encoded as [4] */
} nb200_config;

/* fields readable with nb200_read_buffer (same numbering as oracle probes) */
enum nb200_field {
    NB200_F_X = 0,       /* residual stream x            [n_embd]                 */
    NB200_F_XBA = 2,     /* attention output             [q_dim]                  */
    NB200_F_HB = 4,      /* SwiGLU output                [n_hidden]               */
    NB200_F_Q = 6,       /* raw (pre-norm/rope) q        [q_dim]                  */
    NB200_F_LOGITS = 9,  /* logits                       [vocab]                  */
    NB200_F_KROW = 13,   /* K cache row (layer, pos)     [kv_dim] in reference order */
    NB200_F_VROW = 14,   /* V cache row (layer, pos)     [kv_dim]                 */
    NB200_F_ACT_I8 = 20, /* last dumped Q80 activation codes (as int8 packed in bytes) */
    NB200_F_ACT_SCALE = 21
};

const char *nb200_last_error(void);
int nb200_device_count(void);

/* `image` is a complete model file image (header + tokenizer section + params).  The engine uploads
 * what it needs to HBM; the image may be released after the call returns. */
int nb200_engine_create(nb200_engine **out, const uint8_t *image, uint64_t image_bytes,
                        uint32_t max_seq_len, int device, uint32_t flags);
void nb200_engine_destroy(nb200_engine *e);

/* Tensor parallelism over NVLink peer memory (SURVEY 8e; the reference has no counterpart, it is one CPU
 * process).  Rank r of `tp_size` uploads its row slice of every matrix (whole kv-head groups for QKV and
 * attention; contiguous row ranges for O, W1|W3, W2 and the classifier) and allocates an "exchange block"
 * its peers write into.  After creation every rank must be attached to the others' blocks, either
 *   - across processes: nb200_tp_export() -> 64-byte CUDA IPC handle; all-gather the handles with the
 *     host's own transport (torch.distributed, MPI, a pipe); nb200_tp_attach_ipc(handles in rank order), or
 *   - inside one process: nb200_tp_attach_local(array of the tp_size engines in rank order).
 * From then on all ranks issue the SAME sequence of forward / next_greedy / decode_greedy calls with the
 * same arguments (in lock-step; a rank that waits ~4 s for a missing peer fails with NB200_ECUDA).  Every
 * rank returns the same token ids; nb200_read_logits fills only this rank's slice
 * [rank*V/tp_size, (rank+1)*V/tp_size) of the vector.  Results are bit-identical to tp_size == 1.
 * Fast mode only; needs n_kv_head, n_embd/2, n_hidden and vocab divisible by tp_size, head_dim <= 128. */
int nb200_engine_create_tp(nb200_engine **out, const uint8_t *image, uint64_t image_bytes,
                           uint32_t max_seq_len, int device, uint32_t flags, uint32_t tp_rank, uint32_t tp_size);
int nb200_tp_export(nb200_engine *e, void *handle64);
int nb200_tp_attach_ipc(nb200_engine *e, const void *handles /* tp_size x 64 bytes, rank order */);
int nb200_tp_attach_local(nb200_engine *e, nb200_engine *const *group /* tp_size engines, rank order */);

/* LoRA plug-in (fp32 low-rank branches on wq/wk/wv/wo of the Nano architecture):
 *   nb200_lora_load    <- load_lora_from_buffer  infer/infer.c:513-519 (parse_lora_file :436-500); image_bytes 0 = trust the header
 *   nb200_lora_enable  <- the use_lora switch of llm_forward / transformer_block_forward  infer/infer.c:713, 792, 898
 *   nb200_lora_unload  <- free_lora              infer/infer.c:521-534
 * While a plug-in is active the engine runs its multi-kernel path (two small extra kernels per site and layer). */
int nb200_lora_load(nb200_engine *e, const uint8_t *image, uint64_t image_bytes);
int nb200_lora_enable(nb200_engine *e, int on);
int nb200_lora_unload(nb200_engine *e);

int nb200_get_config(const nb200_engine *e, nb200_config *cfg);

/* Positions: every call that takes one refuses pos >= min(max_seq_len, block_size) with NB200_EINVAL.  The RoPE table has
 * block_size rows, so a position past it has no defined result (the reference reads past its table there).  A context with
 * max_seq_len > block_size is still legal; its rows from block_size on stay zero and non-causal attention reads them as such. */

/* one token through the network; logits stay in HBM.  is_causal=0 is the reference's seq2seq mode
 * (attention over all max_seq_len cache rows, infer.c:849). */
int nb200_forward(nb200_engine *e, uint32_t token, uint32_t pos, uint32_t is_causal);
int nb200_read_logits(nb200_engine *e, float *host_logits);

/* generate_next_token with temperature 0.  `ids` is the caller's output_ids array (host); ids[pos] is
 * consumed, ids[0..pos) feed the repetition penalty.  When is_prefilling the forward pass still runs
 * and ids[pos+1] is returned (infer.c:1146-1149). */
int nb200_next_greedy(nb200_engine *e, const uint32_t *ids, uint32_t pos, int is_prefilling,
                      float repetition_penalty, uint32_t *next_token);

/* generate_next_token with temperature > 0 (infer/infer.c:1156-1189), entirely on the device: repetition penalty, division by the
 * temperature, softmax (:616-634, sequential normaliser), cutoff filter, probability-descending order with ties in index order
 * (what glibc's stable qsort gives `compare` :1053-1059), cumulative top-p cut and CDF walk (sample_top_p :1062-1109).
 * `coin` is the caller's random_f32(&sampler->rng_state) draw (utils.c:959-970).  Returns the sampled id and, if top6 != NULL, the
 * six most probable ids (what the reference hands its observation hook).  32 bytes come back instead of vocab_size * 4. */
int nb200_next_sampled(nb200_engine *e, const uint32_t *ids, uint32_t pos, float repetition_penalty, float temperature, float top_p,
                       float coin, uint32_t *next_token, uint32_t *top6);

/* Device-resident greedy loop: ids[0..n_prompt) is the prompt; positions 0..n_total-2 are run and
 * ids[n_prompt..n_total) are filled with greedy tokens (prompt positions are teacher-forced exactly like
 * llm_session_step).  device_ms (optional) receives the CUDA-event time of the decode segment
 * (positions >= n_prompt-1); prefill_ms the prompt segment.  n_total <= min(max_seq_len, block_size) + 1. */
int nb200_decode_greedy(nb200_engine *e, uint32_t *ids, uint32_t n_prompt, uint32_t n_total,
                        float repetition_penalty, float *prefill_ms, float *device_ms);

/* Batched prompt prefill (no reference counterpart: infer.c:1146-1149 runs the prompt token by token and discards the logits).
 * `ids` is the caller's output_ids array, as for nb200_next_greedy.  Runs the causal forward pass of ids[pos0 .. pos0+n) at
 * positions pos0 .. pos0+n-1 in chunks of up to 16 positions per pass over the
 * weights (nb200_config.reserved[5] reports the chunk size after the first call) and writes their K/V rows; no classifier, no
 * logits, no state besides those rows.  The session then continues with nb200_forward / nb200_next_greedy / nb200_next_sampled
 * at pos0+n, on either execution path.  The K/V rows are bit-identical to what nb200_forward at the same positions writes on
 * the multi-kernel path (NB200_FLAG_NO_STREAM) of an engine created with the same flags; in exact mode that is the strict
 * reference.  Rows outside [pos0, pos0+n) are not touched.  device_ms (optional): CUDA-event time of the call.
 * NB200_EINVAL, with nothing written: n == 0, pos0 + n > min(max_seq_len, block_size), an id >= vocab_size, a tensor-parallel
 * engine, an active LoRA plug-in.
 * Not covered: the streaming kernel's own prompt loop (nb200_decode_greedy and the shim keep running the prompt token by token,
 * so their fast-mode K/V bits do not change), tensor cores, non-causal (seq2seq) attention. */
int nb200_prefill(nb200_engine *e, const uint32_t *ids, uint32_t pos0, uint32_t n, float *device_ms);

/* Speculative greedy decoding (no reference counterpart), lossless: the ids are exactly those of nb200_next_greedy.
 *   nb200_verify_greedy  ids[0..pos] are known (ids[pos] is consumed, as for nb200_next_greedy) and ids[pos+1 .. pos+n) are n-1
 *                        drafted ids.  One pass over the weights runs positions pos .. pos+n-1 as a prefill chunk and the
 *                        batch's classifier and argmax on each, so g_j, the greedy id at pos+j, is exactly what
 *                        nb200_next_greedy(e, ids, pos+j, 0, repetition_penalty) returns on an engine created with the same flags
 *                        plus NB200_FLAG_NO_STREAM (its penalty reads ids[0..pos+j), drafts included).  *n_accepted = a, the
 *                        largest count with g_j == ids[pos+j+1] for every j < a; ids[pos+a+1] = g_a (the correction, or the
 *                        bonus id when every draft is accepted), so ids needs pos+n+1 entries; ids past pos+a+1 keep the
 *                        rejected drafts.  Afterwards the engine is where nb200_next_greedy at pos .. pos+a leaves it: K/V rows
 *                        pos .. pos+a written, rows from pos+a+1 on as they were before the call (the rows the pass wrote there
 *                        are saved first and restored), nb200_read_logits gives the penalised logits at pos+a, and the next
 *                        nb200_next_greedy / nb200_next_sampled at pos+a+1 gives the same bits, on either execution path.
 *                        Launches: the chunk's 1 + 6 * n_layer, the classifier, the argmax; when repetition_penalty != 1 also
 *                        one seen-row kernel, and nb200_next_greedy's seen-set update when ids[0..pos) has new ids.  One host
 *                        synchronise.  nb200_config.reserved[5] / [6] report M and the
 *                        attention kernel after a call, as after nb200_prefill.  device_ms (optional): CUDA-event time of the pass.
 *                        The workspace (M logits rows, M seen rows, the saved K/V rows) is allocated at the first call.
 *                        NB200_EINVAL, with nothing written (cache, logits, seen set, ids): n == 0 or n > M (the chunk size),
 *                        pos + n > min(max_seq_len, block_size), an id >= vocab_size in ids[pos .. pos+n) (and in ids[0..pos)
 *                        when repetition_penalty != 1), a tensor-parallel engine, an active LoRA plug-in.
 *   nb200_decode_lookup  nb200_decode_greedy's arguments and limits, with drafts looked up in the context itself (prompt lookup):
 *                        its ids are bit-identical to nb200_decode_greedy's on an engine with the same flags plus
 *                        NB200_FLAG_NO_STREAM.  Positions 0 .. n_prompt-2 run as prefill chunks.  Then at position p (ids[0..p]
 *                        known): for g = min(ngram_max, p) down to 1, take the largest s <= p-g with ids[s..s+g) ==
 *                        ids[p-g+1 .. p]; the draft is ids[s+g .. s+g+k) with k = min(draft_max, M-1, n_total-2-p,
 *                        min(max_seq_len, block_size)-1-p, p+1-(s+g)); the first g giving k >= 1 wins.  With a draft, one
 *                        nb200_verify_greedy of 1+k positions advances by a+1; without one, one multi-kernel token step (the
 *                        CUDA graph where the engine has one: launches as one token of that path) advances by 1.
 *                        stats (optional): [0] verify passes, [1] steps without a draft, [2] drafted ids, [3] accepted ids.
 *                        prefill_ms / device_ms (optional): CUDA-event time of the prompt and of the decode segment (which
 *                        includes the host's drafting between passes).  Refuses what nb200_verify_greedy refuses, and
 *                        ngram_max == 0 or draft_max == 0.
 * Not covered: sampled speculation (it cannot equal nb200_next_sampled's single coin), LoRA, tensor parallelism, non-causal
 * attention, the shim (llm_session_step is one token per call).  Batched verification: nb200_batch_verify_greedy below. */
int nb200_verify_greedy(nb200_engine *e, uint32_t *ids, uint32_t pos, uint32_t n, float repetition_penalty,
                        uint32_t *n_accepted, float *device_ms);
int nb200_decode_lookup(nb200_engine *e, uint32_t *ids, uint32_t n_prompt, uint32_t n_total, float repetition_penalty,
                        uint32_t ngram_max, uint32_t draft_max, uint32_t stats[4], float *prefill_ms, float *device_ms);

/* Batched multi-session decode (no reference counterpart).  A batch is attached to an engine and shares its weights; it holds
 * n_slots sessions ("slots"), each with its own K / V cache (laid out like the engine's and zeroed at creation, n_kv_head *
 * head_dim * max_seq_len * n_layer * 8 bytes), repetition-penalty seen set and logits row.  n_slots is not capped at the pass size.
 *   nb200_batch_prefill      nb200_prefill into one slot's cache.
 *   nb200_batch_next_greedy  entry i does what nb200_next_greedy(e, ids[i], pos[i], 0, repetition_penalty[i], &next_tokens[i])
 *                            does, in slot slots[i]: it consumes ids[i][pos[i]] at pos[i], ids[i][0..pos[i]) feed the penalty (a
 *                            rewind or a new session in a slot resets its seen set, as for the engine), and the slot's logits end
 *                            up as nb200_read_logits returns them after that call (penalised).  The entries run in passes of up
 *                            to M (info[0], at most 16) positions per pass over the weights.  device_ms (optional): CUDA-event
 *                            time of the call.
 *   nb200_batch_next_sampled entry i with temperature[i] > 0 does what nb200_next_sampled(e, ids[i], pos[i], repetition_penalty[i],
 *                            temperature[i], top_p[i], coin[i], &next_tokens[i], &top6[6 * i]) does, in slot slots[i]: the same
 *                            penalised logits row, sampled id and six observed ids, and the same empty-nucleus rule (the
 *                            first-max id, six zero ids).  An entry with temperature[i] == 0 is exactly nb200_batch_next_greedy's
 *                            entry, with six zero ids, so greedy and sampled sessions share passes.  top6 (n x 6) is optional.
 *                            Everything nb200_batch_next_greedy refuses is refused with the same message, and so is a negative or
 *                            NaN temperature; top_p and coin are not checked, as for nb200_next_sampled.  The sampler's
 *                            workspace is the batch's own, allocated at its first call with a sampled entry (a failed
 *                            allocation fails the call before anything is written) and freed by nb200_batch_destroy; the
 *                            engine's own sampler workspace is never used.  A sampled entry's result depends neither on the
 *                            other entries of the call nor on which of them sample.
 *   nb200_batch_verify_greedy entry i does in slot slots[i] exactly what nb200_verify_greedy(e, ids[i], pos[i], n_pos[i],
 *                            repetition_penalty[i], &n_accepted[i]) does on an engine created with the same flags plus
 *                            NB200_FLAG_NO_STREAM running that session alone: ids[i][pos[i]] is consumed, ids[i][pos[i]+1 ..
 *                            pos[i]+n_pos[i]) are the drafts, n_accepted[i] = a is the largest count whose greedy ids g_j (j < a)
 *                            all match their drafts, and ids[i][pos[i]+a+1] receives g_a (ids[i] needs pos[i]+n_pos[i]+1 entries).
 *                            Afterwards the slot is where nb200_batch_next_greedy at pos .. pos+a leaves it: K/V rows pos .. pos+a
 *                            written, rows from pos+a+1 on as they were before the call, the slot's logits the penalised row at
 *                            pos+a, its seen set at ids[0..pos).  An entry with n_pos[i] == 1 is exactly nb200_batch_next_greedy's
 *                            entry.  Packing: the entries run in call order in passes of at most M rows (info[0]); an entry is
 *                            never split across passes, and a new pass starts when the next entry's n_pos does not fit in the
 *                            rows left.  A row's value depends neither on the packing nor on the other entries, so the packing
 *                            changes only the speed.  Acceptance and the restore of the rows past the accepted ones run on the
 *                            device: one host synchronise per call, at the end.  Launches per pass: 1 + 6 * n_layer (the chunk,
 *                            with a K-row pass per layer), + 3 (classifier, argmax, accept), + 1 when an entry of the pass drafts
 *                            (n_pos > 1: the save of the rows it overwrites), + 1 when an entry of the pass has repetition_penalty
 *                            != 1 (its seen rows); plus, per call, nb200_batch_next_greedy's seen-set update of each penalised slot
 *                            whose ids[0..pos) has new ids.  The workspace (M logits rows, M seen rows, K/V save rows for M-1 rows,
 *                            the per-entry results) is the batch's own, allocated at its first call (a failed allocation fails the
 *                            call before anything is written) and freed by nb200_batch_destroy.  device_ms (optional): CUDA-event
 *                            time of the call.  NB200_EINVAL, with nothing written (every slot's cache, logits and seen set, every
 *                            ids array): everything nb200_batch_next_greedy refuses, with the same messages; n_pos[i] == 0 or
 *                            n_pos[i] > M; pos[i] + n_pos[i] > min(max_seq_len, block_size); an id >= vocab_size in ids[i][pos ..
 *                            pos+n_pos) (and in ids[i][0..pos) when repetition_penalty[i] != 1).
 *   nb200_batch_read_logits / nb200_batch_read_kv  a slot's logits row, and its K / V cache rows as nb200_read_buffer gives them.
 *   nb200_batch_info         [0] M, [1] n_slots, [2] the attention kernel (encoded as nb200_config.reserved[4]), [3] 0.
 * A batch always runs the multi-kernel path's arithmetic, and a row's value depends neither on the other entries of its pass nor
 * on how many there are: each slot's ids, logits and K / V rows are bit-identical to those of an engine created with the same
 * flags plus NB200_FLAG_NO_STREAM running that session alone (nb200_prefill + nb200_next_greedy / nb200_next_sampled) -- also when the batch's own
 * engine runs the streaming kernel -- and in exact mode to the strict reference.  The engine's own cache, logits, seen set,
 * results and nb200_config.reserved[3..6] are not changed by a batch; its calls share the engine's stream.
 * NB200_EINVAL, with nothing written: a tensor-parallel engine or an active LoRA plug-in (checked at every call), n_slots == 0,
 * n == 0, a slot >= n_slots or the same slot twice in one call, a position >= min(max_seq_len, block_size), an id >= vocab_size.
 * Destroy every batch before its engine.  Not covered: non-causal attention, LoRA, tensor parallelism. */
typedef struct nb200_batch nb200_batch;
int nb200_batch_create(nb200_engine *e, uint32_t n_slots, nb200_batch **out);
void nb200_batch_destroy(nb200_batch *b);
int nb200_batch_prefill(nb200_batch *b, uint32_t slot, const uint32_t *ids, uint32_t pos0, uint32_t n, float *device_ms);
int nb200_batch_next_greedy(nb200_batch *b, uint32_t n, const uint32_t *slots, const uint32_t *const *ids, const uint32_t *pos,
                            const float *repetition_penalty, uint32_t *next_tokens, float *device_ms);
int nb200_batch_next_sampled(nb200_batch *b, uint32_t n, const uint32_t *slots, const uint32_t *const *ids, const uint32_t *pos,
                             const float *repetition_penalty, const float *temperature, const float *top_p, const float *coin,
                             uint32_t *next_tokens, uint32_t *top6 /* n x 6, optional */, float *device_ms);
int nb200_batch_verify_greedy(nb200_batch *b, uint32_t n, const uint32_t *slots, uint32_t *const *ids, const uint32_t *pos,
                              const uint32_t *n_pos, const float *repetition_penalty, uint32_t *n_accepted, float *device_ms);
int nb200_batch_read_logits(nb200_batch *b, uint32_t slot, float *host_logits);
int nb200_batch_read_kv(nb200_batch *b, uint32_t slot, int field /* NB200_F_KROW | NB200_F_VROW */, uint32_t layer, uint32_t pos,
                        float *dst, uint32_t count);
int nb200_batch_info(const nb200_batch *b, uint32_t info[4]);

/* introspection for parity tests */
int nb200_read_buffer(nb200_engine *e, int field, uint32_t layer, uint32_t pos, float *dst, uint32_t count);
int nb200_write_x(nb200_engine *e, const float *x, uint32_t count);
/* run exactly one transformer block on the current x at (layer,pos): layer-level parity with
 * oracle-injected inputs (SURVEY 8d check 2). */
int nb200_run_layer(nb200_engine *e, uint32_t layer, uint32_t pos, uint32_t is_causal);
/* per-kernel-class device time (CUDA events around every launch, graph and PDL off): class ids
 * 0 embed, 1 qkv, 2 attention, 3 o-proj, 4 w1|w3, 5 w2, 6 classifier. Used by bench.py's roofline. */
int nb200_profile_tokens(nb200_engine *e, const uint32_t *ids, uint32_t start, uint32_t n, float ms[7], uint32_t counts[7]);
/* debug: clock64() stamps of CTA 0 after every grid barrier of one token in the persistent kernel */
int nb200_read_attn_trace(nb200_engine *e, unsigned long long *stamps32);   /* debug, NB200_ATTN_DBG=1 */
int nb200_trace_token(nb200_engine *e, uint32_t token, uint32_t pos, unsigned long long *stamps, uint32_t cap, uint32_t *count);
uint64_t nb200_kernel_launches(const nb200_engine *e);      /* cumulative kernel launches issued */
uint32_t nb200_launches_per_token(const nb200_engine *e);
uint64_t nb200_weight_bytes(const nb200_engine *e);         /* bytes resident in HBM for weights */

/* ---- op-level entry points (host pointers; each runs the same device code the engine uses) ---- */
int nb200_op_rmsnorm(float *out, const float *x, const float *gain, uint32_t n, uint32_t exact);
int nb200_op_q80_quantize(int8_t *codes, float *scales, const float *x, uint32_t n, uint32_t gs);
/* w_codes [d*n] int8, w_scales [d*n/gs] (file layout, tensor.c:49-62) */
int nb200_op_q80_matvec(float *out, const float *x, const int8_t *w_codes, const float *w_scales,
                        uint32_t n, uint32_t d, uint32_t gs);
int nb200_op_f32_matvec(float *out, const float *x, const float *w, uint32_t n, uint32_t d, uint32_t exact);
/* blocks: 160-byte Q4K blocks in file layout (tensor.h:96-105) */
int nb200_op_q4k_quantize(uint8_t *blocks, const float *x, uint32_t n);
int nb200_op_q4k_matvec(float *out, const float *x, const uint8_t *w_blocks, uint32_t n, uint32_t d);
/* whole-tensor forms on the reference's 160-byte block layout (tensor.h:96-114):
 *   nb200_op_q4k_quantize_blocks <- quantize_tensor_q4k_in_situ  infer/tensor.c:281-310 (rows % 256 == 0)
 *   nb200_op_q4k_matvec_blocks   <- matmul_q4k                   infer/tensor.c:438-471 (x already quantised) */
int nb200_op_q4k_quantize_blocks(uint8_t *blocks, const float *x, uint64_t nblocks);
int nb200_op_q4k_matvec_blocks(float *out, const uint8_t *x_blocks, const uint8_t *w_blocks, uint32_t n, uint32_t d);

#ifdef __cplusplus
}
#endif
#endif /* NANO_B200_H */
