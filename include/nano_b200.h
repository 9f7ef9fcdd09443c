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
    uint32_t reserved[7];   /* [0] execution path: 4 streaming kernel, 1 CUDA graph, 0 direct launches; [1], [2] creation-time calibration:
                               us per token of the streaming kernel / of the multi-kernel graph (0 = the choice was not measured);
                               multi-kernel path, recorded when a kernel is launched or captured into the graph:
                               [3] matvec variants used since creation, bit 3 * epilogue + {0: RB 1, 1: RB 2, 2: RB 4} with the
                                   epilogues store 0, qkv 1, residual 2, swiglu 3, classifier 4 (the exact-mode F32 kernel sets none);
                               [4] attention kernel of the last layer run: 0 none yet, 1 exact, 2 generic split-KV,
                                   3 | kv_mul << 8 the split-KV kernel specialised for that kv_mul */
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
