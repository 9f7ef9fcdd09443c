/*
 * oracle/ref_harness.c -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * Thin shim compiled TOGETHER WITH the unmodified reference sources
 * (/root/reference/infer/{infer,tensor,tokenizer,utils,hal_*_linux}.c, see oracle/Makefile)
 * into oracle/_ref/libnano_ref_<flavour>.so.  It adds nothing to the arithmetic; it only
 *   - installs a no-op observation hook (the reference calls ctx->observation unconditionally,
 *     infer.c:756 ff., and calloc's the context, infer.c:553, so stock binaries crash);
 *   - lets a test copy FwdBuffer fields at a chosen (layer, phase) hook (infer.h:65-76 phases);
 *   - exposes the embedded sort model (main_sort.c:6) which is the reference's only golden fixture;
 *   - exposes llm_forward (infer.c:971, non-static but un-headered), with or without the loaded LoRA plug-in;
 *   - records the six ids of the last sampling observation (orh_last_sample).
 * Everything else (quantize, matmul_quant, matmul_q4k, rmsnorm, ...) is called straight through
 * ctypes on the reference's own non-static symbols.
 */
#include <stdint.h>
#include <string.h>
#include "infer.h"

float *llm_forward(Nano_Context *ctx, uint32_t token, uint32_t pos, uint32_t max_seq_len,
                   uint32_t is_causal, LLM *llm, LoRA *lora);

/* ---- pull in the embedded fixture without its main() ---- */
#define main orh_unused_sort_main
#include "main_sort.c"
#undef main

enum { ORH_MAX_PROBES = 64 };
typedef struct {
    int32_t layer, phase, field;
    float *dst;
    uint32_t count;
    uint32_t hits;
} OrhProbe;

static OrhProbe g_probes[ORH_MAX_PROBES];
static int g_nprobes = 0;

static float *orh_field(Nano_Context *ctx, int field) {
    FwdBuffer *s = &ctx->llm->state;
    switch (field) {
        case 0: return s->x;
        case 1: return s->xb;
        case 2: return s->xba;
        case 3: return s->xb2;
        case 4: return s->hb;
        case 5: return s->hb2;
        case 6: return s->q;
        case 7: return s->k;
        case 8: return s->v;
        case 9: return s->logits;
        case 10: return s->k_cache;
        case 11: return s->v_cache;
        case 12: return s->att;
        default: return NULL;
    }
}

static uint32_t g_last_sample[6];

static void orh_hook(Nano_Observation obs, void *env) {
    Nano_Context *ctx = (Nano_Context *)env;
    if (obs.layer == -1 && obs.phase == NANO_LLM_PHASE_SAMPLE) {      /* sample_top_p's six ids (infer.c:1086-1095) */
        g_last_sample[0] = obs.token_0; g_last_sample[1] = obs.token_1; g_last_sample[2] = obs.token_2;
        g_last_sample[3] = obs.token_3; g_last_sample[4] = obs.token_4; g_last_sample[5] = obs.token_5;
    }
    for (int i = 0; i < g_nprobes; i++) {
        OrhProbe *p = &g_probes[i];
        if (p->layer == obs.layer && p->phase == obs.phase) {
            float *src = orh_field(ctx, p->field);
            if (src && p->dst) memcpy(p->dst, src, (size_t)p->count * sizeof(float));
            p->hits++;
        }
    }
}

static void orh_install(Nano_Context *ctx) {
    ctx->observation = orh_hook;
    ctx->observation_env = ctx;
}

Nano_Context *orh_open_file(const char *path, uint32_t max_seq_len, float penalty, float temperature,
                            float top_p, uint32_t top_k, uint64_t seed) {
    Nano_Context *ctx = llm_context_init((char *)path, NULL, max_seq_len, penalty, temperature, top_p, top_k, seed);
    orh_install(ctx);
    return ctx;
}

Nano_Context *orh_open_buffer(uint8_t *buffer, uint32_t max_seq_len, float penalty, float temperature,
                              float top_p, uint32_t top_k, uint64_t seed) {
    Nano_Context *ctx = llm_context_init_from_buffer(buffer, max_seq_len, penalty, temperature, top_p, top_k, seed);
    orh_install(ctx);
    return ctx;
}

/* NOTE: llm_context_free on a *_from_buffer context munmap()s/free()s memory it does not own
 * (infer.c:372-378); tests simply leak buffer contexts. */
void orh_close_file(Nano_Context *ctx) { llm_context_free(ctx); }

/* LoRA plug-in (infer.c:408-545): the caller keeps `buffer` alive; ctx->lora makes llm_forward / generate_next_token take
 * the low-rank branches (infer.c:792-808, 898-903). */
void orh_load_lora(Nano_Context *ctx, uint8_t *buffer) {
    ctx->lora = load_lora_from_buffer(ctx->llm, buffer);
}

float *orh_forward(Nano_Context *ctx, uint32_t token, uint32_t pos, uint32_t is_causal) {
    return llm_forward(ctx, token, pos, ctx->max_seq_len, is_causal, ctx->llm, ctx->lora);
}

/* the plug-in per call, as the reference's own callers pass it (seq2seq passes NULL while ctx->lora is set, infer.c:1365-1402) */
float *orh_forward_lora(Nano_Context *ctx, uint32_t token, uint32_t pos, uint32_t is_causal, int use_lora) {
    return llm_forward(ctx, token, pos, ctx->max_seq_len, is_causal, ctx->llm, use_lora ? ctx->lora : NULL);
}

uint32_t orh_next(Nano_Context *ctx, uint32_t *ids, uint32_t pos, int is_prefilling) {
    return generate_next_token(ctx, ids, pos, is_prefilling);
}

void orh_config(Nano_Context *ctx, uint32_t out[16]) {
    LLM *m = ctx->llm;
    out[0] = m->config.block_size; out[1] = m->config.vocab_size; out[2] = m->config.n_layer;
    out[3] = m->config.n_embd; out[4] = m->config.n_head; out[5] = m->config.n_kv_head;
    out[6] = m->config.n_hidden; out[7] = m->config.is_shared_classifier; out[8] = m->config.head_dim;
    out[9] = m->arch; out[10] = m->quant_type; out[11] = m->group_size; out[12] = ctx->max_seq_len;
}

float *orh_state(Nano_Context *ctx, int field) { return orh_field(ctx, field); }

void orh_probe_clear(void) { g_nprobes = 0; }

int orh_probe_add(int32_t layer, int32_t phase, int32_t field, float *dst, uint32_t count) {
    if (g_nprobes >= ORH_MAX_PROBES) return -1;
    g_probes[g_nprobes] = (OrhProbe){layer, phase, field, dst, count, 0};
    return g_nprobes++;
}

/* token_0..5 of the last (layer -1, SAMPLE) observation */
void orh_last_sample(uint32_t out[6]) { memcpy(out, g_last_sample, sizeof g_last_sample); }

uint32_t orh_probe_hits(int idx) { return (idx >= 0 && idx < g_nprobes) ? g_probes[idx].hits : 0; }

const uint8_t *orh_sort_model(uint32_t *len) {
    *len = (uint32_t)sizeof(SORT_6_MODEL);
    return SORT_6_MODEL;
}

/* layout report used by tests/test_boundary.py to pin include/nano_infer_abi.h */
#include <stddef.h>
#define ORH_OFF(T, f) out[n++] = (uint32_t)offsetof(T, f)
uint32_t orh_abi_layout(uint32_t *out, uint32_t cap) {
    uint32_t n = 0;
    if (cap < 64) return 0;
    out[n++] = sizeof(LLM_Config); out[n++] = sizeof(LLM_Param); out[n++] = sizeof(FwdBuffer);
    out[n++] = sizeof(LLM); out[n++] = sizeof(Sampler); out[n++] = sizeof(Nano_Context);
    out[n++] = sizeof(Nano_Session); out[n++] = sizeof(Tokenizer); out[n++] = sizeof(Typed_Tensor);
    out[n++] = sizeof(LoRA); out[n++] = sizeof(Nano_Observation);
    ORH_OFF(LLM, config); ORH_OFF(LLM, params); ORH_OFF(LLM, state); ORH_OFF(LLM, arch);
    ORH_OFF(LLM, quant_type); ORH_OFF(LLM, group_size); ORH_OFF(LLM, fd); ORH_OFF(LLM, buffer);
    ORH_OFF(LLM, file_size);
    ORH_OFF(FwdBuffer, x); ORH_OFF(FwdBuffer, xq); ORH_OFF(FwdBuffer, q); ORH_OFF(FwdBuffer, logits);
    ORH_OFF(FwdBuffer, q0);
    ORH_OFF(LLM_Param, token_embedding); ORH_OFF(LLM_Param, wq); ORH_OFF(LLM_Param, q_norm);
    ORH_OFF(LLM_Param, freq_cis_real); ORH_OFF(LLM_Param, token_classifier);
    ORH_OFF(Sampler, probindex); ORH_OFF(Sampler, repetition_penalty); ORH_OFF(Sampler, temperature);
    ORH_OFF(Sampler, top_p); ORH_OFF(Sampler, top_k); ORH_OFF(Sampler, rng_state);
    ORH_OFF(Nano_Context, llm); ORH_OFF(Nano_Context, lora); ORH_OFF(Nano_Context, tokenizer);
    ORH_OFF(Nano_Context, sampler); ORH_OFF(Nano_Context, max_seq_len); ORH_OFF(Nano_Context, random_seed);
    ORH_OFF(Nano_Context, observation); ORH_OFF(Nano_Context, observation_env);
    ORH_OFF(Nano_Session, prompt); ORH_OFF(Nano_Session, num_prompt_tokens); ORH_OFF(Nano_Session, max_seq_len);
    ORH_OFF(Nano_Session, output_ids); ORH_OFF(Nano_Session, output_count); ORH_OFF(Nano_Session, output_text);
    ORH_OFF(Nano_Session, next_token); ORH_OFF(Nano_Session, pos); ORH_OFF(Nano_Session, is_prefilling);
    ORH_OFF(Nano_Session, t_0); ORH_OFF(Nano_Session, t_1); ORH_OFF(Nano_Session, tps);
    ORH_OFF(Tokenizer, vocab_size); ORH_OFF(Tokenizer, unicode_charset); ORH_OFF(Tokenizer, token_list);
    ORH_OFF(Tokenizer, vocab_trie); ORH_OFF(Tokenizer, unicode_to_id_map); ORH_OFF(Tokenizer, token_to_id_map);
    ORH_OFF(Tokenizer, vocab); ORH_OFF(Tokenizer, vocab_scores); ORH_OFF(Tokenizer, sorted_vocab);
    ORH_OFF(Tokenizer, max_token_length); ORH_OFF(Tokenizer, byte_pieces);
    return n;
}
