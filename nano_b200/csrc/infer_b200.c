/*
 * infer_b200.c -- the reference's host API (infer/infer.h, parts of infer/tensor.h) implemented over the
 * B200 engine's C-ABI (include/nano_b200.h).  Builds libnano_infer_b200.so, which replaces `tensor.c infer.c`
 * in the reference's link line (infer/Makefile:145-147):
 *
 *     gcc -DNANO_CLI ... main_cli.c hal_*_linux.c utils.c tokenizer.c  -lnano_infer_b200 -lnano_b200
 *
 * Host code stays C and keeps the reference's semantics (same names, argument meaning, status codes and
 * exit(EXIT_FAILURE) error convention); everything on the per-token path is one call into the CUDA engine.
 * The tokenizer, maps/tries, platform_calloc and the xorshift RNG are the reference's own objects, resolved
 * at link time exactly as before (SURVEY 8b).
 *
 * Deliberate differences (supersets of the reference's behaviour):
 *   - ctx->observation may be NULL (the reference dereferences it unconditionally: infer.c:756 ff.);
 *   - with a hook installed, the per-phase notifications of one token fire in the reference's order BEFORE the
 *     token's single device launch (the GUI only draws a layer diagram from them, ui_llm.c:695-705);
 *   - LoRA plug-ins are uploaded to the GPU at load time (the reference keeps pointers into the caller's buffer);
 *     free_lora releases the device copy and the struct instead of free()ing interior pointers (infer.c:521-534).
 */
#define _GNU_SOURCE
#include <fcntl.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include "nano_b200.h"
#include "nano_infer_abi.h"

#define QWEN_TOKENIZER_ENTRIES 151669          /* infer.c:313 */
#define UNKNOWN_IMAGE_BYTES (1ull << 40)       /* *_from_buffer callers pass no length (infer.h:253) */

static nb200_engine *engine_of(LLM *llm) { return (nb200_engine *)(void *)llm->state.xbuf; }

static void die(const char *what) {
    fprintf(stderr, "nano_b200: %s: %s\n", what, nb200_last_error());
    exit(EXIT_FAILURE);
}

static void notify(Nano_Context *ctx, int32_t layer, int32_t phase) {
    if (ctx && ctx->observation) {
        Nano_Observation o;
        memset(&o, 0, sizeof o);
        o.layer = layer; o.phase = phase;
        ctx->observation(o, ctx->observation_env);
    }
}

/* the notification sequence of one llm_forward (infer.c:756-1003) */
static void notify_forward(Nano_Context *ctx) {
    if (!ctx || !ctx->observation) return;
    const int32_t L = (int32_t)ctx->llm->config.n_layer;
    notify(ctx, -1, NANO_PH_EMBEDDING);
    for (int32_t l = 0; l < L; l++)
        for (int32_t ph = NANO_PH_ATTN_NORM; ph <= NANO_PH_W2; ph++) notify(ctx, l, ph);
    notify(ctx, L, NANO_PH_FINAL_NORM);
    notify(ctx, L, NANO_PH_CLASSIFY);
}

/* ------------------------------------------------------------------------------------------------------ */
/* loading (infer.c:220-346)                                                                               */
/* ------------------------------------------------------------------------------------------------------ */
static uint32_t rd32(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }

/* Nano tokenizer section -> Tokenizer (infer.c:263-307); records are {u8 len,u8 special,u16 0}{u32 id}{u32 cp x len} */
static void build_nano_tokenizer(Tokenizer *tk, const uint8_t *sec) {
    const uint32_t field_bytes = rd32(sec);
    const uint8_t *p = sec + 4;
    tk->vocab_size = rd32(p); p += 4;
    tk->token_list = (wchar_t **)platform_calloc(tk->vocab_size, sizeof(wchar_t *));
    tk->unicode_charset = (wchar_t *)platform_calloc(tk->vocab_size, sizeof(wchar_t));
    tk->unicode_to_id_map = new_map(tk->vocab_size);
    tk->token_to_id_map = new_map(tk->vocab_size);
    tk->vocab_trie = new_trie(tk->vocab_size, 0);
    const uint8_t *end = sec + field_bytes;
    uint32_t nchars = 0;
    while (p < end) {
        const uint32_t hdr = rd32(p), id = rd32(p + 4);
        const uint32_t len = hdr & 0xffu;
        p += 8;
        wchar_t *tok = (wchar_t *)platform_calloc(len + 1, sizeof(wchar_t));
        for (uint32_t i = 0; i < len; i++) tok[i] = (wchar_t)rd32(p + 4 * i);
        if (len == 1) {
            tk->unicode_charset[nchars++] = tok[0];
            map_set(tk->unicode_to_id_map, (uint32_t)tok[0], id);
        }
        p += 4 * (size_t)len;
        if (id < tk->vocab_size) tk->token_list[id] = tok;
    }
    for (uint32_t i = 0; i < tk->vocab_size; i++) {
        wchar_t *t = tk->token_list[i];
        const uint32_t len = t ? (uint32_t)wcslen(t) : 0;
        if (len > 1) {
            uint32_t *ids = string_to_ids(tk->unicode_to_id_map, t);
            add_token(tk->vocab_trie, ids, len, i);
            free(ids);
        }
    }
}

static void load_image(LLM *llm, Tokenizer *tk, uint8_t *image, uint64_t image_bytes, uint32_t max_seq_len) {
    nb200_engine *e = NULL;
    if (nb200_engine_create(&e, image, image_bytes, max_seq_len, 0, 0) != NB200_OK) die("load_llm");
    nb200_config c;
    nb200_get_config(e, &c);
    llm->config.block_size = c.block_size; llm->config.vocab_size = c.vocab_size; llm->config.n_layer = c.n_layer;
    llm->config.n_embd = c.n_embd; llm->config.n_head = c.n_head; llm->config.n_kv_head = c.n_kv_head;
    llm->config.n_hidden = c.n_hidden; llm->config.is_shared_classifier = rd32(image + 52);
    llm->config.head_dim = rd32(image + 56);
    llm->arch = c.arch; llm->quant_type = c.quant; llm->group_size = rd32(image + 64);
    memset(&llm->params, 0, sizeof llm->params);
    memset(&llm->state, 0, sizeof llm->state);
    llm->state.xbuf = (float *)(void *)e;                                   /* engine handle (private area) */
    llm->state.logits = (float *)platform_calloc(c.vocab_size, sizeof(float)); /* host logits, like the reference */
    const uint8_t *tok = image + 256;
    if (llm->arch == NANO_ARCH_NANO) build_nano_tokenizer(tk, tok);
    else build_bpe_tokenizer(tk, (uint8_t *)tok, QWEN_TOKENIZER_ENTRIES);
}

void load_llm_from_buffer(LLM *llm, Tokenizer *tk, uint8_t *buffer, uint32_t max_seq_len) {
    llm->fd = -1; llm->buffer = NULL; llm->file_size = 0;     /* caller owns the bytes; the engine copied what it needs */
    load_image(llm, tk, buffer, UNKNOWN_IMAGE_BYTES, max_seq_len);
}

void load_llm(LLM *llm, Tokenizer *tk, char *model_path, uint32_t max_seq_len) {
    int fd = open(model_path, O_RDONLY);
    if (fd == -1) { fprintf(stderr, "Couldn't open file %s\n", model_path); exit(EXIT_FAILURE); }
    struct stat sb;
    if (fstat(fd, &sb) != 0) { fprintf(stderr, "stat failed!\n"); exit(EXIT_FAILURE); }
    uint8_t *image = (uint8_t *)mmap(NULL, (size_t)sb.st_size, PROT_READ, MAP_PRIVATE, fd, 0);
    if (image == MAP_FAILED) { fprintf(stderr, "mmap failed!\n"); exit(EXIT_FAILURE); }
    llm->fd = fd; llm->buffer = image; llm->file_size = (size_t)sb.st_size;
    load_image(llm, tk, image, (uint64_t)sb.st_size, max_seq_len);
}

void free_llm(LLM *llm, Tokenizer *tk) {
    if (llm->buffer && llm->file_size) munmap(llm->buffer, llm->file_size);
    if (llm->fd > 0) close(llm->fd);
    if (llm->arch == NANO_ARCH_NANO) free_tokenizer(tk); else free_bpe_tokenizer(tk);
    nb200_engine_destroy(engine_of(llm));
    free(llm->state.logits);
    free(llm);
}

/* infer.c:436-519: the factors are uploaded to HBM; the LoRA struct keeps the reference's host view (config + pointers into
 * the caller's buffer) for hosts that inspect it. */
static LoRA *lora_from_image(LLM *llm, uint8_t *buffer, uint64_t bytes) {
    if (!buffer) die("load_lora: null buffer");
    if (nb200_lora_load(engine_of(llm), buffer, bytes) != NB200_OK) die("load_lora");
    LoRA *p = (LoRA *)platform_calloc(1, sizeof(LoRA));
    p->data = (float *)(void *)buffer;
    memcpy(&p->config, buffer + 24, sizeof(LoRA_Config));        /* rank, alpha, n_layer, n_embd, n_head, n_kv_head, n_hidden, lora_config */
    const uint64_t L = llm->config.n_layer, E = llm->config.n_embd, r = p->config.lora_rank;
    const uint64_t kv = (E / llm->config.n_head) * llm->config.n_kv_head;
    float *f = (float *)(void *)(buffer + 256);
    p->params.wq_lora_a = f; f += L * r * E;  p->params.wq_lora_b = f; f += L * E * r;
    p->params.wk_lora_a = f; f += L * r * E;  p->params.wk_lora_b = f; f += L * kv * r;
    p->params.wv_lora_a = f; f += L * r * E;  p->params.wv_lora_b = f; f += L * kv * r;
    p->params.wo_lora_a = f; f += L * r * E;  p->params.wo_lora_b = f;
    return p;
}
/* file buffers that load_lora() allocated itself (the LoRA struct is ABI-fixed and has no room for an ownership flag) */
static struct { LoRA *lora; void *buf; } g_lora_owned[8];
LoRA *load_lora_from_buffer(LLM *llm, uint8_t *buffer) { return lora_from_image(llm, buffer, 0); }
LoRA *load_lora(LLM *llm, char *lora_path) {
    FILE *fp = fopen(lora_path, "rb");
    if (!fp) { fprintf(stderr, "Couldn't open LoRA module file %s\n", lora_path); exit(EXIT_FAILURE); }
    fseek(fp, 0, SEEK_END);
    const uint64_t n = (uint64_t)ftell(fp);
    rewind(fp);
    uint8_t *buf = (uint8_t *)platform_calloc(n + 1, 1);
    if (!buf) die("load_lora: allocation failed");
    if (fread(buf, 1, n, fp) != n) { fclose(fp); exit(EXIT_FAILURE); }
    fclose(fp);
    LoRA *p = lora_from_image(llm, buf, n);
    for (int i = 0; i < 8; i++) if (!g_lora_owned[i].lora) { g_lora_owned[i].lora = p; g_lora_owned[i].buf = buf; break; }
    return p;
}
/* infer.c:521-534 frees interior pointers of a single allocation (undefined behaviour); here: drop the device copy and the struct */
void free_lora(LLM *llm, LoRA *lora) {
    if (llm) nb200_lora_unload(engine_of(llm));
    for (int i = 0; i < 8; i++) if (lora && g_lora_owned[i].lora == lora) { free(g_lora_owned[i].buf); g_lora_owned[i].lora = NULL; g_lora_owned[i].buf = NULL; }
    free(lora);
}

/* ------------------------------------------------------------------------------------------------------ */
/* context / sampler (infer.c:548-581, 1111-1127)                                                          */
/* ------------------------------------------------------------------------------------------------------ */
Sampler *build_sampler(int vocab_size, float repetition_penalty, float temperature, float top_p, uint32_t top_k, uint64_t rng_seed) {
    Sampler *s = (Sampler *)platform_calloc(1, sizeof(Sampler));
    s->vocab_size = vocab_size; s->repetition_penalty = repetition_penalty; s->temperature = temperature;
    s->top_p = top_p; s->top_k = top_k; s->rng_state = rng_seed;
    s->probindex = (ProbIndex *)platform_calloc((size_t)vocab_size, sizeof(ProbIndex));
    return s;
}

void free_sampler(Sampler *s) { if (s) { free(s->probindex); free(s); } }

static Nano_Context *new_context(uint32_t max_seq_len, uint64_t seed) {
    Nano_Context *ctx = (Nano_Context *)platform_calloc(1, sizeof(Nano_Context));
    ctx->max_seq_len = max_seq_len; ctx->random_seed = seed;
    ctx->llm = (LLM *)platform_calloc(1, sizeof(LLM));
    ctx->tokenizer = (Tokenizer *)platform_calloc(1, sizeof(Tokenizer));
    return ctx;
}

Nano_Context *llm_context_init_from_buffer(uint8_t *buffer, uint32_t max_seq_len, float repetition_penalty, float temperature,
                                           float top_p, uint32_t top_k, uint64_t random_seed) {
    Nano_Context *ctx = new_context(max_seq_len, random_seed);
    load_llm_from_buffer(ctx->llm, ctx->tokenizer, buffer, max_seq_len);
    ctx->sampler = build_sampler((int)ctx->llm->config.vocab_size, repetition_penalty, temperature, top_p, top_k, random_seed);
    return ctx;
}

Nano_Context *llm_context_init(char *model_path, char *lora_path, uint32_t max_seq_len, float repetition_penalty,
                               float temperature, float top_p, uint32_t top_k, uint64_t random_seed) {
    Nano_Context *ctx = new_context(max_seq_len, random_seed);
    load_llm(ctx->llm, ctx->tokenizer, model_path, max_seq_len);
    ctx->sampler = build_sampler((int)ctx->llm->config.vocab_size, repetition_penalty, temperature, top_p, top_k, random_seed);
    ctx->lora = lora_path ? load_lora(ctx->llm, lora_path) : NULL;
    return ctx;
}

void llm_context_free(Nano_Context *ctx) {
    if (!ctx) return;
    free_llm(ctx->llm, ctx->tokenizer);
    free(ctx->tokenizer);
    free_sampler(ctx->sampler);
    free(ctx);
}

/* ------------------------------------------------------------------------------------------------------ */
/* one token (infer.c:971-1018, 1135-1193)                                                                 */
/* ------------------------------------------------------------------------------------------------------ */
float *llm_forward(Nano_Context *ctx, uint32_t token, uint32_t pos, uint32_t max_seq_len, uint32_t is_causal, LLM *llm, LoRA *lora) {
    (void)max_seq_len;
    notify_forward(ctx);
    nb200_engine *e = engine_of(llm);
    if (nb200_lora_enable(e, lora != NULL) != NB200_OK) die("llm_forward (use_lora)");
    if (nb200_forward(e, token, pos, is_causal) != NB200_OK) die("llm_forward");
    if (nb200_read_logits(e, llm->state.logits) != NB200_OK) die("llm_forward (logits)");
    return llm->state.logits;
}

static int by_prob_desc(const void *a, const void *b) {          /* infer.c:1053-1059 */
    const ProbIndex *x = (const ProbIndex *)a, *y = (const ProbIndex *)b;
    if (x->prob > y->prob) return -1;
    if (x->prob < y->prob) return 1;
    return 0;
}

static void softmax_inplace(float *v, int n) {                    /* infer.c:616-634 */
    float top = v[0];
    for (int i = 1; i < n; i++) if (v[i] > top) top = v[i];
    float total = 0.0f;
    for (int i = 0; i < n; i++) { v[i] = expf(v[i] - top); total += v[i]; }
    for (int i = 0; i < n; i++) v[i] /= total;
}

/* nucleus sampling, infer.c:1062-1109 */
static int sample_nucleus(Nano_Context *ctx, float *prob, int n, float top_p, ProbIndex *pi, float coin) {
    const float cutoff = (1.0f - top_p) / (n - 1);
    int m = 0;
    for (int i = 0; i < n; i++) if (prob[i] >= cutoff) { pi[m].index = i; pi[m].prob = prob[i]; m++; }
    qsort(pi, (size_t)m, sizeof(ProbIndex), by_prob_desc);
    float cum = 0.0f;
    int last = m - 1;
    for (int i = 0; i < m; i++) { cum += pi[i].prob; if (cum > top_p) { last = i; break; } }
    if (ctx && ctx->observation) {
        Nano_Observation o;
        memset(&o, 0, sizeof o);
        o.layer = -1; o.phase = NANO_PH_SAMPLE;
        uint32_t *t = &o.token_0;
        for (int i = 0; i < 6; i++) t[i] = (m > i) ? (uint32_t)pi[i].index : 0u;
        ctx->observation(o, ctx->observation_env);
    }
    if (m == 0) {               /* no candidate (the reference reads pi[-1]): first-max argmax, as the device sampler does */
        int best = 0;
        for (int i = 1; i < n; i++) if (prob[i] > prob[best]) best = i;
        return best;
    }
    const float r = coin * cum;
    float cdf = 0.0f;
    for (int i = 0; i <= last; i++) { cdf += pi[i].prob; if (r < cdf) return pi[i].index; }
    return pi[last].index;
}

uint32_t generate_next_token(Nano_Context *ctx, uint32_t *output_ids, uint32_t pos, int is_prefilling) {
    LLM *llm = ctx->llm;
    Sampler *sp = ctx->sampler;
    nb200_engine *e = engine_of(llm);
    if (is_prefilling == 1 || sp->temperature == 0.0f) {
        /* whole step on the device: forward + penalty over ids[0..pos) + first-max argmax; 4 bytes come back */
        notify_forward(ctx);
        if (is_prefilling != 1) notify(ctx, -1, NANO_PH_SAMPLE);
        uint32_t next = 0;
        if (nb200_lora_enable(e, ctx->lora != NULL) != NB200_OK) die("generate_next_token (use_lora)");
        if (nb200_next_greedy(e, output_ids, pos, is_prefilling == 1, sp->repetition_penalty, &next) != NB200_OK) die("generate_next_token");
        return next;
    }
    /* temperature > 0 (infer.c:1156-1189): penalty, temperature, softmax, cutoff, ordered top-p all on the device; the coin is the
     * Sampler's own xorshift draw; 32 bytes come back.  NB200_HOST_SAMPLER=1 keeps the host restatement (logits D2H) for comparison. */
    const char *hs = getenv("NB200_HOST_SAMPLER");
    const int host_sampler = (hs && atoi(hs) != 0) ? 1 : 0;
    if (!host_sampler) {
        notify_forward(ctx);
        if (nb200_lora_enable(e, ctx->lora != NULL) != NB200_OK) die("generate_next_token (use_lora)");
        const float coin = random_f32(&sp->rng_state);
        uint32_t next = 0, top6[6];
        if (nb200_next_sampled(e, output_ids, pos, sp->repetition_penalty, sp->temperature, sp->top_p, coin, &next, top6) != NB200_OK) die("generate_next_token (sampling)");
        if (ctx->observation) {
            Nano_Observation o;
            memset(&o, 0, sizeof o);
            o.layer = -1; o.phase = NANO_PH_SAMPLE;
            ctx->observation(o, ctx->observation_env);                      /* infer.c:1152 */
            uint32_t *t = &o.token_0;
            for (int i = 0; i < 6; i++) t[i] = top6[i];
            ctx->observation(o, ctx->observation_env);                      /* infer.c:1086-1096 */
        }
        return next;
    }
    float *logits = llm_forward(ctx, output_ids[pos], pos, ctx->max_seq_len, 1, llm, ctx->lora);
    notify(ctx, -1, NANO_PH_SAMPLE);
    const uint32_t V = (uint32_t)sp->vocab_size;
    uint8_t *seen = (uint8_t *)calloc(V, 1);
    if (seen) {
        for (uint32_t i = 0; i < pos; i++) seen[output_ids[i]] = 1;
        for (uint32_t v = 0; v < V; v++) if (seen[v]) logits[v] /= sp->repetition_penalty;
        free(seen);
    }
    for (uint32_t v = 0; v < V; v++) logits[v] /= sp->temperature;
    softmax_inplace(logits, (int)V);
    const float coin = random_f32(&sp->rng_state);
    return (uint32_t)sample_nucleus(ctx, logits, (int)V, sp->top_p, sp->probindex, coin);   /* infer.c:1183: always the top-p branch */
}

/* ------------------------------------------------------------------------------------------------------ */
/* sessions (infer.c:1196-1362)                                                                            */
/* ------------------------------------------------------------------------------------------------------ */
Nano_Session *llm_session_init(Nano_Context *ctx, wchar_t *prompt, uint32_t max_seq_len, int32_t is_thinking_enabled) {
    Nano_Session *s = (Nano_Session *)platform_calloc(1, sizeof(Nano_Session));
    s->prompt = (wchar_t *)platform_calloc(max_seq_len + 1, sizeof(wchar_t));
    wcscpy(s->prompt, prompt ? prompt : L"");
    s->max_seq_len = max_seq_len;
    s->output_ids = (uint32_t *)platform_calloc(max_seq_len + 1, sizeof(uint32_t));
    uint32_t *toks = NULL;
    if (ctx->llm->arch == NANO_ARCH_NANO) toks = encode_nano(ctx->tokenizer, s->prompt, &s->num_prompt_tokens);
    else if (ctx->llm->arch == NANO_ARCH_QWEN2 || ctx->llm->arch == NANO_ARCH_QWEN3)
        toks = apply_qwen_chat_template(ctx->tokenizer, s->prompt, &s->num_prompt_tokens, is_thinking_enabled);
    else { printf("Error: unknown LLM arch.\n"); return NULL; }
    for (uint32_t i = 0; i < s->num_prompt_tokens && i <= max_seq_len; i++) s->output_ids[i] = toks[i];
    s->next_token = toks[0];
    free(toks);
    return s;
}

static wchar_t *detok(Nano_Context *ctx, uint32_t *ids, uint32_t n) {
    return (ctx->llm->arch == NANO_ARCH_NANO) ? decode_nano(ctx->tokenizer, ids, n) : decode_bpe(ctx->tokenizer, ids, n);
}

int32_t llm_session_step(Nano_Context *ctx, Nano_Session *s) {
    /* past the model's RoPE table no position has a defined result (the engine refuses it): end the session like at max_seq_len */
    if (s->pos >= s->max_seq_len || s->pos >= ctx->llm->config.block_size) return NANO_STOP_ERROR;
    const uint32_t arch = ctx->llm->arch;
    if (arch != NANO_ARCH_NANO && arch != NANO_ARCH_QWEN2 && arch != NANO_ARCH_QWEN3) { printf("Error: unknown LLM arch.\n"); return NANO_STOP_ERROR; }
    if (s->output_text) { free(s->output_text); s->output_text = NULL; }
    s->is_prefilling = (s->pos + 1 < s->num_prompt_tokens) ? 1 : 0;
    s->next_token = generate_next_token(ctx, s->output_ids, s->pos, s->is_prefilling);
    if (s->is_prefilling) {
        s->output_text = detok(ctx, s->output_ids, s->pos);
    } else {
        s->output_ids[s->num_prompt_tokens + s->output_count++] = s->next_token;
        s->output_text = detok(ctx, s->output_ids + s->num_prompt_tokens, s->output_count);
    }
    s->pos++;
    if (arch == NANO_ARCH_NANO && (s->next_token == 0 || s->next_token == 3)) return NANO_STOP_NORMAL;
    if (arch != NANO_ARCH_NANO && !s->is_prefilling && (s->next_token == 151643 || s->next_token == 151645)) return NANO_STOP_NORMAL;
    return s->is_prefilling ? NANO_RUN_PREFILL : NANO_RUN_DECODE;
}

void llm_session_free(Nano_Session *s) {
    if (!s) return;
    free(s->prompt); free(s->output_ids); free(s->output_text); free(s);
}

int32_t generate_sync(Nano_Context *ctx, wchar_t *prompt, uint32_t max_seq_len, int32_t (*on_prefilling)(Nano_Session *),
                      int32_t (*on_decoding)(Nano_Session *), int32_t (*on_finished)(Nano_Session *)) {
    Nano_Session *s = llm_session_init(ctx, prompt, max_seq_len, 1);
    int32_t status;
    for (;;) {
        status = llm_session_step(ctx, s);
        if (status == NANO_RUN_PREFILL) {
            if (on_prefilling(s) == NANO_STOP_IN_PREFILL) { status = NANO_STOP_IN_PREFILL; break; }
        } else if (status == NANO_RUN_DECODE) {
            if (on_decoding(s) == NANO_STOP_IN_DECODE) { status = NANO_STOP_IN_DECODE; break; }
        } else if (status == NANO_STOP_NORMAL) {
            status = on_finished(s); break;
        } else {
            on_finished(s); status = NANO_STOP_ERROR; break;
        }
    }
    llm_session_free(s);
    return status;
}

/* infer.c:1365-1402: n_layer relaxation sweeps with global attention, then one sweep collecting argmaxes */
void seq2seq(Nano_Context *ctx, wchar_t *input_list, wchar_t *output_list, uint32_t max_seq_len) {
    uint32_t n_in = 0;
    uint32_t *in = encode_nano(ctx->tokenizer, input_list, &n_in);
    uint32_t *out = (uint32_t *)platform_calloc(max_seq_len, sizeof(uint32_t));
    LLM *llm = ctx->llm;
    nb200_engine *e = engine_of(llm);
    const uint32_t V = llm->config.vocab_size;
    if (nb200_lora_enable(e, 0) != NB200_OK) die("seq2seq (use_lora)");       /* the reference passes lora = NULL for the whole of seq2seq (infer.c:1365-1402) */
    for (uint32_t sweep = 0; sweep < llm->config.n_layer; sweep++)
        for (uint32_t pos = 0; pos < max_seq_len; pos++) {
            notify_forward(ctx);
            if (nb200_forward(e, in[pos], pos, 0) != NB200_OK) die("seq2seq");
        }
    for (uint32_t pos = 0; pos < max_seq_len; pos++) {
        float *lg = llm_forward(ctx, in[pos], pos, max_seq_len, 0, llm, NULL);
        uint32_t best = 0;
        for (uint32_t v = 1; v < V; v++) if (lg[v] > lg[best]) best = v;      /* sample_argmax: first max */
        out[pos] = best;
    }
    wchar_t *txt = decode_nano(ctx->tokenizer, out, max_seq_len);
    wcscpy(output_list, txt);
    free(txt); free(in); free(out);
}

/* ------------------------------------------------------------------------------------------------------ */
/* tensor.h helpers with host-pointer semantics                                                            */
/* ------------------------------------------------------------------------------------------------------ */
void dequantize(Q80_Tensor *qx, float *x, int n, uint32_t group_size) {         /* tensor.c:15-19 (load-time helper) */
    for (int i = 0; i < n; i++) x[i] = qx->q[i] * qx->s[(uint32_t)i / group_size];
}

void quantize(Q80_Tensor *qx, float *x, int n, uint32_t group_size) {           /* tensor.c:21-46 on the GPU */
    if (nb200_op_q80_quantize(qx->q, qx->s, x, (uint32_t)n, group_size) != NB200_OK) die("quantize");
}

Typed_Tensor *parse_quantized_tensors(void **ptr, int n, int size_each, uint32_t group_size) {   /* tensor.c:49-62 */
    uint8_t *p = (uint8_t *)*ptr;
    Typed_Tensor *r = (Typed_Tensor *)platform_malloc((size_t)n * sizeof(Typed_Tensor));
    for (int i = 0; i < n; i++) {
        r[i].tensor_q80.q = (int8_t *)p; p += size_each;
        r[i].tensor_q80.s = (float *)(void *)p; p += ((size_t)size_each / group_size) * sizeof(float);
    }
    *ptr = p;
    return r;
}

/* Q4K framing: {u64 bytes}{u32 tag}{u32 ndim}{u32 shape[6]}{u32 nblocks} + 160-byte blocks (tensor.h:96-135) */
uint64_t bytes_num_of_q4k_tensor(uint8_t *Q) { return 44ull + (uint64_t)rd32(Q + 40) * 160ull; }

uint8_t *make_q4k_tensor(uint32_t ndim, uint32_t shape[]) {
    uint64_t lines = 1;
    for (uint32_t i = 0; i + 1 < ndim; i++) lines *= shape[i];
    const uint32_t bpl = (shape[ndim - 1] + 255u) / 256u;
    const uint64_t nb = lines * bpl, total = 44ull + nb * 160ull;
    uint8_t *T = (uint8_t *)platform_calloc(total, 1);
    const uint32_t tag = 0x42u, nb32 = (uint32_t)nb;
    memcpy(T, &total, 8); memcpy(T + 8, &tag, 4); memcpy(T + 12, &ndim, 4);
    for (uint32_t i = 0; i < ndim && i < 6; i++) memcpy(T + 16 + 4 * i, &shape[i], 4);
    memcpy(T + 40, &nb32, 4);
    return T;
}

/* tensor.c:281-310 on the GPU.  Every 256-element block of a "line" (last dimension) is quantised independently; lines
 * whose length is not a multiple of 256 are refused: the reference's own partial-block source offset (`t + i*line_dim +
 * j*d`, tensor.c:307) is only right for such lines when they are shorter than one block. */
void quantize_tensor_q4k_in_situ(float *t, uint32_t ndim, uint32_t shape[], uint8_t *T) {
    if (!t || !T || ndim == 0 || ndim > 6 || rd32(T + 12) != ndim) die("quantize_tensor_q4k_in_situ: bad tensor");
    const uint32_t line = shape[ndim - 1];
    if (line == 0 || line % 256u) die("quantize_tensor_q4k_in_situ: last dimension must be a multiple of 256");
    uint64_t lines = 1;
    for (uint32_t i = 0; i + 1 < ndim; i++) lines *= shape[i];
    for (uint32_t i = 0; i < ndim; i++) memcpy(T + 16 + 4 * i, &shape[i], 4);
    const uint64_t nb = lines * (line / 256u);
    if (nb != rd32(T + 40)) die("quantize_tensor_q4k_in_situ: block count mismatch");
    if (nb200_op_q4k_quantize_blocks(T + 44, t, nb) != NB200_OK) die("quantize_tensor_q4k_in_situ");
}

uint8_t *quantize_tensor_q4k(float *t, uint32_t ndim, uint32_t shape[]) {          /* tensor.c:312-316 */
    uint8_t *T = make_q4k_tensor(ndim, shape);
    quantize_tensor_q4k_in_situ(t, ndim, shape, T);
    return T;
}

/* tensor.c:438-471: W(d,n) or W(l,d,n)[layer] times an already-quantised x(n); host pointers in and out */
void matmul_q4k(float *xout, uint8_t *x, uint8_t *w, uint32_t layer) {
    const uint32_t wdim = rd32(w + 12);
    if (wdim != 2 && wdim != 3) die("matmul_q4k: weight tensor must have 2 or 3 dimensions");
    const uint32_t l = (wdim == 3) ? rd32(w + 16) : 1u, d = rd32(w + 16 + 4 * (wdim - 2)), n = rd32(w + 16 + 4 * (wdim - 1));
    if (rd32(x + 16) != n) die("matmul_q4k: x length differs from the weight's last dimension");
    if (wdim == 2) layer = 0;
    if (layer >= l) die("matmul_q4k: layer out of range");
    if (n % 256u) die("matmul_q4k: last dimension must be a multiple of 256");
    const uint64_t bpr = n / 256u;
    if (nb200_op_q4k_matvec_blocks(xout, x + 44, w + 44 + (uint64_t)layer * d * bpr * 160ull, n, d) != NB200_OK) die("matmul_q4k");
}

uint8_t *pack_q4k_tensor(uint8_t *Q) { return Q; }
uint8_t *unpack_q4k_tensor(uint8_t *buffer, uint64_t *p_total_bytes) { memcpy(p_total_bytes, buffer, 8); return buffer; }

void dequantize_tensor_q4k(uint8_t *Q, float *out, uint32_t *ndim, uint32_t *shape) {   /* tensor.c:318-344 (load-time helper) */
    *ndim = rd32(Q + 12);
    for (uint32_t i = 0; i < *ndim; i++) shape[i] = rd32(Q + 16 + 4 * i);
    const uint32_t n = shape[*ndim - 1], bpl = (n + 255u) / 256u;
    uint64_t lines = 1;
    for (uint32_t i = 0; i + 1 < *ndim; i++) lines *= shape[i];
    const uint8_t *blk = Q + 44;
    for (uint64_t r = 0; r < lines; r++)
        for (uint32_t j = 0; j < bpl; j++, blk += 160) {
            float ss, sb; memcpy(&ss, blk + 12, 4); memcpy(&sb, blk + 16, 4);
            const uint8_t *c = blk + 20;
            const uint32_t len = rd32(blk + 4);
            float *dst = out + r * n + (uint64_t)j * len;
            for (uint32_t i = 0; i < len && i < 256; i++) {
                const uint32_t g = i >> 5, k = g & 3;
                const uint32_t s6 = (g < 4) ? (c[k] & 0x3fu) : ((((c[k] >> 6) << 4) | (c[8 + k] & 0x0fu)) & 0x3fu);
                const uint32_t b6 = (g < 4) ? (c[4 + k] & 0x3fu) : ((((c[4 + k] >> 6) << 4) | (c[8 + k] >> 4)) & 0x3fu);
                const uint8_t byte = blk[32 + (i >> 1)];
                const uint32_t code = (i & 1) ? (byte >> 4) : (byte & 0x0fu);
                dst[i] = (float)code * ((float)s6 * ss) - (float)b6 * sb;
            }
        }
}
