/*
 * oracle/nano_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * Plain-C restatement of the reference CPU engine's decode path (bd4sur/Nano infer/infer.c +
 * infer/tensor.c).  It is the CHECKER for the CUDA engine: only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  The product libraries never
 * link or dlopen it, and there is no CPU fallback in the product.
 *
 * Parity status: PINNED.  tests/test_oracle_vs_reference.py checks this file bit-for-bit against the
 * unmodified reference compiled with strict flags (oracle/_ref/libnano_ref_strict.so), on the
 * reference's embedded sort model (main_sort.c:6-3098, README.md:379 "114515 -> 111455") and on
 * synthetic F32/Q80/Q4K files; tests/golden/ holds the resulting fixtures for boxes without
 * /root/reference.
 *
 * Build with strict IEEE flags (-O2 -fno-fast-math -ffp-contract=off): every float expression below
 * is written in the reference's evaluation order and must not be contracted or re-associated.
 *
 * Each function cites the reference lines it follows.
 */
#include <float.h>
#include <math.h>
#include <omp.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define NOR_ARCH_NANO 0
#define NOR_ARCH_QWEN2 2
#define NOR_ARCH_QWEN3 3
#define NOR_QUANT_F32 0x00
#define NOR_QUANT_Q80 0x80
#define NOR_QUANT_Q4K 0x42
#define NOR_Q4K_BLOCK_BYTES 160
#define NOR_Q4K_TENSOR_HDR 44

/* ------------------------------------------------------------------------------------------ */
/* unaligned little-endian readers (file sections are not aligned: SURVEY Appendix A)          */
/* ------------------------------------------------------------------------------------------ */
static inline uint32_t rd_u32(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }
static inline uint64_t rd_u64(const uint8_t *p) { uint64_t v; memcpy(&v, p, 8); return v; }
static inline float rd_f32(const uint8_t *p) { float v; memcpy(&v, p, 4); return v; }
static inline void wr_u32(uint8_t *p, uint32_t v) { memcpy(p, &v, 4); }
static inline void wr_f32(uint8_t *p, float v) { memcpy(p, &v, 4); }

/* ------------------------------------------------------------------------------------------ */
/* Elementary ops                                                                              */
/* ------------------------------------------------------------------------------------------ */

/* OpenMP team size for the row-parallel loops (the reference leaves it to OMP_NUM_THREADS). Tiny loops
 * stay serial: forking a 200-thread team per 256-row matvec dominates on many-core hosts. */
static int g_threads = 8;
void nor_set_threads(int n) { g_threads = n > 0 ? n : 1; }
int nor_max_threads(void) { return omp_get_num_procs(); }
#define NOR_PAR(work) num_threads(g_threads) if ((work) >= (1 << 18))

/* infer.c:601-614 */
void nor_rmsnorm(float *out, const float *x, const float *gain, int n) {
    float acc = 0.0f;
    for (int i = 0; i < n; i++) acc += x[i] * x[i];
    acc /= n;
    acc += 1e-5f;
    acc = 1.0f / sqrtf(acc);
    for (int i = 0; i < n; i++) out[i] = gain[i] * (acc * x[i]);
}

/* infer.c:616-634 */
void nor_softmax(float *v, int n) {
    float top = v[0];
    for (int i = 1; i < n; i++) if (v[i] > top) top = v[i];
    float total = 0.0f;
    for (int i = 0; i < n; i++) { v[i] = expf(v[i] - top); total += v[i]; }
    for (int i = 0; i < n; i++) v[i] /= total;
}

/* infer.c:637-651 : out[d] = W[d][n] . x[n], strictly left-to-right per row */
void nor_matvec_f32(float *out, const float *x, const uint8_t *w_bytes, int n, int d) {
    #pragma omp parallel for NOR_PAR((long)d * n)
    for (int r = 0; r < d; r++) {
        const uint8_t *row = w_bytes + (size_t)r * n * 4;
        float acc = 0.0f;
        for (int j = 0; j < n; j++) acc += rd_f32(row + 4 * (size_t)j) * x[j];
        out[r] = acc;
    }
}

/* tensor.c:21-46.  An all-zero group gives scale 0 and 0/0 in the reference (UB cast that yields 0
 * on x86-64); normalised to code 0 here (SURVEY Appendix B). */
void nor_q80_quantize(int8_t *codes, float *scales, const float *x, int n, int gs) {
    int ngroups = n / gs;
    for (int g = 0; g < ngroups; g++) {
        const float *xg = x + (size_t)g * gs;
        float amax = 0.0f;
        for (int i = 0; i < gs; i++) { float a = (float)fabs(xg[i]); if (a > amax) amax = a; }
        float sc = amax / 127.0f;
        scales[g] = sc;
        for (int i = 0; i < gs; i++) {
            if (sc == 0.0f) { codes[g * gs + i] = 0; continue; }
            float t = xg[i] / sc;
            codes[g * gs + i] = (int8_t)round(t);
        }
    }
}

/* infer.c:654-679 : exact int32 group dots, then ((float)isum * ws) * xs accumulated left-to-right */
void nor_matvec_q80(float *out, const int8_t *xq, const float *xs, const int8_t *wq, const uint8_t *ws_bytes,
                    int n, int d, int gs) {
    int ngroups = n / gs;
    #pragma omp parallel for NOR_PAR((long)d * n)
    for (int r = 0; r < d; r++) {
        const int8_t *wrow = wq + (size_t)r * n;
        float acc = 0.0f;
        for (int g = 0; g < ngroups; g++) {
            int32_t isum = 0;
            for (int k = 0; k < gs; k++) isum += (int32_t)xq[g * gs + k] * (int32_t)wrow[g * gs + k];
            float wscale = rd_f32(ws_bytes + 4 * ((size_t)r * ngroups + g));
            acc += ((float)isum) * wscale * xs[g];
        }
        out[r] = acc;
    }
}

/* infer.c:681-690 : adjacent pairs (Nano / Qwen2) */
static void rope_adjacent(float *h, int hd, const float *cr, const float *ci) {
    for (int i = 0; i < hd; i += 2) {
        float a = h[i], b = h[i + 1];
        float c = cr[i / 2], s = ci[i / 2];
        h[i] = a * c - b * s;
        h[i + 1] = a * s + b * c;
    }
}

/* infer.c:692-706 : half-split pairs (Qwen3) */
static void rope_halfsplit(float *h, int hd, const float *cr, const float *ci) {
    int half = hd / 2;
    for (int i = 0; i < half; i++) {
        float c = cr[i], s = ci[i];
        float a = h[i], b = h[i + half];
        h[i] = a * c - b * s;
        h[i + half] = b * c + a * s;
    }
}

void nor_rope(float *h, int hd, const float *cr, const float *ci, int halfsplit) {
    if (halfsplit) rope_halfsplit(h, hd, cr, ci); else rope_adjacent(h, hd, cr, ci);
}

/* ------------------------------------------------------------------------------------------ */
/* Q4K : 256-element blocks, 8 groups of 32, 6-bit group scales/biases (tensor.c:83-471)       */
/* block bytes: [0]u32 tag [4]u32 len [8]u32 meta [12]f32 s_scale [16]f32 s_bias [20]u8 sb[12] */
/*              [32]u8 nib[128]                                                                */
/* ------------------------------------------------------------------------------------------ */

/* tensor.c:4-9 : magic-constant round-half-even */
static inline int q4k_rne(float f) {
    float t = f + 12582912.f;
    int32_t i; memcpy(&i, &t, 4);
    return (i & 0x007fffff) - 0x00400000;
}

/* tensor.c:113-141 */
static void q4k_group_params(const uint8_t *blk, float *gscale, float *gbias) {
    const uint8_t *sb = blk + 20;
    float ss = rd_f32(blk + 12), sbias = rd_f32(blk + 16);
    for (int g = 0; g < 4; g++) {
        uint8_t s_lo = sb[g] & 0x3f;
        uint8_t b_lo = sb[4 + g] & 0x3f;
        uint8_t s_hi = (uint8_t)((((sb[g] >> 6) << 4) | (sb[8 + g] & 0x0f)) & 0x3f);
        uint8_t b_hi = (uint8_t)((((sb[4 + g] >> 6) << 4) | ((sb[8 + g] & 0xf0) >> 4)) & 0x3f);
        gscale[g] = (float)s_lo * ss;      gbias[g] = (float)b_lo * sbias;
        gscale[g + 4] = (float)s_hi * ss;  gbias[g + 4] = (float)b_hi * sbias;
    }
}

/* tensor.c:144-242 ; len <= 256 valid elements */
void nor_q4k_quantize_block(uint8_t *blk, const float *x, uint32_t len) {
    float gs[8], gb[8];
    wr_u32(blk, NOR_QUANT_Q4K);
    wr_u32(blk + 4, len);
    /* bytes 8..11 (meta) are left as the caller initialised them (calloc'd => 0) */
    for (uint32_t g = 0; g < 8; g++) {
        float lo = FLT_MAX, hi = FLT_TRUE_MIN;   /* NB: max starts at the smallest positive denormal */
        for (uint32_t i = g * 32; i < (g + 1) * 32 && i < len; i++) {
            float v = x[i];
            if (v > hi) hi = v;
            if (v < lo) lo = v;
        }
        gs[g] = (lo <= 0.0f) ? ((hi - lo) / 15.0f) : (hi / 15.0f);
        gb[g] = (lo <= 0.0f) ? (-lo) : 0.0f;
    }
    uint8_t code[256];
    memset(code, 0, sizeof code);
    for (uint32_t i = 0; i < len; i++) {
        uint32_t g = i / 32;
        float s = gs[g], b = gb[g];
        code[i] = (!s) ? 0 : (uint8_t)(q4k_rne((x[i] + b) / s) & 0x0f);
    }
    uint8_t *nib = blk + 32;
    for (uint32_t i = 0; i < 256; i += 2) nib[i >> 1] = (uint8_t)((code[i] & 0x0f) | (code[i + 1] << 4));

    float smax = FLT_TRUE_MIN, bmax = FLT_TRUE_MIN;
    for (int g = 0; g < 8; g++) { if (gs[g] > smax) smax = gs[g]; if (gb[g] > bmax) bmax = gb[g]; }
    float ss = smax / 63.0f, sbias = bmax / 63.0f;
    wr_f32(blk + 12, ss);
    wr_f32(blk + 16, sbias);
    uint8_t s6[8], b6[8];
    for (int g = 0; g < 8; g++) {
        s6[g] = (!ss) ? 0 : (uint8_t)(q4k_rne(gs[g] / ss) & 0x3f);
        b6[g] = (!sbias) ? 0 : (uint8_t)(q4k_rne(gb[g] / sbias) & 0x3f);
    }
    uint8_t *sb = blk + 20;
    for (int g = 0; g < 4; g++) {
        sb[g]     = (uint8_t)(((s6[4 + g] & 0x30) << 2) | (s6[g] & 0x3f));
        sb[4 + g] = (uint8_t)(((b6[4 + g] & 0x30) << 2) | (b6[g] & 0x3f));
        sb[8 + g] = (uint8_t)(((b6[4 + g] & 0x0f) << 4) | (s6[4 + g] & 0x0f));
    }
}

/* tensor.c:253-278 : value = code*s - b */
uint32_t nor_q4k_dequant_block(const uint8_t *blk, float *out) {
    float gs[8], gb[8];
    uint32_t len = rd_u32(blk + 4);
    q4k_group_params(blk, gs, gb);
    const uint8_t *nib = blk + 32;
    for (uint32_t i = 0; i < len && i < 256; i++) {
        uint8_t c = (i & 1) ? (uint8_t)((nib[i >> 1] >> 4) & 0x0f) : (uint8_t)(nib[i >> 1] & 0x0f);
        out[i] = (float)c * gs[i / 32] - gb[i / 32];
    }
    return len;
}

/* tensor.c:359-434 */
static float q4k_block_dot(const uint8_t *p, const uint8_t *q) {
    float ps[8], pb[8], qs[8], qb[8];
    uint32_t len = rd_u32(p + 4);
    q4k_group_params(p, ps, pb);
    q4k_group_params(q, qs, qb);
    float total = 0.0f;
    for (uint32_t g = 0; g < 8; g++) {
        int32_t glen = (len >= (g + 1) * 32) ? 32 : (int32_t)len - (int32_t)(32 * g);
        if (glen <= 0) break;
        int32_t s_pq = 0, s_p = 0, s_q = 0;
        for (int32_t i = 0; i < glen; i++) {
            uint32_t e = g * 32 + (uint32_t)i;
            int32_t a = (e & 1) ? (p[32 + (e >> 1)] >> 4) : (p[32 + (e >> 1)] & 0x0f);
            int32_t b = (e & 1) ? (q[32 + (e >> 1)] >> 4) : (q[32 + (e >> 1)] & 0x0f);
            s_pq += a * b; s_p += a; s_q += b;
        }
        float sp = ps[g], sq = qs[g], bp = pb[g], bq = qb[g];
        float term = sp * sq * (float)s_pq
                   - sp * bq * (float)s_p
                   - sq * bp * (float)s_q
                   + glen * bp * bq;
        total += term;
    }
    return total;
}

/* tensor.c:281-310 restricted to n % 256 == 0 or a single short line (the reference's partial-block
 * offset is only right in those cases, SURVEY Appendix B). blocks_out: nblk*160 bytes, zero-filled. */
void nor_q4k_quantize_rows(uint8_t *blocks_out, const float *x, uint64_t nrows, uint32_t n) {
    uint32_t bpr = (n + 255) / 256;
    #pragma omp parallel for NOR_PAR((long)nrows * n)
    for (uint64_t r = 0; r < nrows; r++) {
        for (uint32_t j = 0; j < bpr; j++) {
            uint32_t len = (n >= (j + 1) * 256) ? 256 : (n - j * 256);
            nor_q4k_quantize_block(blocks_out + (r * bpr + j) * NOR_Q4K_BLOCK_BYTES, x + r * n + (uint64_t)j * len, len);
        }
    }
}

/* tensor.c:438-471 : rows [row0,row0+d) of a block array with bpr blocks per row */
void nor_matvec_q4k(float *out, const uint8_t *xblocks, const uint8_t *wblocks, uint64_t row0, uint32_t d, uint32_t n) {
    uint32_t bpr = (n + 255) / 256;
    #pragma omp parallel for NOR_PAR((long)d * n)
    for (uint32_t r = 0; r < d; r++) {
        const uint8_t *wrow = wblocks + (row0 + r) * bpr * NOR_Q4K_BLOCK_BYTES;
        float acc = 0.0f;
        for (uint32_t j = 0; j < bpr; j++)
            acc += q4k_block_dot(wrow + (size_t)j * NOR_Q4K_BLOCK_BYTES, xblocks + (size_t)j * NOR_Q4K_BLOCK_BYTES);
        out[r] = acc;
    }
}

/* ------------------------------------------------------------------------------------------ */
/* Model: pointers into the caller's file image + private activation / KV buffers             */
/* ------------------------------------------------------------------------------------------ */
typedef struct { const uint8_t *q; const uint8_t *s; } Q80Ref;       /* per-layer tensor: codes, scales */

typedef struct NorModel {
    uint32_t arch, quant, gs;
    uint32_t block_size, vocab, L, E, H, KV, F, tied, hd, q_dim, kv_dim, max_seq;
    const uint8_t *norm_attn, *norm_ffn, *norm_final;      /* f32 */
    const uint8_t *qnorm, *knorm;                          /* f32 [L][hd] (arch 3) */
    /* F32: byte pointers to [L][d][n]; Q80: arrays of L refs; Q4K: block arrays (after 44 B header) */
    const uint8_t *emb_f32; Q80Ref emb_q80; const uint8_t *emb_q4k;
    const uint8_t *w_f32[7]; Q80Ref *w_q80[7]; const uint8_t *w_q4k[7];   /* order: wq wk wv wo w1 w2 w3 */
    Q80Ref cls_q80; int cls_untied;
    float *rope_cos, *rope_sin; int rope_owned;
    /* state */
    float *x, *xb, *xba, *xb2, *hb, *hb2, *q, *att, *logits, *kc, *vc, *embrow;
    int8_t *aq; float *as; uint8_t *ablk;
    /* probe */
    int32_t p_layer, p_phase, p_field; float *p_dst; uint32_t p_count, p_hits;
} NorModel;

enum { NOR_PH_EMB = 1, NOR_PH_ATTN_NORM, NOR_PH_QKV, NOR_PH_ROPE, NOR_PH_MHA, NOR_PH_O, NOR_PH_FFN_NORM,
       NOR_PH_W13, NOR_PH_W2, NOR_PH_FINAL_NORM, NOR_PH_CLS };   /* same ids as infer.h:65-76 */

static void probe(NorModel *m, int layer, int phase, float *kptr, float *vptr) {
    if (!m->p_dst || m->p_layer != layer || m->p_phase != phase) return;
    float *src = NULL;
    switch (m->p_field) {
        case 0: src = m->x; break; case 1: src = m->xb; break; case 2: src = m->xba; break;
        case 3: src = m->xb2; break; case 4: src = m->hb; break; case 5: src = m->hb2; break;
        case 6: src = m->q; break; case 7: src = kptr; break; case 8: src = vptr; break;
        case 9: src = m->logits; break;
    }
    if (src) memcpy(m->p_dst, src, (size_t)m->p_count * 4);
    m->p_hits++;
}

void nor_set_probe(NorModel *m, int32_t layer, int32_t phase, int32_t field, float *dst, uint32_t count) {
    m->p_layer = layer; m->p_phase = phase; m->p_field = field; m->p_dst = dst; m->p_count = count; m->p_hits = 0;
}

static const uint8_t *take_q80(const uint8_t **cur, Q80Ref *refs, uint64_t count, uint64_t each, uint32_t gs) {
    const uint8_t *p = *cur;
    for (uint64_t i = 0; i < count; i++) {       /* tensor.c:49-62 */
        refs[i].q = p; p += each;
        refs[i].s = p; p += (each / gs) * 4;
    }
    *cur = p;
    return p;
}

static const uint8_t *take_q4k(const uint8_t **cur) {   /* tensor.c:352-355 framing */
    const uint8_t *p = *cur;
    uint64_t total = rd_u64(p);
    *cur = p + total;
    return p + NOR_Q4K_TENSOR_HDR;
}

/* infer.c:220-320 (header), :100-217 (parameter map), :15-85 (buffers). The tokenizer section is
 * skipped via its length field; tokenisation is outside the hot path. */
NorModel *nor_open(const uint8_t *file, uint64_t file_len, uint32_t max_seq) {
    (void)file_len;
    NorModel *m = (NorModel *)calloc(1, sizeof(NorModel));
    m->arch = rd_u32(file + 4 * 4);
    m->block_size = rd_u32(file + 4 * 6); m->vocab = rd_u32(file + 4 * 7); m->L = rd_u32(file + 4 * 8);
    m->E = rd_u32(file + 4 * 9); m->H = rd_u32(file + 4 * 10); m->KV = rd_u32(file + 4 * 11);
    m->F = rd_u32(file + 4 * 12); m->tied = rd_u32(file + 4 * 13); m->hd = rd_u32(file + 4 * 14);
    uint32_t qt = rd_u32(file + 4 * 15);
    m->quant = (qt == NOR_QUANT_F32 || qt == NOR_QUANT_Q80 || qt == NOR_QUANT_Q4K) ? qt : NOR_QUANT_Q80;
    m->gs = rd_u32(file + 4 * 16);
    m->max_seq = max_seq;
    if (m->arch != NOR_ARCH_QWEN3) m->hd = m->E / m->H;
    m->q_dim = (m->arch == NOR_ARCH_QWEN3) ? m->hd * m->H : m->E;
    m->kv_dim = (m->arch == NOR_ARCH_QWEN3) ? m->hd * m->KV : (m->E * m->KV) / m->H;

    uint32_t tok_bytes = rd_u32(file + 256);
    const uint8_t *cur = file + 256 + tok_bytes;
    uint64_t L = m->L, E = m->E, V = m->vocab, F = m->F, QD = m->q_dim, KD = m->kv_dim;
    m->norm_attn = cur; cur += L * E * 4;
    m->norm_ffn = cur;  cur += L * E * 4;
    m->norm_final = cur; cur += E * 4;
    const uint64_t rows[7] = {QD, KD, KD, E, F, E, F};
    const uint64_t cols[7] = {E, E, E, QD, E, F, E};
    if (m->quant == NOR_QUANT_F32) {
        m->emb_f32 = cur; cur += V * E * 4;
        for (int t = 0; t < 7; t++) { m->w_f32[t] = cur; cur += L * rows[t] * cols[t] * 4; }
    } else if (m->quant == NOR_QUANT_Q80) {
        take_q80(&cur, &m->emb_q80, 1, V * E, m->gs);
        for (int t = 0; t < 7; t++) {
            m->w_q80[t] = (Q80Ref *)calloc(L, sizeof(Q80Ref));
            take_q80(&cur, m->w_q80[t], L, rows[t] * cols[t], m->gs);
        }
    } else {
        m->emb_q4k = take_q4k(&cur);
        for (int t = 0; t < 7; t++) m->w_q4k[t] = take_q4k(&cur);
    }
    if (m->arch == NOR_ARCH_QWEN2) cur += L * (QD + 2 * KD) * 4;          /* biases: parsed, never applied */
    if (m->arch == NOR_ARCH_QWEN3) { m->qnorm = cur; cur += L * m->hd * 4; m->knorm = cur; cur += L * m->hd * 4; }
    uint64_t half = m->hd / 2, tbl = (uint64_t)m->block_size * half;
    m->rope_cos = (float *)malloc(tbl * 4 + 4);
    m->rope_sin = (float *)malloc(tbl * 4 + 4);
    m->rope_owned = 1;
    if (m->arch == NOR_ARCH_QWEN3) {                       /* infer.c:189-204, theta = 1e6, host libm */
        for (uint32_t pos = 0; pos < m->block_size; pos++)
            for (uint32_t i = 0; i < half; i++) {
                float freq = 1.0f / powf(1000000.0f, (float)(i * 2) / (float)m->hd);
                m->rope_cos[pos * half + i] = cosf(pos * freq);
                m->rope_sin[pos * half + i] = sinf(pos * freq);
            }
        cur += 2 * tbl * 4;   /* the reference advances past a table even when the file has none */
    } else {
        memcpy(m->rope_cos, cur, tbl * 4); cur += tbl * 4;
        memcpy(m->rope_sin, cur, tbl * 4); cur += tbl * 4;
    }
    if (m->quant == NOR_QUANT_Q80 && !m->tied) { take_q80(&cur, &m->cls_q80, 1, E * V, m->gs); m->cls_untied = 1; }

    uint64_t maxd = F > QD ? F : QD; if (E > maxd) maxd = E;
    m->x = calloc(E, 4); m->xb = calloc(E, 4); m->xba = calloc(QD, 4); m->xb2 = calloc(E, 4);
    m->hb = calloc(F, 4); m->hb2 = calloc(F, 4); m->q = calloc(QD, 4);
    m->att = calloc((uint64_t)m->H * max_seq, 4); m->logits = calloc(V, 4); m->embrow = calloc(E, 4);
    m->kc = calloc(L * max_seq * KD, 4); m->vc = calloc(L * max_seq * KD, 4);
    m->aq = calloc(maxd, 1); m->as = calloc(maxd, 4);
    m->ablk = calloc(((maxd + 255) / 256) * NOR_Q4K_BLOCK_BYTES, 1);
    return m;
}

void nor_close(NorModel *m) {
    for (int t = 0; t < 7; t++) free(m->w_q80[t]);
    free(m->rope_cos); free(m->rope_sin);
    free(m->x); free(m->xb); free(m->xba); free(m->xb2); free(m->hb); free(m->hb2); free(m->q);
    free(m->att); free(m->logits); free(m->embrow); free(m->kc); free(m->vc); free(m->aq); free(m->as); free(m->ablk);
    free(m);
}

void nor_config(const NorModel *m, uint32_t out[16]) {
    out[0] = m->block_size; out[1] = m->vocab; out[2] = m->L; out[3] = m->E; out[4] = m->H; out[5] = m->KV;
    out[6] = m->F; out[7] = m->tied; out[8] = m->hd; out[9] = m->arch; out[10] = m->quant; out[11] = m->gs;
    out[12] = m->max_seq; out[13] = m->q_dim; out[14] = m->kv_dim;
}

float *nor_kcache(NorModel *m) { return m->kc; }
float *nor_vcache(NorModel *m) { return m->vc; }
float *nor_logits(NorModel *m) { return m->logits; }

/* one projection: out[d] = W_t[layer] . act ; the activation has already been quantised if needed */
static void project(NorModel *m, int t, uint32_t layer, float *out, const float *act, uint32_t n, uint32_t d) {
    if (m->quant == NOR_QUANT_F32) {
        nor_matvec_f32(out, act, m->w_f32[t] + (uint64_t)layer * d * n * 4, (int)n, (int)d);
    } else if (m->quant == NOR_QUANT_Q80) {
        const Q80Ref *w = &m->w_q80[t][layer];
        nor_matvec_q80(out, m->aq, m->as, (const int8_t *)w->q, w->s, (int)n, (int)d, (int)m->gs);
    } else {
        nor_matvec_q4k(out, m->ablk, m->w_q4k[t], (uint64_t)layer * d, d, n);
    }
}

/* activation quantisation preceding a group of projections (infer.c:776,782,889,893,926,931,954,958) */
static void prep_act(NorModel *m, const float *act, uint32_t n) {
    if (m->quant == NOR_QUANT_Q80) nor_q80_quantize(m->aq, m->as, act, (int)n, (int)m->gs);
    else if (m->quant == NOR_QUANT_Q4K) {
        uint32_t nb = (n + 255) / 256;
        memset(m->ablk, 0, (size_t)nb * NOR_Q4K_BLOCK_BYTES);
        nor_q4k_quantize_rows(m->ablk, act, 1, n);
    }
}

/* infer.c:987-988 with the load-time dequantisation (infer.c:126-127,147-149) applied to one row */
static void fetch_embedding(NorModel *m, uint32_t token, float *dst) {
    uint64_t E = m->E;
    if (m->quant == NOR_QUANT_F32) {
        memcpy(dst, m->emb_f32 + (uint64_t)token * E * 4, E * 4);
    } else if (m->quant == NOR_QUANT_Q80) {
        const int8_t *codes = (const int8_t *)m->emb_q80.q + (uint64_t)token * E;
        for (uint64_t i = 0; i < E; i++)
            dst[i] = codes[i] * rd_f32(m->emb_q80.s + 4 * (((uint64_t)token * E + i) / m->gs));   /* tensor.c:15-19 */
    } else {
        uint32_t bpr = (m->E + 255) / 256;
        for (uint32_t j = 0; j < bpr; j++)
            nor_q4k_dequant_block(m->emb_q4k + ((uint64_t)token * bpr + j) * NOR_Q4K_BLOCK_BYTES, dst + j * 256);
    }
}

/* infer.c:713-966 */
static void layer_forward(NorModel *m, uint32_t layer, uint32_t pos, int causal) {
    uint32_t E = m->E, F = m->F, hd = m->hd, QD = m->q_dim, KD = m->kv_dim, S = m->max_seq;
    uint32_t kv_mul = m->H / m->KV;
    const float *cr = m->rope_cos + (uint64_t)pos * hd / 2, *ci = m->rope_sin + (uint64_t)pos * hd / 2;
    float *gain = (float *)malloc(E * 4);
    float *kbase = m->kc + (uint64_t)layer * S * KD, *vbase = m->vc + (uint64_t)layer * S * KD;
    float *krow = kbase + (uint64_t)pos * KD, *vrow = vbase + (uint64_t)pos * KD;

    probe(m, (int)layer, NOR_PH_ATTN_NORM, krow, vrow);
    memcpy(gain, m->norm_attn + (uint64_t)layer * E * 4, E * 4);
    nor_rmsnorm(m->xb, m->x, gain, (int)E);
    probe(m, (int)layer, NOR_PH_QKV, krow, vrow);
    prep_act(m, m->xb, E);
    project(m, 0, layer, m->q, m->xb, E, QD);
    project(m, 1, layer, krow, m->xb, E, KD);
    project(m, 2, layer, vrow, m->xb, E, KD);
    probe(m, (int)layer, NOR_PH_ROPE, krow, vrow);

    if (m->arch == NOR_ARCH_QWEN3) {                     /* infer.c:824-835 */
        float hg[512];
        memcpy(hg, m->qnorm + (uint64_t)layer * hd * 4, hd * 4);
        for (uint32_t h = 0; h < m->H; h++) { float *v = m->q + h * hd; nor_rmsnorm(v, v, hg, (int)hd); rope_halfsplit(v, (int)hd, cr, ci); }
        memcpy(hg, m->knorm + (uint64_t)layer * hd * 4, hd * 4);
        for (uint32_t h = 0; h < m->KV; h++) { float *v = krow + h * hd; nor_rmsnorm(v, v, hg, (int)hd); rope_halfsplit(v, (int)hd, cr, ci); }
    } else {                                             /* infer.c:814-823 */
        for (uint32_t h = 0; h < m->H; h++) rope_adjacent(m->q + h * hd, (int)hd, cr, ci);
        for (uint32_t h = 0; h < m->KV; h++) rope_adjacent(krow + h * hd, (int)hd, cr, ci);
    }
    probe(m, (int)layer, NOR_PH_MHA, krow, vrow);

    uint32_t span = causal ? pos + 1 : S;                /* infer.c:841-879 */
    #pragma omp parallel for NOR_PAR((long)m->H * span * hd * 8)
    for (uint32_t h = 0; h < m->H; h++) {
        const float *qh = m->q + h * hd;
        float *att = m->att + (uint64_t)h * S;
        uint32_t kvh = h / kv_mul;
        for (uint32_t t = 0; t < span; t++) {
            const float *kt = kbase + (uint64_t)t * KD + kvh * hd;
            float sc = 0.0f;
            for (uint32_t i = 0; i < hd; i++) sc += qh[i] * kt[i];
            sc /= sqrtf(hd);
            att[t] = sc;
        }
        nor_softmax(att, (int)span);
        float *o = m->xba + h * hd;
        memset(o, 0, hd * 4);
        for (uint32_t t = 0; t < span; t++) {
            const float *vt = vbase + (uint64_t)t * KD + kvh * hd;
            float a = att[t];
            for (uint32_t i = 0; i < hd; i++) o[i] += a * vt[i];
        }
    }
    probe(m, (int)layer, NOR_PH_O, krow, vrow);

    prep_act(m, m->xba, QD);
    project(m, 3, layer, m->xb2, m->xba, QD, E);
    for (uint32_t i = 0; i < E; i++) m->x[i] += m->xb2[i];
    probe(m, (int)layer, NOR_PH_FFN_NORM, krow, vrow);

    memcpy(gain, m->norm_ffn + (uint64_t)layer * E * 4, E * 4);
    nor_rmsnorm(m->xb, m->x, gain, (int)E);
    probe(m, (int)layer, NOR_PH_W13, krow, vrow);
    prep_act(m, m->xb, E);
    project(m, 4, layer, m->hb, m->xb, E, F);
    project(m, 6, layer, m->hb2, m->xb, E, F);
    for (uint32_t i = 0; i < F; i++) {                   /* infer.c:937-944 */
        float v = m->hb[i];
        v *= (1.0f / (1.0f + expf(-v)));
        v *= m->hb2[i];
        m->hb[i] = v;
    }
    probe(m, (int)layer, NOR_PH_W2, krow, vrow);
    prep_act(m, m->hb, F);
    project(m, 5, layer, m->xb, m->hb, F, E);
    for (uint32_t i = 0; i < E; i++) m->x[i] += m->xb[i];
    free(gain);
}

/* infer.c:971-1018 */
float *nor_forward(NorModel *m, uint32_t token, uint32_t pos, int causal) {
    uint32_t E = m->E, V = m->vocab;
    fetch_embedding(m, token, m->x);
    for (uint32_t l = 0; l < m->L; l++) layer_forward(m, l, pos, causal);
    probe(m, (int)m->L, NOR_PH_FINAL_NORM, NULL, NULL);
    float *gain = (float *)malloc(E * 4);
    memcpy(gain, m->norm_final, E * 4);
    nor_rmsnorm(m->x, m->x, gain, (int)E);
    free(gain);
    probe(m, (int)m->L, NOR_PH_CLS, NULL, NULL);
    if (m->quant == NOR_QUANT_F32) {
        nor_matvec_f32(m->logits, m->x, m->emb_f32, (int)E, (int)V);    /* tied: infer.c:215 */
    } else if (m->quant == NOR_QUANT_Q80) {
        const Q80Ref *c = m->cls_untied ? &m->cls_q80 : &m->emb_q80;
        prep_act(m, m->x, E);
        nor_matvec_q80(m->logits, m->aq, m->as, (const int8_t *)c->q, c->s, (int)E, (int)V, (int)m->gs);
    } else {
        prep_act(m, m->x, E);
        nor_matvec_q4k(m->logits, m->ablk, m->emb_q4k, 0, V, E);
    }
    return m->logits;
}

/* greedy half of infer.c:1135-1193 : penalty over ids[0..pos), first-max argmax (infer.c:1026-1037) */
uint32_t nor_next_greedy(NorModel *m, const uint32_t *ids, uint32_t pos, int prefilling, float penalty) {
    float *lg = nor_forward(m, ids[pos], pos, 1);
    if (prefilling) return ids[pos + 1];
    uint8_t *seen = (uint8_t *)calloc(m->vocab, 1);
    for (uint32_t i = 0; i < pos; i++) seen[ids[i]] = 1;
    for (uint32_t v = 0; v < m->vocab; v++) if (seen[v]) lg[v] /= penalty;
    free(seen);
    uint32_t best = 0; float bv = lg[0];
    for (uint32_t v = 1; v < m->vocab; v++) if (lg[v] > bv) { bv = lg[v]; best = v; }
    return best;
}

/* ------------------------------------------------------------------------------------------ */
/* Temperature / top-p sampling (infer.c:1174-1189, sample_top_p :1062-1109)                    */
/* ------------------------------------------------------------------------------------------ */
typedef struct { float prob; uint32_t index; } NorProbIndex;

/* infer.c:1053-1059 */
static int nor_prob_desc(const NorProbIndex *a, const NorProbIndex *b) {
    if (a->prob > b->prob) return -1;
    if (a->prob < b->prob) return 1;
    return 0;
}

/* stable merge sort by nor_prob_desc: the order glibc's (merge-sort) qsort gives the reference */
static void nor_sort_stable(NorProbIndex *a, NorProbIndex *tmp, uint32_t n) {
    for (uint32_t w = 1; w < n; w *= 2) {
        for (uint32_t lo = 0; lo < n; lo += 2 * w) {
            const uint32_t mid = lo + w < n ? lo + w : n, hi = lo + 2 * w < n ? lo + 2 * w : n;
            uint32_t i = lo, j = mid, k = lo;
            while (i < mid && j < hi) tmp[k++] = nor_prob_desc(&a[j], &a[i]) < 0 ? a[j++] : a[i++];
            while (i < mid) tmp[k++] = a[i++];
            while (j < hi) tmp[k++] = a[j++];
        }
        memcpy(a, tmp, (size_t)n * sizeof *a);
    }
}

/* One sampling step on `logits` [V] (penalty already applied; not modified).
 * out[0] = id, out[1..6] = the observation hook's six ids (0 where n0 <= i), out[7] = n0, out[8] = last (0xffffffff if n0 = 0).
 * sorted_p / sorted_i (optional, V entries): the n0 candidates in sorted order.
 * n0 = 0 (no probability reaches the cutoff) is undefined in the reference (probindex[-1]); here, as in the engine, the id is
 * the first-max argmax of the probabilities and the six ids are 0. */
void nor_sample_top_p(const float *logits, uint32_t V, float temperature, float top_p, float coin, uint32_t out[9],
                      float *sorted_p, uint32_t *sorted_i) {
    float *p = (float *)malloc((size_t)V * 4);
    NorProbIndex *pi = (NorProbIndex *)malloc((size_t)V * sizeof *pi), *tmp = (NorProbIndex *)malloc((size_t)V * sizeof *pi);
    for (uint32_t q = 0; q < V; q++) p[q] = logits[q] / temperature;            /* infer.c:1174-1176 */
    nor_softmax(p, (int)V);                                                     /* :1178 */
    const float cutoff = (1.0f - top_p) / (float)((int)V - 1);                  /* :1064 */
    uint32_t n0 = 0;
    for (uint32_t i = 0; i < V; i++)
        if (p[i] >= cutoff) { pi[n0].index = i; pi[n0].prob = p[i]; n0++; }
    nor_sort_stable(pi, tmp, n0);
    memset(out, 0, 9 * sizeof(uint32_t));
    out[7] = n0;
    for (uint32_t i = 0; i < 6; i++) out[1 + i] = n0 > i ? pi[i].index : 0u;
    if (sorted_p) for (uint32_t i = 0; i < n0; i++) sorted_p[i] = pi[i].prob;
    if (sorted_i) for (uint32_t i = 0; i < n0; i++) sorted_i[i] = pi[i].index;
    if (n0 == 0) {
        uint32_t best = 0;
        for (uint32_t i = 1; i < V; i++) if (p[i] > p[best]) best = i;
        out[0] = best; out[8] = 0xffffffffu;
    } else {
        float cum = 0.0f;                                                       /* :1075-1083 */
        uint32_t last = n0 - 1;
        for (uint32_t i = 0; i < n0; i++) { cum += pi[i].prob; if (cum > top_p) { last = i; break; } }
        const float r = coin * cum;                                             /* :1099-1108 */
        float cdf = 0.0f;
        uint32_t pick = last;
        for (uint32_t i = 0; i <= last; i++) { cdf += pi[i].prob; if (r < cdf) { pick = i; break; } }
        out[0] = pi[pick].index; out[8] = last;
    }
    free(p); free(pi); free(tmp);
}

/* ------------------------------------------------------------------------------------------ */
/* glibc-independent float exp used by the exact-mode CUDA path is validated against expf here */
/* ------------------------------------------------------------------------------------------ */
float nor_expf(float v) { return expf(v); }
void nor_expf_array(float *dst, const float *src, uint64_t n) { for (uint64_t i = 0; i < n; i++) dst[i] = expf(src[i]); }
