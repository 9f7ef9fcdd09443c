// engine.cu -- host side of libnano_b200.so: model-file parser, HBM layout/upload, CUDA-graph token
// step, and the C-ABI declared in include/nano_b200.h.
//
// HBM layout (free to differ from the file; the contract is the file format and the C API):
//   per layer, one fused row-major matrix per launch so each weight byte is streamed exactly once:
//     QKV  : rows = q_dim + 2*kv_dim  (wq rows, then wk, then wv)          n = n_embd
//     O    : rows = n_embd                                                  n = q_dim
//     W13  : rows = 2*n_hidden, row 2i = w1[i], row 2i+1 = w3[i]            n = n_embd
//     W2   : rows = n_embd                                                  n = n_hidden
//   CLS/embedding : rows = vocab (one copy when tied)                       n = n_embd
//   Q80 : int8 codes [rows][n] + fp32 scales [rows][n/gs]
//   Q4K : nibble plane [rows][n/2] (16-byte groups, 128-bit loads) + 20-byte side records
//         {s_scale, s_bias, sb[12]} [rows][n/256]; the constant 12 bytes {tag,len,meta} of each 160-byte
//         file block are dropped (148 B/block streamed instead of 160)
//   F32 : float [rows][n]
//   KV cache : [L][KV][max_seq][hd] fp32, head-major (a split-KV CTA reads one contiguous stream);
//              the reference's layout is [L][pos][kv_dim] (infer.c:46-51)
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../include/nano_b200.h"
#include "kernels.cuh"
#include "stream_host.h"
#include "sample_host.h"

using namespace nb;

namespace {

thread_local std::string g_err;

int fail(int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

#define CK(call)                                                                                     \
    do {                                                                                             \
        cudaError_t e_ = (call);                                                                     \
        if (e_ != cudaSuccess)                                                                       \
            return fail(NB200_ECUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

inline uint32_t rd_u32(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }
inline uint64_t rd_u64(const uint8_t *p) { uint64_t v; memcpy(&v, p, 8); return v; }

struct Mat {            // one fused device matrix
    void *w = nullptr;  // codes / floats / nibble plane
    void *aux = nullptr;
    uint32_t rows = 0, n = 0;
};

// staging -> (nibble plane, side records) with a row mapping dst_row = row_off + src_row * row_stride
__global__ void k_q4k_split(const uint8_t *__restrict__ blocks, uint64_t nblocks, uint32_t bpr, uint8_t *nib, uint8_t *side,
                            uint32_t row_off, uint32_t row_stride) {
    const uint64_t total = nblocks * 37;       // 32 nibble words + 5 side words per block
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t b = i / 37; const uint32_t wd = (uint32_t)(i % 37);
        const uint64_t srow = b / bpr; const uint32_t j = (uint32_t)(b % bpr);
        const uint64_t drow = row_off + srow * row_stride;
        const uint32_t *src = reinterpret_cast<const uint32_t *>(blocks + b * 160);
        if (wd < 32) reinterpret_cast<uint32_t *>(nib + (drow * bpr + j) * 128)[wd] = src[8 + wd];
        else reinterpret_cast<uint32_t *>(side + (drow * bpr + j) * 20)[wd - 32] = src[3 + (wd - 32)];
    }
}

}  // namespace

struct nb200_engine {
    Dims d{};
    uint32_t flags = 0;
    int device = 0, num_sms = 148;
    cudaStream_t stream = nullptr;
    std::vector<Mat> qkv, wo, w13, w2;
    Mat cls, emb;
    float *norm_attn = nullptr, *norm_ffn = nullptr, *norm_final = nullptr, *qnorm = nullptr, *knorm = nullptr;
    float *rope_cos = nullptr, *rope_sin = nullptr;
    float *x = nullptr, *q = nullptr, *kraw = nullptr, *xba = nullptr, *hb = nullptr, *logits = nullptr;
    float *kc = nullptr, *vc = nullptr, *att_exact = nullptr;
    float *ws_m = nullptr, *ws_l = nullptr, *ws_acc = nullptr;
    uint32_t *tickets = nullptr, *ids_dev = nullptr, *cls_idx = nullptr;
    float *cls_val = nullptr;
    uint8_t *seen = nullptr;
    DevState *st = nullptr;
    DevState *st_host = nullptr;      // pinned
    uint32_t *tok_host = nullptr;     // pinned result slot
    int8_t *dump_codes = nullptr; float *dump_scales = nullptr;
    uint32_t nsplit_max = 1, chunk_cap = 32, attn_smem = 0, cls_grid = 1;
    cudaGraphExec_t graph = nullptr;
    bool use_pdl = true;
    unsigned long long *trace_dev = nullptr;
    // grid-wide persistent streaming kernel (stream.cuh): the default path in fast mode on one GPU
    float calib_ms[2] = {0.0f, 0.0f};      // ms per token of {streaming, multi-kernel} measured by calibrate_paths (0 = not calibrated)
    bool use_stream = false; const void *st_kern = nullptr; StreamArgs sa{}; uint32_t st_smem = 0, st_grid = 0;
    uint32_t *st_err_host = nullptr, *st_err_dev = nullptr;      // mapped pinned word: the code a device-side spin recorded before trapping
    uint32_t st_epoch = 0;                                       // exchange epochs handed out so far (stream.cuh)
    void *samp_ws = nullptr; size_t samp_cub = 0; uint32_t *samp_host = nullptr;       // device-side sampler workspace (sample.cu), pinned result
    uint64_t stream_bytes = 0;
    unsigned int *bar = nullptr;
    uint64_t launches = 0, weight_bytes = 0;
    uint32_t launches_per_token = 0;
    uint32_t mv_mask = 0, attn_kind = 0;      // multi-kernel variants launched or captured so far (nb200_config.reserved[3], [4])
    std::vector<uint32_t> seen_mirror;   // ids whose seen[] flag is set, by position
    bool seen_valid = false;
    std::vector<void *> allocs;
    // tensor parallel (kernels.cuh "Tensor parallelism"): exchange block = [TpHdr | x | xba | hb]; d holds the LOCAL head counts
    uint32_t tp_rank = 0, tp_size = 1;
    bool tied = false;
    // LoRA plug-in (nb200_lora_load): fp32 factors [L][rank][n] / [L][rows][rank] for q, k, v, o; scratch t [4][rank], o1 [E]
    struct Lora { uint32_t rank = 0, alpha = 0; float *a[4] = {}, *b[4] = {}; float *t = nullptr, *o1 = nullptr; bool loaded = false, active = false; } lora;
    bool path_stream = false;     // what the model would run on without a plug-in
    unsigned long long *attn_dbg = nullptr;          // NB200_ATTN_DBG=1: %globaltimer stamps of layer L/2's attention kernel
    uint32_t g_H = 0, g_KV = 0, g_q_dim = 0, g_kv_dim = 0;     // whole-model values (== d.* on one GPU)
    unsigned char *tp_block = nullptr; size_t tp_block_bytes = 0;
    uint32_t tp_off_x = 0, tp_off_xba = 0, tp_off_hb = 0;
    unsigned char *tp_peer[kTpMax] = {};
    std::vector<void *> tp_ipc_opened;
    bool tp_attached = false;
    // per-kernel-class event profiling (nb200_profile_tokens)
    bool prof_on = false; int prof_tag = 0;
    struct ProfRec { int tag; cudaEvent_t a, b; };
    std::vector<ProfRec> prof;
};

namespace {

int dmalloc(nb200_engine *e, void **p, size_t bytes) {
    if (bytes == 0) bytes = 16;
    cudaError_t err = cudaMalloc(p, bytes);
    if (err != cudaSuccess) return fail(NB200_ENOMEM, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(err));
    e->allocs.push_back(*p);
    return 0;
}
#define DM(ptr, bytes) do { int r_ = dmalloc(e, (void **)&(ptr), (bytes)); if (r_) return r_; } while (0)

// ---------------- kernel launch plumbing ----------------
template <typename Args>
int launch(nb200_engine *e, void (*kern)(const Args), dim3 grid, dim3 block, size_t smem, const Args &args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = e ? e->stream : nullptr;
    cudaLaunchAttribute attr[1];
    if (e && e->use_pdl) {
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr; cfg.numAttrs = 1;
    }
    // the 48 KB default covers static + dynamic shared memory together: a dynamic size just under 48 KB needs the opt-in too
    if (smem > 40 * 1024) {
        cudaFuncAttributes fa;
        CK(cudaFuncGetAttributes(&fa, (const void *)kern));
        if (smem + fa.sharedSizeBytes > 48 * 1024) CK(cudaFuncSetAttribute((const void *)kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    if (e && e->prof_on) {
        nb200_engine::ProfRec r{e->prof_tag, nullptr, nullptr};
        CK(cudaEventCreate(&r.a)); CK(cudaEventCreate(&r.b));
        CK(cudaEventRecord(r.a, e->stream));
        CK(cudaLaunchKernelEx(&cfg, kern, args));
        CK(cudaEventRecord(r.b, e->stream));
        e->prof.push_back(r);
    } else {
        CK(cudaLaunchKernelEx(&cfg, kern, args));
    }
    if (e) e->launches++;
    return 0;
}

typedef void (*MatvecKern)(const MatvecArgs);

template <int QUANT, int EPI, bool TP>
MatvecKern pick_matvec(int rb, int lpg) {
    // constexpr: F32 / Q4K must not instantiate the Q80 (RB, LPG) table (92 kernels no selection could reach)
    if constexpr (QUANT == 0x80) {
#define NB_PICK(RB_, L_) if (rb == RB_ && lpg == L_) return k_matvec<QUANT, EPI, RB_, L_, TP>;
        if constexpr (EPI != EPI_SWIGLU) { NB_PICK(1, 2) NB_PICK(1, 4) NB_PICK(1, 8) NB_PICK(1, 16) }      // SwiGLU pairs rows: RB even
        NB_PICK(2, 2) NB_PICK(2, 4) NB_PICK(2, 8) NB_PICK(2, 16)
        NB_PICK(4, 2) NB_PICK(4, 4) NB_PICK(4, 8) NB_PICK(4, 16)
#undef NB_PICK
        return nullptr;
    } else {
        if (rb == 2) return k_matvec<QUANT, EPI, 2, 8, TP>;
        return k_matvec<QUANT, EPI, 4, 8, TP>;
    }
}

template <int EPI>
MatvecKern pick_matvec_q(uint32_t quant, int rb, int lpg, bool tp) {
    if (tp && EPI != EPI_STORE) {      // the tensor-parallel variants (STORE is an op-level kernel only)
        constexpr int E2 = (EPI == EPI_STORE) ? EPI_RESID : EPI;
        if (quant == 0x00u) return pick_matvec<0x00, E2, true>(rb, lpg);
        if (quant == 0x80u) return pick_matvec<0x80, E2, true>(rb, lpg);
        return pick_matvec<0x42, E2, true>(rb, lpg);
    }
    if (quant == 0x00u) return pick_matvec<0x00, EPI, false>(rb, lpg);
    if (quant == 0x80u) return pick_matvec<0x80, EPI, false>(rb, lpg);
    return pick_matvec<0x42, EPI, false>(rb, lpg);
}

int grid_mult() {
    static int m = -1;
    if (m < 0) { const char *s = getenv("NB200_GRID_MULT"); m = s ? atoi(s) : 1; if (m < 1) m = 1; }
    return m;
}

// one fused matvec launch
int run_matvec(nb200_engine *e, int epi, const Mat &m, MatvecArgs a, bool norm, int num_sms) {
    const Dims &d = a.d;
    a.w = m.w; a.w_aux = m.aux; a.rows = m.rows; a.n = m.n;
    const uint32_t smem = act_smem_bytes(d.quant, m.n, d.gs ? d.gs : 1);
    (void)norm;
    if (d.quant == 0x00u && d.exact) {
        MatvecKern k = nullptr;
        switch (epi) {
            case EPI_STORE: k = k_matvec_f32_exact<EPI_STORE>; break;
            case EPI_QKV: k = k_matvec_f32_exact<EPI_QKV>; break;
            case EPI_RESID: k = k_matvec_f32_exact<EPI_RESID>; break;
            case EPI_SWIGLU: k = k_matvec_f32_exact<EPI_SWIGLU>; break;
            default: break;     // CLS keeps the fast kernel below (argmax fused); exactness handled by caller
        }
        if (k) {
            const uint32_t units = (epi == EPI_SWIGLU) ? m.rows / 2 : m.rows;
            const uint32_t grid = (units + 255) / 256;
            return launch<MatvecArgs>(e, k, dim3(grid), dim3(256), smem, a);
        }
    }
    const uint32_t total_warps = (uint32_t)num_sms * grid_mult() * kWarps;
    // 4 rows per block once there are >= 2 waves of such blocks, else 2.  (Measured on Qwen3-4B W1|W3, 19456 rows: RB=4 372
    // tok/s vs RB=2 359, although RB=4 leaves the third wave almost empty.)
    int rb = (m.rows >= total_warps * 8) ? 4 : 2;
    // few long rows (O / W2 of the larger models): one row per warp keeps every warp busy, 4 tiles in flight each
    if (d.quant == 0x80u && epi != EPI_SWIGLU && m.rows <= total_warps && m.n >= 2048 && !getenv("NB200_NO_RB1")) rb = 1;
    // NB200_MATVEC_RB=1|2|4 forces the row block (tests): RB = 1 exists for Q80 matrices other than W1|W3 only, the others keep 2
    if (const char *f = getenv("NB200_MATVEC_RB")) {
        const int want = atoi(f);
        if (want == 2 || want == 4) rb = want;
        else if (want == 1) rb = (d.quant == 0x80u && epi != EPI_SWIGLU) ? 1 : 2;
    }
    const int lpg = (d.quant == 0x80u) ? (int)(d.gs / 16) : 8;
    MatvecKern k = nullptr;
    const bool tp = a.tp.size > 1;
    switch (epi) {
        case EPI_STORE: k = pick_matvec_q<EPI_STORE>(d.quant, rb, lpg, tp); break;
        case EPI_QKV: k = pick_matvec_q<EPI_QKV>(d.quant, rb, lpg, tp); break;
        case EPI_RESID: k = pick_matvec_q<EPI_RESID>(d.quant, rb, lpg, tp); break;
        case EPI_SWIGLU: k = pick_matvec_q<EPI_SWIGLU>(d.quant, rb, lpg, tp); break;
        case EPI_CLS: k = pick_matvec_q<EPI_CLS>(d.quant, rb, lpg, tp); break;
    }
    if (!k) return fail(NB200_EINVAL, "no matvec kernel for quant=0x%x gs=%u", d.quant, d.gs);
    const uint32_t nblocks = (m.rows + rb - 1) / rb;
    uint32_t grid = (nblocks + kWarps - 1) / kWarps;
    const uint32_t cap = (uint32_t)num_sms * grid_mult();
    if (grid > cap) grid = cap;
    if (epi == EPI_CLS && e) { if (grid > e->cls_grid) grid = e->cls_grid; }
    if (e) e->mv_mask |= 1u << (3 * epi + (rb == 1 ? 0 : rb == 2 ? 1 : 2));
    return launch<MatvecArgs>(e, k, dim3(grid), dim3(kThreads), smem, a);
}

MatvecArgs base_args(nb200_engine *e) {
    MatvecArgs a{};
    a.d = e->d; a.st = e->st;
    return a;
}

// Exchange ids within one token: layer l publishes attention = 4l+1, O = 4l+2, W1|W3 = 4l+3, W2 = 4l+4; the classifier's
// argmax all-gather is 4L+1.  Each kernel waits for the exchange that produced its input vector.
TpArgs tp_args(nb200_engine *e, uint32_t wait_ph, uint32_t signal_ph, uint32_t row_base, uint32_t out_off) {
    TpArgs t{};
    if (e->tp_size <= 1) return t;
    t.size = e->tp_size; t.rank = e->tp_rank; t.wait_ph = wait_ph; t.signal_ph = signal_ph; t.nph = 4 * e->d.L + 1;
    t.row_base = row_base; t.out_off = out_off;
    for (uint32_t p = 0; p < e->tp_size; p++) t.peer[p] = e->tp_peer[p];
    return t;
}

int run_embed(nb200_engine *e) {
    EmbedArgs a{};
    a.w = e->emb.w; a.w_aux = e->emb.aux; a.x = e->x; a.ids = e->ids_dev; a.st = e->st; a.d = e->d; a.ll = e->tp_size > 1;
    e->prof_tag = 0;
    return launch<EmbedArgs>(e, k_embed, dim3(1), dim3(256), 0, a);
}

int run_layer(nb200_engine *e, uint32_t l) {
    const Dims &d = e->d;
    const size_t kvl = (size_t)d.KV * d.max_seq * d.hd;
    int r;
    {   // F1: rmsnorm + quantise + QKV matvec + KV store
        MatvecArgs a = base_args(e);
        a.src = e->x; a.gain = e->norm_attn + (size_t)l * d.E;
        a.out = e->q; a.out_k = e->kraw; a.out_v = e->vc + l * kvl;
        a.dump_codes = e->dump_codes; a.dump_scales = e->dump_scales;
        a.tp = tp_args(e, 4 * l, 0, 0, 0);
        e->prof_tag = 1;
        if ((r = run_matvec(e, EPI_QKV, e->qkv[l], a, true, e->num_sms))) return r;
    }
    if (e->lora.active) {   // q/k/v LoRA branches on xb = rmsnorm(x)*gain, added before RoPE (infer.c:792-808)
        const uint32_t rk = e->lora.rank;
        LoraAArgs la{};
        la.src = e->x; la.gain = e->norm_attn + (size_t)l * d.E; la.n = d.E; la.nmat = 3; la.rank = rk; la.t = e->lora.t; la.exact = d.exact;
        for (int m = 0; m < 3; m++) la.A[m] = e->lora.a[m] + (size_t)l * rk * d.E;
        if ((r = launch<LoraAArgs>(e, k_lora_a, dim3((3 * rk + kWarps - 1) / kWarps), dim3(kThreads), 3 * d.E * 4, la))) return r;
        LoraBArgs lb{};
        lb.t = e->lora.t; lb.nmat = 3; lb.rank = rk; lb.scale = (float)e->lora.alpha / (float)rk;
        lb.rows[0] = d.q_dim; lb.rows[1] = d.kv_dim; lb.rows[2] = d.kv_dim;
        lb.B[0] = e->lora.b[0] + (size_t)l * d.q_dim * rk; lb.B[1] = e->lora.b[1] + (size_t)l * d.kv_dim * rk; lb.B[2] = e->lora.b[2] + (size_t)l * d.kv_dim * rk;
        lb.dst[0] = e->q; lb.dst[1] = e->kraw; lb.dst[2] = nullptr; lb.vcache = e->vc + l * kvl; lb.store = 0; lb.st = e->st; lb.d = d;
        if ((r = launch<LoraBArgs>(e, k_lora_b, dim3((d.q_dim + 2 * d.kv_dim + 255) / 256), dim3(256), 0, lb))) return r;
    }
    e->prof_tag = 2;
    if (!d.exact) {   // F2: head-norm + RoPE + split-KV attention
        AttnArgs a{};
        a.q = e->q; a.kraw = e->kraw; a.kc = e->kc + l * kvl; a.vc = e->vc + l * kvl;
        a.qnorm = e->qnorm ? e->qnorm + (size_t)l * d.hd : nullptr;
        a.knorm = e->knorm ? e->knorm + (size_t)l * d.hd : nullptr;
        a.rope_cos = e->rope_cos; a.rope_sin = e->rope_sin; a.xba = e->xba;
        a.ws_m = e->ws_m; a.ws_l = e->ws_l; a.ws_acc = e->ws_acc; a.ticket = e->tickets;
        a.st = e->st; a.nsplit_max = e->nsplit_max; a.chunk_cap = e->chunk_cap; a.d = d;
        a.dbg = (l == d.L / 2) ? e->attn_dbg : nullptr;
        void (*kern)(const AttnArgs) = k_attention;
        uint32_t smem = e->attn_smem;
        const bool tp = e->tp_size > 1;
        if (tp) a.tp = tp_args(e, 0, 4 * l + 1, e->tp_rank * d.q_dim, e->tp_off_xba);
        if (d.hd <= 128 && (d.arch != 3u || (d.hd & (d.hd - 1)) == 0) && (tp || !getenv("NB200_GENERIC_ATTN"))) {
            switch (d.kv_mul) {
                case 1: kern = tp ? k_attention_fast<1, true> : k_attention_fast<1>; break;
                case 2: kern = tp ? k_attention_fast<2, true> : k_attention_fast<2>; break;
                case 4: kern = tp ? k_attention_fast<4, true> : k_attention_fast<4>; break;
                case 8: kern = tp ? k_attention_fast<8, true> : k_attention_fast<8>; break;
                default: break;
            }
            if (kern != k_attention) smem = attn_fast_smem_floats(d.kv_mul, d.hd, e->chunk_cap, e->nsplit_max, kWarps) * 4u;
        }
        e->attn_kind = (kern == k_attention) ? 2u : (3u | (d.kv_mul << 8));
        if ((r = launch<AttnArgs>(e, kern, dim3(e->nsplit_max, d.KV), dim3(kern != k_attention ? kThreads : kAttnThreads), smem, a))) return r;
    } else {
        AttnExactArgs a{};
        a.q = e->q; a.kraw = e->kraw; a.kc = e->kc + l * kvl; a.vc = e->vc + l * kvl;
        a.qnorm = e->qnorm ? e->qnorm + (size_t)l * d.hd : nullptr;
        a.knorm = e->knorm ? e->knorm + (size_t)l * d.hd : nullptr;
        a.rope_cos = e->rope_cos; a.rope_sin = e->rope_sin; a.xba = e->xba; a.att = e->att_exact; a.st = e->st; a.d = d;
        e->attn_kind = 1u;
        if ((r = launch<AttnExactArgs>(e, k_attention_exact, dim3(d.H), dim3(kAttnThreads), 2 * d.hd * 4, a))) return r;
    }
    if (e->lora.active) {   // o branch on the attention output; added to the O result before the residual (infer.c:898-903)
        const uint32_t rk = e->lora.rank;
        LoraAArgs la{};
        la.src = e->xba; la.gain = nullptr; la.n = d.q_dim; la.nmat = 1; la.rank = rk; la.t = e->lora.t + 3 * rk; la.exact = d.exact;
        la.A[0] = e->lora.a[3] + (size_t)l * rk * d.q_dim;
        e->prof_tag = 3;
        if ((r = launch<LoraAArgs>(e, k_lora_a, dim3((rk + kWarps - 1) / kWarps), dim3(kThreads), 3 * d.q_dim * 4, la))) return r;
        LoraBArgs lb{};
        lb.t = e->lora.t + 3 * rk; lb.nmat = 1; lb.rank = rk; lb.scale = (float)e->lora.alpha / (float)rk;
        lb.rows[0] = d.E; lb.B[0] = e->lora.b[3] + (size_t)l * d.E * rk; lb.dst[0] = e->lora.o1; lb.store = 1; lb.st = e->st; lb.d = d;
        if ((r = launch<LoraBArgs>(e, k_lora_b, dim3((d.E + 255) / 256), dim3(256), 0, lb))) return r;
    }
    {   // F3: quantise(xba) + O matvec + residual
        MatvecArgs a = base_args(e);
        a.src = e->xba; a.gain = nullptr; a.out = e->x;
        a.lora_add = e->lora.active ? e->lora.o1 : nullptr;
        a.tp = tp_args(e, 4 * l + 1, 4 * l + 2, e->tp_rank * e->wo[l].rows, e->tp_off_x);
        e->prof_tag = 3;
        if ((r = run_matvec(e, EPI_RESID, e->wo[l], a, false, e->num_sms))) return r;
    }
    {   // F4: rmsnorm + quantise + W1|W3 matvec + SwiGLU
        MatvecArgs a = base_args(e);
        a.src = e->x; a.gain = e->norm_ffn + (size_t)l * d.E; a.out = e->hb;
        a.tp = tp_args(e, 4 * l + 2, 4 * l + 3, e->tp_rank * (e->w13[l].rows / 2), e->tp_off_hb);
        e->prof_tag = 4;
        if ((r = run_matvec(e, EPI_SWIGLU, e->w13[l], a, true, e->num_sms))) return r;
    }
    {   // F5: quantise(hb) + W2 matvec + residual
        MatvecArgs a = base_args(e);
        a.src = e->hb; a.gain = nullptr; a.out = e->x;
        a.tp = tp_args(e, 4 * l + 3, 4 * l + 4, e->tp_rank * e->w2[l].rows, e->tp_off_x);
        e->prof_tag = 5;
        if ((r = run_matvec(e, EPI_RESID, e->w2[l], a, false, e->num_sms))) return r;
    }
    return 0;
}

int run_classifier(nb200_engine *e) {
    e->prof_tag = 6;
    MatvecArgs a = base_args(e);
    a.src = e->x; a.gain = e->norm_final; a.out = e->logits;
    if (e->d.quant == 0x00u && e->d.exact) {
        int r = run_matvec(e, EPI_STORE, e->cls, a, true, e->num_sms);
        if (r) return r;
        FinalizeArgs f{e->logits, e->d.V, e->seen, e->seen, e->ids_dev, e->st};
        return launch<FinalizeArgs>(e, k_cls_finalize, dim3(1), dim3(1024), 0, f);
    }
    a.st_rw = e->st; a.seen = e->seen; a.seen_rw = e->seen; a.cls_val = e->cls_val; a.cls_idx = e->cls_idx; a.ids = e->ids_dev;
    a.tp = tp_args(e, 4 * e->d.L, 4 * e->d.L + 1, e->tp_rank * e->cls.rows, 0);
    return run_matvec(e, EPI_CLS, e->cls, a, true, e->num_sms);
}

int run_token(nb200_engine *e) {
    int r;
    if ((r = run_embed(e))) return r;
    for (uint32_t l = 0; l < e->d.L; l++) if ((r = run_layer(e, l))) return r;
    return run_classifier(e);
}

// n_steps tokens in ONE cooperative launch of the streaming kernel
int launch_stream(nb200_engine *e, uint32_t n_steps) {
    if (n_steps == 0) return 0;
    StreamArgs g = e->sa;
    g.n_steps = n_steps; g.trace = e->trace_dev;
    g.epoch_base = e->st_epoch;
    e->st_epoch += n_steps * 5u * e->d.L;
    CK(cudaMemsetAsync(e->bar, 0, sizeof(unsigned int), e->stream));
    void *params[] = {&g};
    CK(cudaLaunchCooperativeKernel(e->st_kern, dim3(e->st_grid), dim3(kThreads), params, e->st_smem, e->stream));
    e->launches++;
    return 0;
}

int launch_token(nb200_engine *e) {
    if (e->tp_size > 1 && !e->tp_attached) return fail(NB200_EINVAL, "tensor-parallel engine: attach the peer ranks first (nb200_tp_attach_*)");
    if (e->use_stream) return launch_stream(e, 1);
    if (e->graph) {
        CK(cudaGraphLaunch(e->graph, e->stream));
        e->launches += e->launches_per_token;
        return 0;
    }
    return run_token(e);
}

int capture_graph(nb200_engine *e) {
    cudaGraph_t g = nullptr;
    CK(cudaStreamBeginCapture(e->stream, cudaStreamCaptureModeThreadLocal));
    const uint64_t before = e->launches;
    int r = run_token(e);
    cudaError_t ce = cudaStreamEndCapture(e->stream, &g);
    e->launches_per_token = (uint32_t)(e->launches - before);
    e->launches = before;
    if (r) { if (g) cudaGraphDestroy(g); cudaGetLastError(); return r; }     // the invalidated capture must not reach the next caller's error check
    if (ce != cudaSuccess) return fail(NB200_ECUDA, "graph capture failed: %s", cudaGetErrorString(ce));
    ce = cudaGraphInstantiate(&e->graph, g, 0);
    cudaGraphDestroy(g);
    if (ce != cudaSuccess) { e->graph = nullptr; return fail(NB200_ECUDA, "graph instantiate failed: %s", cudaGetErrorString(ce)); }
    return 0;
}

// ---------------- uploads ----------------
int upload_rows(void *dst, size_t dpitch, const uint8_t *src, size_t spitch, size_t width, size_t height) {
    CK(cudaMemcpy2D(dst, dpitch, src, spitch, width, height, cudaMemcpyHostToDevice));
    return 0;
}

struct Q80Src { const uint8_t *q, *s; };

int alloc_mat(nb200_engine *e, Mat &m, uint32_t rows, uint32_t n) {
    const Dims &d = e->d;
    m.rows = rows; m.n = n;
    size_t wb, ab;
    if (d.quant == 0x00u) { wb = (size_t)rows * n * 4; ab = 0; }
    else if (d.quant == 0x80u) { wb = (size_t)rows * n; ab = (size_t)rows * (n / d.gs) * 4; }
    else { wb = (size_t)rows * n / 2; ab = (size_t)rows * (n / 256) * 20; }
    DM(m.w, wb + 64);
    if (ab) DM(m.aux, ab + 64);
    e->weight_bytes += wb + ab;
    return 0;
}

// copy `srows` source rows into the fused matrix at dst_row = off + i*stride
int put_rows(nb200_engine *e, Mat &m, const uint8_t *w, const uint8_t *aux, uint32_t srows, uint32_t off, uint32_t stride,
             uint8_t *staging) {
    const Dims &d = e->d;
    const uint32_t n = m.n;
    if (d.quant == 0x00u) {
        return upload_rows((uint8_t *)m.w + (size_t)off * n * 4, (size_t)stride * n * 4, w, (size_t)n * 4, (size_t)n * 4, srows);
    } else if (d.quant == 0x80u) {
        const uint32_t G = n / d.gs;
        int r = upload_rows((uint8_t *)m.w + (size_t)off * n, (size_t)stride * n, w, n, n, srows);
        if (r) return r;
        return upload_rows((uint8_t *)m.aux + (size_t)off * G * 4, (size_t)stride * G * 4, aux, (size_t)G * 4, (size_t)G * 4, srows);
    } else {
        const uint32_t bpr = n / 256;
        const uint64_t nblocks = (uint64_t)srows * bpr;
        CK(cudaMemcpy(staging, w, nblocks * 160, cudaMemcpyHostToDevice));
        const uint64_t total = nblocks * 37;
        const uint32_t grid = (uint32_t)((total + 255) / 256 > 4096 ? 4096 : (total + 255) / 256);
        k_q4k_split<<<grid, 256>>>(staging, nblocks, bpr, (uint8_t *)m.w, (uint8_t *)m.aux, off, stride);
        CK(cudaGetLastError());
        CK(cudaDeviceSynchronize());
        return 0;
    }
}

// ---------------- streaming path: per-CTA tile-ordered weight stream + schedule (stream.cuh) ----------------
uint32_t env_u32(const char *name, uint32_t dflt) { const char *s = getenv(name); return (s && *s) ? (uint32_t)strtoul(s, nullptr, 10) : dflt; }

// returns 0 and sets e->use_stream when the model fits the streaming kernel; 0 without setting it otherwise
int setup_stream(nb200_engine *e) {
    const Dims &d = e->d;
    if (d.exact || e->tp_size > 1) return 0;
    StreamKern k = pick_stream(d);
    if (!k) return 0;
    uint32_t maxn = d.E; if (d.q_dim > maxn) maxn = d.q_dim; if (d.F > maxn) maxn = d.F;
    if (maxn > st_prep_max_n(d.quant, d.gs)) return 0;
    if (d.quant == 0x80u && (d.E % 16 || d.q_dim % 16 || d.F % 16)) return 0;
    int coop = 0;
    CK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, e->device));
    if (!coop) return 0;
    const uint32_t NC = (uint32_t)e->num_sms;
    if (d.KV > NC || (d.E + NC - 1) / NC > (uint32_t)kStOwnMax) return 0;
    const uint32_t L = d.L;

    StreamArgs &g = e->sa;
    memset(&g, 0, sizeof g);
    struct KM { uint32_t rows, n, unit; } km[5] = {
        {d.q_dim + 2 * d.kv_dim, d.E, 1}, {d.E, d.q_dim, 1}, {2 * d.F, d.E, 2}, {d.E, d.F, 1}, {d.V, d.E, 1}};
    uint32_t main_b[5], aux_b[5], unit_b_max = 0;
    for (int i = 0; i < 5; i++) {
        const uint32_t n = km[i].n;
        main_b[i] = (d.quant == 0x00u) ? n * 4u : (d.quant == 0x80u) ? n : n / 2u;
        aux_b[i] = (d.quant == 0x00u) ? 0u : (d.quant == 0x80u) ? (n / d.gs) * 4u : (n / 256u) * 20u;
        StKind &sk = g.kind[i];
        sk.units = km[i].rows / km[i].unit; sk.unit_rows = km[i].unit; sk.n = n;
        sk.row_stride = main_b[i] + 16u;
        sk.aux_stride = (d.quant == 0x80u) ? ((n / d.gs) | 1u) * 4u : aux_b[i];
        const uint32_t ub = km[i].unit * (sk.row_stride + sk.aux_stride);
        if (ub > unit_b_max) unit_b_max = ub;
    }
    // shared-memory plan: [activation operand 0 | activation operand 1 | embedding row | attention workspace | ring].  Nothing aliases, so a
    // phase never waits for the slowest warp of the previous one before it writes its operand.  The ring stage is 16 KB by default and
    // shrinks in 1 KB steps (never below one row unit of the longest row) until kStSegTiles + 4 stages fit beside the fixed regions.
    auto al = [](uint32_t v) { return (v + 127u) & ~127u; };
    const uint32_t nsplit_max = e->nsplit_max;          // num_sms / kv heads (<= 64), as the multi-kernel path
    const uint32_t act_b = al(act_region_bytes(d.quant, maxn, d.gs ? d.gs : 1));
    g.off_act = 0; g.off_act2 = act_b; g.off_xs = 2 * act_b; g.off_attn = g.off_xs + al(d.E * 4u);
    int max_optin = 0;
    CK(cudaDeviceGetAttribute(&max_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, e->device));
    cudaFuncAttributes fattr;
    CK(cudaFuncGetAttributes(&fattr, (const void *)k));
    const uint32_t static_smem = al((uint32_t)fattr.sharedSizeBytes);   // mbarriers, row ranges, residual rows, reduction scratch
    const uint32_t min_stage = (unit_b_max + 16u + 1023u) & ~1023u;
    uint32_t stage_bytes = env_u32("NB200_STAGE_KB", 16) * 1024u;
    if (stage_bytes < min_stage) stage_bytes = min_stage;
    const uint32_t nst_cap = env_u32("NB200_STAGES", kStMaxStages) < (uint32_t)kStMaxStages ? env_u32("NB200_STAGES", kStMaxStages) : (uint32_t)kStMaxStages;
    uint32_t kv_rows = 0, region0 = 0, nst = 0;
    for (;; stage_bytes -= 1024u) {
        kv_rows = (stage_bytes / (2u * d.hd * 4u)) & ~3u;
        if (kv_rows < 4) return 0;
        const uint32_t attn_b = al(st_attn_smem_floats(d.kv_mul, d.hd, nsplit_max, (uint32_t)kStSegTiles * kv_rows) * 4u);
        region0 = g.off_attn + attn_b;
        nst = (uint32_t)max_optin > static_smem + region0 ? ((uint32_t)max_optin - static_smem - region0) / stage_bytes : 0u;
        if (nst > nst_cap) nst = nst_cap;
        if (nst >= (uint32_t)kStSegTiles + 4u) break;   // an attention segment keeps kStSegTiles tiles resident while the next ones arrive
        if (stage_bytes < min_stage + 1024u) return 0;
    }
    g.off_ring = region0;
    uint64_t off = 0;
    uint32_t ntl[5];
    for (int i = 0; i < 5; i++) {
        StKind &sk = g.kind[i];
        const uint32_t rowb = sk.row_stride + sk.aux_stride;
        const uint32_t max_rows = ((sk.units + NC - 1) / NC) * sk.unit_rows;
        uint32_t T = (stage_bytes - 16u) / rowb;
        T -= T % sk.unit_rows;
        if (T > max_rows) T = max_rows;
        if (T < sk.unit_rows) return 0;
        // many rows per CTA: throughput mode, every tile is consumed by one warp -- small tiles so that all 15 warps have one.
        // 64 rows: measured on H100 against 16 / 32 (Nano-168M Q80 1519 vs 1473 / 1443 tok/s, Qwen3-0.6B Q4K 892 vs 879 / 886)
        sk.owned = (max_rows >= env_u32("NB200_OWNED_ROWS", 64) || (uint64_t)max_rows * rowb >= (uint64_t)env_u32("NB200_OWNED_KB", 32) * 1024u) ? 1u : 0u;
        if (sk.owned) {
            uint32_t t2 = (max_rows + kConsWarps - 1) / kConsWarps;
            t2 = ((t2 + sk.unit_rows - 1) / sk.unit_rows) * sk.unit_rows;
            if (t2 < 2u) t2 = 2u;
            if (t2 < T) T = t2;
        }
        sk.tile_rows = T;
        sk.tile_stride = (T * rowb + 15u) & ~15u;
        ntl[i] = (max_rows + T - 1) / T;
        if (i == SK_CLS) off = 0;
        sk.off = off;
        off += (uint64_t)ntl[i] * sk.tile_stride;
        off = (off + 127u) & ~(uint64_t)127u;
        if (i == SK_W2) g.layer_stride = off;
    }
    g.cls_off = (uint64_t)L * g.layer_stride;
    g.kind[SK_CLS].off = 0;
    g.cta_stride = (g.cls_off + (uint64_t)ntl[SK_CLS] * g.kind[SK_CLS].tile_stride + 127u) & ~(uint64_t)127u;

    const uint32_t smem = region0 + nst * stage_bytes;
    cudaError_t ce = cudaFuncSetAttribute((const void *)k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    int occ = 0;
    if (ce == cudaSuccess) ce = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, (const void *)k, kThreads, smem);
    if (ce != cudaSuccess || occ < 1) { cudaGetLastError(); return 0; }

    // device objects: the stream copy of the weights
    uint8_t *stream = nullptr;
    const uint64_t total = g.cta_stride * NC + 256;
    DM(stream, total);
    CK(cudaMemset(stream, 0, total));
    auto build = [&](int ki, const Mat &m, uint64_t base_off) -> int {
        const StKind &sk = g.kind[ki];
        uint32_t gx = ((sk.units + NC - 1) / NC) * sk.unit_rows; if (gx > 1024) gx = 1024; if (gx < 1) gx = 1;
        CK(stream_build_launch((const uint8_t *)m.w, (const uint8_t *)m.aux, main_b[ki], aux_b[ki], sk, stream, g.cta_stride, base_off, gx, NC));
        return 0;
    };
    int r;
    for (uint32_t l = 0; l < L; l++) {
        const uint64_t lb = (uint64_t)l * g.layer_stride;
        if ((r = build(SK_QKV, e->qkv[l], lb)) || (r = build(SK_O, e->wo[l], lb)) || (r = build(SK_W13, e->w13[l], lb)) || (r = build(SK_W2, e->w2[l], lb))) return r;
    }
    if ((r = build(SK_CLS, e->cls, g.cls_off))) return r;
    CK(cudaDeviceSynchronize());
    e->stream_bytes = total;

    if (!e->bar) { DM(e->bar, 64); CK(cudaMemset(e->bar, 0, 64)); }
    CK(cudaHostAlloc(&e->st_err_host, 64, cudaHostAllocMapped));
    memset(e->st_err_host, 0, 64);
    CK(cudaHostGetDevicePointer((void **)&e->st_err_dev, e->st_err_host, 0));

    g.stream = stream; g.nstages = nst; g.stage_bytes = stage_bytes; g.kv_tile_rows = kv_rows;
    g.kv_tile_magic = (uint32_t)((0x100000000ull + kv_rows - 1) / kv_rows);
    g.g_attn = e->norm_attn; g.g_ffn = e->norm_ffn; g.g_final = e->norm_final;
    g.qnorm = e->qnorm; g.knorm = e->knorm; g.rope_cos = e->rope_cos; g.rope_sin = e->rope_sin;
    g.emb_w = e->emb.w; g.emb_aux = e->emb.aux;
    g.logits = e->logits; g.kc = e->kc; g.vc = e->vc;
    {   // activation exchange words {value, epoch}, zeroed once: epoch 0 is never handed out
        auto words = [&](unsigned long long *&p, size_t n) -> int { DM(p, n * 8 + 256); CK(cudaMemset(p, 0, n * 8 + 256)); return 0; };
        const uint32_t ns[3] = {d.E, d.q_dim, d.F};
        if ((r = words(g.xq, (size_t)d.q_dim + 2 * d.kv_dim))) return r;
        for (int i = 0; i < 3; i++) {
            g.rs[i] = ((ns[i] + 31u) & ~31u) + 32u;                 // replicas 256 bytes apart at least: different L2 slices
            if ((r = words(g.xv[i], (size_t)g.rs[i] * kStRep))) return r;
        }
        if ((r = words(g.xws, (size_t)d.KV * nsplit_max * d.kv_mul * (d.hd + 2)))) return r;
    }
    g.cls_val = e->cls_val; g.cls_idx = e->cls_idx;
    g.st = e->st; g.ids = e->ids_dev; g.seen = e->seen; g.bar = e->bar; g.err = e->st_err_dev;
    g.n_steps = 1; g.nsplit_max = nsplit_max;
    uint32_t ct = 32768u / (d.hd * 8u); ct &= ~7u; if (ct < 32) ct = 32;      // measured: ~32 KB of K+V per (kv head, split) item
    g.chunk_target = env_u32("NB200_ATTN_CHUNK", ct);
    g.ablate = env_u32("NB200_ABLATE", 0);
    if (g.chunk_target < 8) g.chunk_target = 8;
    g.d = d;
    e->st_kern = (const void *)k; e->st_smem = smem; e->st_grid = NC; e->use_stream = true; e->launches_per_token = 1;
    return 0;
}

}  // namespace

// =================================================================================================
// C-ABI
// =================================================================================================
extern "C" {

const char *nb200_last_error(void) { return g_err.c_str(); }

int nb200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

void nb200_engine_destroy(nb200_engine *e) {
    if (!e) return;
    cudaSetDevice(e->device);
    if (e->stream) cudaStreamSynchronize(e->stream);
    if (e->graph) cudaGraphExecDestroy(e->graph);
    for (void *p : e->tp_ipc_opened) cudaIpcCloseMemHandle(p);
    for (void *p : e->allocs) cudaFree(p);
    if (e->st_host) cudaFreeHost(e->st_host);
    if (e->samp_host) cudaFreeHost(e->samp_host);
    if (e->tok_host) cudaFreeHost(e->tok_host);
    if (e->stream) cudaStreamDestroy(e->stream);
    delete e;
}

static int finish_paths(nb200_engine *e);
static int calibrate_paths(nb200_engine *e);
static int push_state(nb200_engine *e, uint32_t pos, uint32_t causal, uint32_t n_prompt, uint32_t advance, float penalty,
                      uint32_t token, uint32_t use_token);

// Positions [0, pos_limit) are the ones a call may run: the device RoPE table holds min(block_size, max_seq) rows, and the
// kernels index it by position unguarded.  Rows from block_size to max_seq of a longer context stay zero.
static uint32_t pos_limit(const Dims &d) { return d.block_size < d.max_seq ? d.block_size : d.max_seq; }

static int create_impl(nb200_engine **out, const uint8_t *img, uint64_t image_bytes, uint32_t max_seq_len, int device,
                       uint32_t flags, uint32_t tp_rank, uint32_t tp_size) {
    if (!out || !img || image_bytes < 260 || max_seq_len == 0) return fail(NB200_EINVAL, "bad arguments");
    if (tp_size < 1 || tp_size > (uint32_t)kTpMax || tp_rank >= tp_size) return fail(NB200_EINVAL, "bad tensor-parallel rank/size");
    *out = nullptr;
    if (nb200_device_count() <= 0) return fail(NB200_ENODEV, "no CUDA device: nano_b200 has no CPU path");
    if (rd_u32(img) != 0x42443453u || rd_u32(img + 4) != 0x55524c4du) return fail(NB200_EINVAL, "bad magic (not a BD4SURLM file)");
    CK(cudaSetDevice(device));
    {   // hosts that reach the engine through the reference API (infer.h has no flags argument) use the environment
        const char *ex = getenv("NB200_EXACT");
        if (ex && atoi(ex) != 0) flags |= NB200_FLAG_EXACT;
    }
    nb200_engine *e = new nb200_engine();
    struct Guard { nb200_engine *e; bool ok = false; ~Guard() { if (!ok) nb200_engine_destroy(e); } } guard{e};
    e->device = device; e->flags = flags; e->tp_rank = tp_rank; e->tp_size = tp_size;
    e->use_pdl = !(flags & NB200_FLAG_NO_PDL);
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    e->num_sms = prop.multiProcessorCount;
    CK(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));

    // ---- header (infer.c:231-256) ----
    Dims &d = e->d;
    d.arch = rd_u32(img + 16);
    d.block_size = rd_u32(img + 24); d.V = rd_u32(img + 28); d.L = rd_u32(img + 32); d.E = rd_u32(img + 36);
    d.H = rd_u32(img + 40); d.KV = rd_u32(img + 44); d.F = rd_u32(img + 48);
    const uint32_t tied = rd_u32(img + 52);
    uint32_t head_dim = rd_u32(img + 56);
    const uint32_t qt = rd_u32(img + 60);
    d.quant = (qt == 0x00u || qt == 0x80u || qt == 0x42u) ? qt : 0x80u;
    d.gs = rd_u32(img + 64);
    d.exact = (flags & NB200_FLAG_EXACT) ? 1u : 0u;
    if (!d.L || !d.E || !d.H || !d.KV || !d.F || !d.V || d.H % d.KV) return fail(NB200_EINVAL, "bad model dimensions");
    if (d.arch != 3u) head_dim = d.E / d.H;
    d.hd = head_dim;
    d.q_dim = (d.arch == 3u) ? d.hd * d.H : d.E;
    d.kv_dim = (d.arch == 3u) ? d.hd * d.KV : (d.E * d.KV) / d.H;
    d.kv_mul = d.H / d.KV;
    d.max_seq = max_seq_len;
    if (d.hd % 4 || d.hd > 512 || d.hd == 0) return fail(NB200_EINVAL, "head_dim %u unsupported (need multiple of 4, <= 512)", d.hd);
    if (d.quant == 0x00u && (d.E % 4 || d.q_dim % 4 || d.F % 4)) return fail(NB200_EINVAL, "F32 path needs dims %% 4 == 0");
    if (d.quant == 0x80u) {
        if (d.gs != 32 && d.gs != 64 && d.gs != 128 && d.gs != 256) return fail(NB200_EINVAL, "Q80 group size %u unsupported (32/64/128/256)", d.gs);
        if (d.E % d.gs || d.q_dim % d.gs || d.F % d.gs) return fail(NB200_EINVAL, "Q80 dims must be multiples of the group size");
    }
    if (d.quant == 0x42u && (d.E % 256 || d.q_dim % 256 || d.F % 256))
        return fail(NB200_EINVAL, "Q4K needs n %% 256 == 0 (the reference's partial-block offset is wrong otherwise, tensor.c:307)");
    if (d.quant != 0x80u) d.gs = (d.quant == 0x42u) ? 32 : 1;
    e->g_H = d.H; e->g_KV = d.KV; e->g_q_dim = d.q_dim; e->g_kv_dim = d.kv_dim;
    const uint32_t T = tp_size;
    if (T > 1) {
        // row shards: whole kv-head groups for QKV/attention, contiguous row ranges for O / W1|W3 / W2 / classifier
        if (d.exact) return fail(NB200_EINVAL, "tensor parallel runs in fast mode only");
        if (d.KV % T || d.E % (2 * T) || d.F % T || d.V % T) return fail(NB200_EINVAL, "tensor parallel size %u does not divide kv heads / n_embd / n_hidden / vocab", T);
        if (d.hd > 128 || (d.arch == 3u && (d.hd & (d.hd - 1)) != 0)) return fail(NB200_EINVAL, "tensor parallel needs head_dim <= 128 (power of two for Qwen3)");
        const uint32_t kvm = d.H / d.KV;      // only these ratios have a tensor-parallel attention kernel (run_layer)
        if (kvm != 1 && kvm != 2 && kvm != 4 && kvm != 8) return fail(NB200_EINVAL, "tensor parallel needs n_head / n_kv_head in {1, 2, 4, 8} (got %u)", kvm);
    }

    // ---- parameter map (infer.c:100-217) ----
    const uint32_t tok_bytes = rd_u32(img + 256);
    const uint8_t *cur = img + 256 + tok_bytes;
    const uint8_t *end = img + image_bytes;
    const uint64_t L = d.L, E = d.E, V = d.V, F = d.F, QD = d.q_dim, KD = d.kv_dim;
    auto need = [&](uint64_t bytes) { return cur <= end && (uint64_t)(end - cur) >= bytes; };
    if (cur > end || !need((2 * L + 1) * E * 4)) return fail(NB200_EINVAL, "file truncated (norms)");
    DM(e->norm_attn, L * E * 4); DM(e->norm_ffn, L * E * 4); DM(e->norm_final, E * 4);
    CK(cudaMemcpy(e->norm_attn, cur, L * E * 4, cudaMemcpyHostToDevice)); cur += L * E * 4;
    CK(cudaMemcpy(e->norm_ffn, cur, L * E * 4, cudaMemcpyHostToDevice)); cur += L * E * 4;
    CK(cudaMemcpy(e->norm_final, cur, E * 4, cudaMemcpyHostToDevice)); cur += E * 4;

    const uint64_t rows[7] = {QD, KD, KD, E, F, E, F};
    const uint64_t cols[7] = {E, E, E, QD, E, F, E};
    // source pointers per tensor kind and layer
    std::vector<const uint8_t *> src_w[7], src_a[7];
    const uint8_t *emb_w = nullptr, *emb_a = nullptr;
    if (d.quant == 0x00u) {
        if (!need(V * E * 4)) return fail(NB200_EINVAL, "file truncated (embedding)");
        emb_w = cur; cur += V * E * 4;
        for (int t = 0; t < 7; t++) {
            if (!need(L * rows[t] * cols[t] * 4)) return fail(NB200_EINVAL, "file truncated (tensor %d)", t);
            for (uint64_t l = 0; l < L; l++) { src_w[t].push_back(cur); src_a[t].push_back(nullptr); cur += rows[t] * cols[t] * 4; }
        }
    } else if (d.quant == 0x80u) {
        auto take = [&](uint64_t each, const uint8_t *&w, const uint8_t *&a) {
            w = cur; cur += each; a = cur; cur += (each / d.gs) * 4;
        };
        if (!need(V * E + V * E / d.gs * 4)) return fail(NB200_EINVAL, "file truncated (embedding)");
        take(V * E, emb_w, emb_a);
        for (int t = 0; t < 7; t++) {
            const uint64_t each = rows[t] * cols[t];
            if (!need(L * (each + each / d.gs * 4))) return fail(NB200_EINVAL, "file truncated (tensor %d)", t);
            for (uint64_t l = 0; l < L; l++) { const uint8_t *w, *a; take(each, w, a); src_w[t].push_back(w); src_a[t].push_back(a); }
        }
    } else {
        auto frame = [&](const uint8_t *&blocks, uint64_t expect_blocks) -> int {
            if (!need(44)) return fail(NB200_EINVAL, "file truncated (Q4K frame)");
            const uint64_t total = rd_u64(cur);
            const uint32_t nblk = rd_u32(cur + 40);
            if (nblk != expect_blocks || total != 44 + (uint64_t)nblk * 160 || !need(total))
                return fail(NB200_EINVAL, "unexpected Q4K tensor frame (blocks %u, expected %llu)", nblk, (unsigned long long)expect_blocks);
            blocks = cur + 44; cur += total;
            return 0;
        };
        int r;
        if ((r = frame(emb_w, V * (E / 256)))) return r;
        for (int t = 0; t < 7; t++) {
            const uint8_t *blocks;
            const uint64_t per_layer = rows[t] * (cols[t] / 256);
            if ((r = frame(blocks, L * per_layer))) return r;
            for (uint64_t l = 0; l < L; l++) { src_w[t].push_back(blocks + l * per_layer * 160); src_a[t].push_back(nullptr); }
        }
    }
    if (d.arch == 2u) {                                 // Qwen2 biases: parsed, never applied (infer.c:175-179, 788-790)
        if (!need(L * (QD + 2 * KD) * 4)) return fail(NB200_EINVAL, "file truncated (Qwen2 biases)");
        cur += L * (QD + 2 * KD) * 4;
    }
    if (d.arch == 3u) {
        if (!need(2 * L * d.hd * 4)) return fail(NB200_EINVAL, "file truncated (q/k norm)");
        DM(e->qnorm, L * d.hd * 4); DM(e->knorm, L * d.hd * 4);
        CK(cudaMemcpy(e->qnorm, cur, L * d.hd * 4, cudaMemcpyHostToDevice)); cur += L * d.hd * 4;
        CK(cudaMemcpy(e->knorm, cur, L * d.hd * 4, cudaMemcpyHostToDevice)); cur += L * d.hd * 4;
    }
    {   // RoPE tables: rows [0, min(block_size, max_seq)) are the only ones a context of max_seq can index
        const uint32_t half = d.hd / 2;
        const uint32_t nrows = pos_limit(d);
        const size_t tb = (size_t)nrows * half * 4;
        DM(e->rope_cos, tb); DM(e->rope_sin, tb);
        if (d.arch == 3u) {   // rebuilt with theta = 1e6 on the host libm, exactly infer.c:189-204
            std::vector<float> c((size_t)nrows * half), s((size_t)nrows * half), fr(half);
            for (uint32_t i = 0; i < half; i++) fr[i] = 1.0f / powf(1000000.0f, (float)(i * 2) / (float)d.hd);
            for (uint32_t p = 0; p < nrows; p++)
                for (uint32_t i = 0; i < half; i++) { c[(size_t)p * half + i] = cosf(p * fr[i]); s[(size_t)p * half + i] = sinf(p * fr[i]); }
            CK(cudaMemcpy(e->rope_cos, c.data(), tb, cudaMemcpyHostToDevice));
            CK(cudaMemcpy(e->rope_sin, s.data(), tb, cudaMemcpyHostToDevice));
            // the reference steps over a table it never reads (infer.c:201-202); files of tied models may simply end here
            // (Q4K files of arch 3 always do, tools/export_q4k.c:176-204) -- only an untied classifier needs the gap to exist
            const uint64_t gap = 2 * (uint64_t)d.block_size * half * 4;
            if (need(gap)) cur += gap;
            else if (!tied && d.quant == 0x80u) return fail(NB200_EINVAL, "file truncated (RoPE gap before the classifier)");
            else cur = end;
        } else {
            const size_t full = (size_t)d.block_size * half * 4;
            if (!need(2 * full)) return fail(NB200_EINVAL, "file truncated (RoPE table)");
            CK(cudaMemcpy(e->rope_cos, cur, tb, cudaMemcpyHostToDevice));
            CK(cudaMemcpy(e->rope_sin, cur + full, tb, cudaMemcpyHostToDevice));
            cur += 2 * full;
        }
    }
    const uint8_t *cls_w = nullptr, *cls_a = nullptr;
    if (d.quant == 0x00u && !tied)      // the reference points an untied F32 classifier at the start of the parameter block (infer.c:215): refuse, do not copy the bug
        return fail(NB200_EINVAL, "untied F32 classifier is not supported (the reference's own pointer for it is wrong, infer.c:215)");
    if (d.quant == 0x80u && !tied) {
        if (cur > end || !need(V * E + V * E / d.gs * 4)) return fail(NB200_EINVAL, "file truncated (classifier)");
        cls_w = cur; cls_a = cur + V * E;
    }

    // ---- upload with re-layout ----
    uint8_t *staging = nullptr;
    if (d.quant == 0x42u) {
        uint64_t mx = V * (E / 256);
        for (int t = 0; t < 7; t++) { const uint64_t pl = rows[t] * (cols[t] / 256); if (pl > mx) mx = pl; }
        CK(cudaMalloc(&staging, mx * 160));
    }
    struct StagingFree { uint8_t *p; ~StagingFree() { if (p) cudaFree(p); } } sfree{staging};
    int r;
    // source rows [row0, ...) of an [rows x n] tensor in the file's own layout
    auto srcw = [&](const uint8_t *w, uint64_t row0, uint64_t n) -> const uint8_t * {
        return w + (d.quant == 0x00u ? row0 * n * 4 : d.quant == 0x80u ? row0 * n : row0 * (n / 256) * 160);
    };
    auto srca = [&](const uint8_t *a, uint64_t row0, uint64_t n) -> const uint8_t * { return a ? a + row0 * (n / d.gs) * 4 : nullptr; };
    const uint64_t QDl = QD / T, KDl = KD / T, El = E / T, Fl = F / T, Vl = V / T, rk = tp_rank;
    e->qkv.resize(L); e->wo.resize(L); e->w13.resize(L); e->w2.resize(L);
    for (uint64_t l = 0; l < L; l++) {
        if ((r = alloc_mat(e, e->qkv[l], (uint32_t)(QDl + 2 * KDl), (uint32_t)E))) return r;
        if ((r = put_rows(e, e->qkv[l], srcw(src_w[0][l], rk * QDl, E), srca(src_a[0][l], rk * QDl, E), (uint32_t)QDl, 0, 1, staging))) return r;
        if ((r = put_rows(e, e->qkv[l], srcw(src_w[1][l], rk * KDl, E), srca(src_a[1][l], rk * KDl, E), (uint32_t)KDl, (uint32_t)QDl, 1, staging))) return r;
        if ((r = put_rows(e, e->qkv[l], srcw(src_w[2][l], rk * KDl, E), srca(src_a[2][l], rk * KDl, E), (uint32_t)KDl, (uint32_t)(QDl + KDl), 1, staging))) return r;
        if ((r = alloc_mat(e, e->wo[l], (uint32_t)El, (uint32_t)QD))) return r;
        if ((r = put_rows(e, e->wo[l], srcw(src_w[3][l], rk * El, QD), srca(src_a[3][l], rk * El, QD), (uint32_t)El, 0, 1, staging))) return r;
        if ((r = alloc_mat(e, e->w13[l], (uint32_t)(2 * Fl), (uint32_t)E))) return r;
        if ((r = put_rows(e, e->w13[l], srcw(src_w[4][l], rk * Fl, E), srca(src_a[4][l], rk * Fl, E), (uint32_t)Fl, 0, 2, staging))) return r;
        if ((r = put_rows(e, e->w13[l], srcw(src_w[6][l], rk * Fl, E), srca(src_a[6][l], rk * Fl, E), (uint32_t)Fl, 1, 2, staging))) return r;
        if ((r = alloc_mat(e, e->w2[l], (uint32_t)El, (uint32_t)F))) return r;
        if ((r = put_rows(e, e->w2[l], srcw(src_w[5][l], rk * El, F), srca(src_a[5][l], rk * El, F), (uint32_t)El, 0, 1, staging))) return r;
    }
    // every rank keeps the whole embedding table (one row is read per token); the classifier reads its V/T row slice
    const uint64_t wb_before_emb = e->weight_bytes;
    if ((r = alloc_mat(e, e->emb, (uint32_t)V, (uint32_t)E))) return r;
    if ((r = put_rows(e, e->emb, emb_w, emb_a, (uint32_t)V, 0, 1, staging))) return r;
    if (cls_w) {
        e->weight_bytes = wb_before_emb;
        if ((r = alloc_mat(e, e->cls, (uint32_t)Vl, (uint32_t)E))) return r;
        if ((r = put_rows(e, e->cls, srcw(cls_w, rk * Vl, E), srca(cls_a, rk * Vl, E), (uint32_t)Vl, 0, 1, staging))) return r;
    } else {
        e->cls = e->emb; e->tied = true;
        if (T > 1) {
            e->weight_bytes = wb_before_emb + (e->weight_bytes - wb_before_emb) / T;
            e->cls.rows = (uint32_t)Vl;
            const uint64_t row0 = rk * Vl;
            if (d.quant == 0x00u) e->cls.w = (uint8_t *)e->emb.w + row0 * E * 4;
            else if (d.quant == 0x80u) { e->cls.w = (uint8_t *)e->emb.w + row0 * E; e->cls.aux = (uint8_t *)e->emb.aux + row0 * (E / d.gs) * 4; }
            else { e->cls.w = (uint8_t *)e->emb.w + row0 * E / 2; e->cls.aux = (uint8_t *)e->emb.aux + row0 * (E / 256) * 20; }
        }
    }
    // from here on d carries the LOCAL head counts (attention and the QKV epilogue index local heads)
    d.H /= T; d.KV /= T; d.q_dim = (uint32_t)QDl; d.kv_dim = (uint32_t)KDl;

    // ---- activations, KV cache, workspaces ----
    const size_t kv_floats = (size_t)L * d.KV * d.max_seq * d.hd;
    if (T > 1) {
        // exchange block: the three replicated activation vectors live where the peers can write them
        auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
        e->tp_off_x = kTpHdrBytes; e->tp_off_xba = (uint32_t)(e->tp_off_x + al(E * 8)); e->tp_off_hb = (uint32_t)(e->tp_off_xba + al(QD * 8));
        e->tp_block_bytes = e->tp_off_hb + al(F * 8);      // {value, epoch} 64-bit elements
        DM(e->tp_block, e->tp_block_bytes);
        CK(cudaMemset(e->tp_block, 0, e->tp_block_bytes));
        e->x = (float *)(e->tp_block + e->tp_off_x); e->xba = (float *)(e->tp_block + e->tp_off_xba); e->hb = (float *)(e->tp_block + e->tp_off_hb);
        e->tp_peer[tp_rank] = e->tp_block;
    } else {
        DM(e->x, E * 4); DM(e->xba, QD * 4); DM(e->hb, F * 4);
    }
    DM(e->q, QD * 4); DM(e->kraw, KD * 4); DM(e->logits, V * 4);
    DM(e->kc, kv_floats * 4); DM(e->vc, kv_floats * 4);
    CK(cudaMemset(e->kc, 0, kv_floats * 4)); CK(cudaMemset(e->vc, 0, kv_floats * 4));   // calloc'd in the reference (infer.c:47)
    CK(cudaMemset(e->x, 0, E * 4)); CK(cudaMemset(e->logits, 0, V * 4));
    // Execution paths: the streaming kernel (stream.cuh) is the default in fast mode on one GPU; the CUDA-graph multi-kernel
    // path serves exact mode, tensor parallelism, LoRA and shapes the streaming kernel does not take.
    uint32_t nsm = (uint32_t)e->num_sms / e->g_KV;  // (kv head, split) items <= one per SM; same split in every path and TP size => identical bits
    if (nsm < 1) nsm = 1; if (nsm > 64) nsm = 64;
    // the merging CTA stages nsplit x kv_mul x head_dim partial accumulators in shared memory: keep that under 160 KB
    // (only shapes with few kv heads AND many q heads per kv head are affected; none of the BASELINE configs)
    while (nsm > 1 && (size_t)attn_fast_smem_floats(d.kv_mul, d.hd, 0, nsm, kWarps) * 4 > 160u * 1024u) nsm--;
    e->nsplit_max = nsm;
    uint32_t cap = (d.max_seq + nsm - 1) / nsm; cap = (cap + 7u) & ~7u; if (cap < 32) cap = 32;
    e->chunk_cap = cap;
    uint32_t lpr = 1; while (lpr * 4 < d.hd) lpr <<= 1; if (lpr > 32) lpr = 32;
    const uint32_t rpw = 32 / lpr;
    e->attn_smem = (uint32_t)((d.kv_mul * d.hd + d.hd + cap + (size_t)kAttnWarps * rpw * d.hd) * 4);
    DM(e->ws_m, (size_t)d.H * nsm * 4); DM(e->ws_l, (size_t)d.H * nsm * 4); DM(e->ws_acc, (size_t)d.H * nsm * d.hd * 4);
    DM(e->tickets, d.KV * 4); CK(cudaMemset(e->tickets, 0, d.KV * 4));
    if (d.exact) DM(e->att_exact, (size_t)d.H * d.max_seq * 4);
    DM(e->ids_dev, ((size_t)d.max_seq + 8) * 4); CK(cudaMemset(e->ids_dev, 0, ((size_t)d.max_seq + 8) * 4));
    DM(e->seen, V); CK(cudaMemset(e->seen, 0, V));
    e->cls_grid = (uint32_t)e->num_sms * grid_mult();
    DM(e->cls_val, (size_t)e->cls_grid * 4); DM(e->cls_idx, (size_t)e->cls_grid * 4);
    DM(e->st, sizeof(DevState)); CK(cudaMemset(e->st, 0, sizeof(DevState)));
    const size_t maxn = F > QD ? (F > E ? F : E) : (QD > E ? QD : E);
    DM(e->dump_codes, maxn * 2 + 64); DM(e->dump_scales, maxn * 4 + 64);
    if (getenv("NB200_ATTN_DBG")) { DM(e->attn_dbg, 32 * 8); CK(cudaMemset(e->attn_dbg, 0, 32 * 8)); }
    CK(cudaHostAlloc(&e->st_host, sizeof(DevState), cudaHostAllocDefault));
    CK(cudaHostAlloc(&e->tok_host, 64, cudaHostAllocDefault));
    memset(e->st_host, 0, sizeof(DevState));
    CK(cudaDeviceSynchronize());

    {
        // Default path in fast mode on one GPU.  The streaming kernel is set up whenever the shape allows it.  F32 / Q4K models and Q80
        // models under 256 MB of weights always run it (latency-bound: one launch, no kernel boundary per phase).  For larger Q80 models
        // neither path wins everywhere (on one H100 the multi-kernel path is ahead for Qwen3-0.6B @2048, DESIGN.md section 5.2),
        // so the engine times both at the middle of its context and keeps the faster one (calibrate_paths).
        // NB200_STREAM=1 forces the streaming kernel where the shape allows it, NB200_STREAM=0 / NB200_FLAG_NO_STREAM forbid it.
        const char *st_env = getenv("NB200_STREAM");
        const bool st_forced = st_env && atoi(st_env) == 1, st_off = (st_env && atoi(st_env) == 0) || (flags & NB200_FLAG_NO_STREAM);
        if (T == 1 && !st_off) { if ((r = setup_stream(e))) return r; }
        e->path_stream = e->use_stream;
        if (T == 1 && (r = finish_paths(e))) return r;      // tensor-parallel engines capture after the peers are attached
        const bool st_always = d.quant != 0x80u || e->weight_bytes < (256ull << 20);
        if (e->use_stream && !st_forced && !st_always && (r = calibrate_paths(e))) return r;
    }
    guard.ok = true;
    *out = e;
    return 0;
}

static int finish_paths(nb200_engine *e) {
    int r = 0;
    if (e->use_stream) {
        // nothing to capture: a token (or a whole run of tokens) is one launch
    } else if (!(e->flags & NB200_FLAG_NO_GRAPH)) {
        r = capture_graph(e);
        if (r && e->use_pdl) {          // retry without PDL edges before giving up on the graph
            e->use_pdl = false;
            r = capture_graph(e);
        }
        if (r) return r;
    } else {
        e->launches_per_token = 2 + (5 + (e->lora.active ? 4u : 0u)) * e->d.L;
    }
    return 0;
}

// Both fast paths are ready: time `n` decode steps on each from the middle of the usable context (device loop, CUDA events on the
// engine's stream, one untimed round first) and keep the faster.  The steps write K/V rows at positions pos0.., logits, x and the
// ids; all of it is cleared again afterwards, because non-causal attention reads every cache row, written or not, and a fresh
// engine must compute what the reference's calloc'd context does.
static int calibrate_paths(nb200_engine *e) {
    const uint32_t n = 8;
    const uint32_t lim = pos_limit(e->d);
    if (lim < 4 * n) return 0;
    const uint32_t pos0 = lim / 2;
    struct Events { cudaEvent_t ev[2] = {nullptr, nullptr}; ~Events() { for (auto v : ev) if (v) cudaEventDestroy(v); } } evs;
    for (auto &v : evs.ev) CK(cudaEventCreate(&v));
    float ms[2] = {0.0f, 0.0f};
    int r;
    for (int path = 0; path < 2; path++) {
        e->use_stream = (path == 0);
        if (path == 1) { e->launches_per_token = 0; if ((r = finish_paths(e))) return r; }      // captures the multi-kernel graph
        for (int rep = 0; rep < 2; rep++) {
            CK(cudaMemsetAsync(e->ids_dev, 0, (size_t)(pos0 + 1) * 4, e->stream));
            if ((r = push_state(e, pos0, 1, pos0 + 1, 1, 1.0f, 0, 0))) return r;
            CK(cudaEventRecord(evs.ev[0], e->stream));
            if (e->use_stream) { if ((r = launch_stream(e, n))) return r; }
            else for (uint32_t i = 0; i < n; i++) if ((r = launch_token(e))) return r;
            CK(cudaEventRecord(evs.ev[1], e->stream));
            CK(cudaStreamSynchronize(e->stream));
            CK(cudaEventElapsedTime(&ms[path], evs.ev[0], evs.ev[1]));
        }
    }
    e->calib_ms[0] = ms[0] / n; e->calib_ms[1] = ms[1] / n;
    e->use_stream = ms[0] <= ms[1];
    e->path_stream = e->use_stream;
    if (e->use_stream) e->launches_per_token = 1;
    e->launches = 0;
    const Dims &d = e->d;                                                                 // as created
    const size_t kv_floats = (size_t)d.L * d.KV * d.max_seq * d.hd;
    CK(cudaMemsetAsync(e->kc, 0, kv_floats * 4, e->stream)); CK(cudaMemsetAsync(e->vc, 0, kv_floats * 4, e->stream));
    CK(cudaMemsetAsync(e->x, 0, (size_t)d.E * 4, e->stream)); CK(cudaMemsetAsync(e->logits, 0, (size_t)d.V * 4, e->stream));
    CK(cudaMemsetAsync(e->ids_dev, 0, ((size_t)d.max_seq + 8) * 4, e->stream));
    CK(cudaMemsetAsync(e->seen, 0, d.V, e->stream));
    e->seen_valid = false; e->seen_mirror.clear();
    CK(cudaStreamSynchronize(e->stream));
    return 0;
}

int nb200_engine_create(nb200_engine **out, const uint8_t *img, uint64_t image_bytes, uint32_t max_seq_len, int device,
                        uint32_t flags) {
    return create_impl(out, img, image_bytes, max_seq_len, device, flags, 0, 1);
}

int nb200_engine_create_tp(nb200_engine **out, const uint8_t *img, uint64_t image_bytes, uint32_t max_seq_len, int device,
                           uint32_t flags, uint32_t tp_rank, uint32_t tp_size) {
    return create_impl(out, img, image_bytes, max_seq_len, device, flags, tp_rank, tp_size);
}

// (de)activate the loaded plug-in: LoRA runs on the multi-kernel path only, so the path and the graph are rebuilt
static int lora_set_active(nb200_engine *e, bool on) {
    if (on == e->lora.active) return 0;
    CK(cudaSetDevice(e->device));
    CK(cudaStreamSynchronize(e->stream));
    if (e->graph) { cudaGraphExecDestroy(e->graph); e->graph = nullptr; }
    e->lora.active = on;
    e->use_stream = on ? false : e->path_stream;
    e->launches_per_token = e->use_stream ? 1u : 0u;
    return finish_paths(e);
}

/* nb200_lora_load <- load_lora_from_buffer infer/infer.c:513-519 (parse_lora_file :436-500, malloc_fwd_buffer_with_lora :413-433).
 * image_bytes == 0: trust the header like the reference does. */
int nb200_lora_load(nb200_engine *e, const uint8_t *img, uint64_t image_bytes) {
    if (!e || !img) return fail(NB200_EINVAL, "null argument");
    if (e->tp_size > 1) return fail(NB200_EINVAL, "LoRA is not available on tensor-parallel engines");
    if (e->lora.loaded) return fail(NB200_EINVAL, "a LoRA plug-in is already loaded");
    const Dims &d = e->d;
    if (d.arch != 0u) return fail(NB200_EINVAL, "LoRA plug-ins are defined for the Nano architecture only (infer.c:792)");
    if (image_bytes && image_bytes < 256) return fail(NB200_EINVAL, "LoRA image truncated");
    const uint32_t rank = rd_u32(img + 24), alpha = rd_u32(img + 28);
    const uint32_t L = rd_u32(img + 32), E = rd_u32(img + 36), H = rd_u32(img + 40), KV = rd_u32(img + 44), F = rd_u32(img + 48);
    if (L != d.L || E != d.E || H != d.H || KV != d.KV || F != d.F) return fail(NB200_EINVAL, "LoRA module does not fit the base model");
    if (rank == 0 || rank > 64) return fail(NB200_EINVAL, "LoRA rank %u unsupported (1..64)", rank);
    const uint64_t la = (uint64_t)L * rank * E;
    const uint64_t lens[8] = {la, (uint64_t)L * d.q_dim * rank, la, (uint64_t)L * d.kv_dim * rank, la, (uint64_t)L * d.kv_dim * rank, la, (uint64_t)L * E * rank};
    uint64_t total = 0; for (uint64_t v : lens) total += v;
    if (image_bytes && image_bytes < 256 + total * 4) return fail(NB200_EINVAL, "LoRA image truncated (need %llu bytes)", (unsigned long long)(256 + total * 4));
    CK(cudaSetDevice(e->device));
    const float *p = reinterpret_cast<const float *>(img + 256);
    for (int m = 0; m < 4; m++) {
        DM(e->lora.a[m], lens[2 * m] * 4); DM(e->lora.b[m], lens[2 * m + 1] * 4);
        CK(cudaMemcpy(e->lora.a[m], p, lens[2 * m] * 4, cudaMemcpyHostToDevice)); p += lens[2 * m];
        CK(cudaMemcpy(e->lora.b[m], p, lens[2 * m + 1] * 4, cudaMemcpyHostToDevice)); p += lens[2 * m + 1];
    }
    DM(e->lora.t, 4 * rank * 4); DM(e->lora.o1, (size_t)E * 4);
    e->lora.rank = rank; e->lora.alpha = alpha; e->lora.loaded = true;
    return lora_set_active(e, true);
}

/* use_lora of llm_forward (infer.c:713, 792, 898): run with (1) or without (0) the loaded plug-in */
int nb200_lora_enable(nb200_engine *e, int on) {
    if (!e) return fail(NB200_EINVAL, "null engine");
    if (!e->lora.loaded) return on ? fail(NB200_EINVAL, "no LoRA plug-in loaded") : 0;
    return lora_set_active(e, on != 0);
}

/* nb200_lora_unload <- free_lora infer/infer.c:521-534 */
int nb200_lora_unload(nb200_engine *e) {
    if (!e) return fail(NB200_EINVAL, "null engine");
    if (!e->lora.loaded) return 0;
    int r = lora_set_active(e, false);
    auto drop = [&](float *&p) {
        if (!p) return;
        for (auto it = e->allocs.begin(); it != e->allocs.end(); ++it) if (*it == (void *)p) { e->allocs.erase(it); break; }
        cudaFree(p); p = nullptr;
    };
    for (int m = 0; m < 4; m++) { drop(e->lora.a[m]); drop(e->lora.b[m]); }
    drop(e->lora.t); drop(e->lora.o1);
    e->lora.loaded = false; e->lora.rank = 0;
    return r;
}

int nb200_tp_export(nb200_engine *e, void *handle64) {
    if (!e || !handle64 || e->tp_size <= 1) return fail(NB200_EINVAL, "not a tensor-parallel engine");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    CK(cudaSetDevice(e->device));
    cudaIpcMemHandle_t h;
    CK(cudaIpcGetMemHandle(&h, e->tp_block));
    memcpy(handle64, &h, 64);
    return 0;
}

static int tp_finish_attach(nb200_engine *e) {
    e->tp_attached = true;
    return finish_paths(e);
}

int nb200_tp_attach_ipc(nb200_engine *e, const void *handles) {
    if (!e || !handles || e->tp_size <= 1) return fail(NB200_EINVAL, "not a tensor-parallel engine");
    if (e->tp_attached) return fail(NB200_EINVAL, "already attached");
    CK(cudaSetDevice(e->device));
    for (uint32_t p = 0; p < e->tp_size; p++) {
        if (p == e->tp_rank) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, (const uint8_t *)handles + (size_t)p * 64, 64);
        void *ptr = nullptr;
        cudaError_t ce = cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess);
        if (ce != cudaSuccess) return fail(NB200_ECUDA, "cudaIpcOpenMemHandle(rank %u) failed: %s", p, cudaGetErrorString(ce));
        e->tp_ipc_opened.push_back(ptr);
        e->tp_peer[p] = (unsigned char *)ptr;
    }
    return tp_finish_attach(e);
}

int nb200_tp_attach_local(nb200_engine *e, nb200_engine *const *group) {
    if (!e || !group || e->tp_size <= 1) return fail(NB200_EINVAL, "not a tensor-parallel engine");
    if (e->tp_attached) return fail(NB200_EINVAL, "already attached");
    CK(cudaSetDevice(e->device));
    for (uint32_t p = 0; p < e->tp_size; p++) {
        nb200_engine *g = group[p];
        if (!g || g->tp_size != e->tp_size || g->tp_rank != p || g->tp_block_bytes != e->tp_block_bytes) return fail(NB200_EINVAL, "group[%u] is not rank %u of this group", p, p);
        if (p == e->tp_rank) continue;
        if (g->device != e->device) {
            int can = 0;
            CK(cudaDeviceCanAccessPeer(&can, e->device, g->device));
            if (!can) return fail(NB200_ECUDA, "device %d cannot access device %d", e->device, g->device);
            cudaError_t ce = cudaDeviceEnablePeerAccess(g->device, 0);
            if (ce != cudaSuccess && ce != cudaErrorPeerAccessAlreadyEnabled) return fail(NB200_ECUDA, "cudaDeviceEnablePeerAccess: %s", cudaGetErrorString(ce));
            cudaGetLastError();
        }
        e->tp_peer[p] = g->tp_block;
    }
    return tp_finish_attach(e);
}

int nb200_get_config(const nb200_engine *e, nb200_config *c) {
    if (!e || !c) return fail(NB200_EINVAL, "null argument");
    memset(c, 0, sizeof *c);
    const Dims &d = e->d;
    c->arch = d.arch; c->quant = d.quant; c->group_size = (d.quant == 0x80u) ? d.gs : 0;
    c->block_size = d.block_size; c->vocab_size = d.V; c->n_layer = d.L; c->n_embd = d.E;
    c->n_head = e->g_H; c->n_kv_head = e->g_KV; c->n_hidden = d.F; c->tied = e->tied ? 1u : 0u; c->head_dim = d.hd;
    c->q_dim = e->g_q_dim; c->kv_dim = e->g_kv_dim; c->max_seq_len = d.max_seq; c->tp_rank = e->tp_rank; c->tp_size = e->tp_size;
    c->reserved[0] = e->use_stream ? 4u : (e->graph ? 1u : 0u);      // execution path: 4 streaming kernel, 1 graph, 0 direct launches
    c->reserved[1] = (uint32_t)(e->calib_ms[0] * 1000.0f + 0.5f);     // calibrate_paths: microseconds per token of the streaming kernel ...
    c->reserved[2] = (uint32_t)(e->calib_ms[1] * 1000.0f + 0.5f);     // ... and of the multi-kernel graph (0 = the choice was not measured)
    c->reserved[3] = e->mv_mask;
    c->reserved[4] = e->attn_kind;
    return 0;
}

// after a stream sync: did a tensor-parallel spin give up on a peer?
static int tp_check(nb200_engine *e) {
    if (e->tp_size <= 1) return 0;
    uint32_t t = 0;
    CK(cudaMemcpy(&t, e->tp_block + offsetof(TpHdr, timeout), 4, cudaMemcpyDeviceToHost));
    if (t) return fail(NB200_ECUDA, "tensor parallel: rank %u timed out waiting for a peer (ranks must issue the same calls)", e->tp_rank);
    return 0;
}

static int push_state(nb200_engine *e, uint32_t pos, uint32_t causal, uint32_t n_prompt, uint32_t advance, float penalty,
                      uint32_t token, uint32_t use_token) {
    DevState *h = e->st_host;
    CK(cudaStreamSynchronize(e->stream));      // the pinned slot may still be in flight
    memset(h, 0, sizeof(DevState));
    h->pos = pos; h->is_causal = causal; h->n_prompt = n_prompt; h->advance = advance; h->penalty = penalty;
    h->token = token; h->use_token = use_token;
    CK(cudaMemcpyAsync(e->st, h, sizeof(DevState), cudaMemcpyHostToDevice, e->stream));
    return 0;
}

int nb200_forward(nb200_engine *e, uint32_t token, uint32_t pos, uint32_t is_causal) {
    if (!e) return fail(NB200_EINVAL, "null engine");
    if (pos >= pos_limit(e->d) || token >= e->d.V) return fail(NB200_EINVAL, "token/pos out of range");
    CK(cudaSetDevice(e->device));
    int r;
    if ((r = push_state(e, pos, is_causal ? 1u : 0u, 0, 0, 1.0f, token, 1))) return r;
    if ((r = launch_token(e))) return r;
    CK(cudaStreamSynchronize(e->stream));
    return tp_check(e);
}

int nb200_read_logits(nb200_engine *e, float *host_logits) {
    if (!e || !host_logits) return fail(NB200_EINVAL, "null argument");
    CK(cudaSetDevice(e->device));
    CK(cudaMemcpyAsync(host_logits, e->logits, (size_t)e->d.V * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return 0;
}

static int sync_seen(nb200_engine *e, const uint32_t *ids, uint32_t pos) {
    uint32_t have = (uint32_t)e->seen_mirror.size();
    bool ok = e->seen_valid && have <= pos && (have == 0 || memcmp(e->seen_mirror.data(), ids, (size_t)have * 4) == 0);
    if (!ok) {
        CK(cudaMemsetAsync(e->seen, 0, e->d.V, e->stream));
        e->seen_mirror.clear(); have = 0; e->seen_valid = true;
    }
    if (pos > have) {
        for (uint32_t i = have; i < pos; i++) if (ids[i] >= e->d.V) return fail(NB200_EINVAL, "id out of range");
        CK(cudaMemcpyAsync(e->ids_dev + have, ids + have, (size_t)(pos - have) * 4, cudaMemcpyHostToDevice, e->stream));
        k_mark_seen<<<1, 256, 0, e->stream>>>(e->seen, e->ids_dev, have, pos);
        CK(cudaGetLastError());
        e->launches++;
        e->seen_mirror.insert(e->seen_mirror.end(), ids + have, ids + pos);
    }
    return 0;
}

int nb200_next_greedy(nb200_engine *e, const uint32_t *ids, uint32_t pos, int is_prefilling, float penalty, uint32_t *next) {
    if (!e || !ids || !next) return fail(NB200_EINVAL, "null argument");
    if (pos >= pos_limit(e->d) || ids[pos] >= e->d.V) return fail(NB200_EINVAL, "token/pos out of range");
    CK(cudaSetDevice(e->device));
    int r;
    if ((r = push_state(e, pos, 1, 0, 0, is_prefilling ? 1.0f : penalty, ids[pos], 1))) return r;
    if (!is_prefilling && penalty != 1.0f) { if ((r = sync_seen(e, ids, pos))) return r; }
    if ((r = launch_token(e))) return r;
    CK(cudaMemcpyAsync(e->tok_host, &e->st->next_token, 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    *next = is_prefilling ? ids[pos + 1] : *e->tok_host;
    return tp_check(e);
}

/* nb200_next_sampled <- generate_next_token, temperature > 0 branch (infer.c:1156-1189: penalty, /= temperature, softmax, coin, sample_top_p).
 * The whole step runs on the device; `coin` is the host's random_f32 draw.  top6 (optional): the six most probable ids (observation hook). */
int nb200_next_sampled(nb200_engine *e, const uint32_t *ids, uint32_t pos, float penalty, float temperature, float top_p, float coin,
                       uint32_t *next, uint32_t *top6) {
    if (!e || !ids || !next) return fail(NB200_EINVAL, "null argument");
    if (pos >= pos_limit(e->d) || ids[pos] >= e->d.V) return fail(NB200_EINVAL, "token/pos out of range");
    if (!(temperature > 0.0f)) return fail(NB200_EINVAL, "temperature must be > 0 (use nb200_next_greedy for 0)");
    if (e->tp_size > 1) return fail(NB200_EINVAL, "device-side sampling is not available on tensor-parallel engines (logits are sharded)");
    CK(cudaSetDevice(e->device));
    if (!e->samp_ws) {
        const size_t bytes = sample_workspace_bytes(e->d.V, &e->samp_cub);
        DM(e->samp_ws, bytes);
        CK(cudaHostAlloc(&e->samp_host, 64, cudaHostAllocDefault));
    }
    int r;
    if ((r = push_state(e, pos, 1, 0, 0, penalty, ids[pos], 1))) return r;
    if (penalty != 1.0f) { if ((r = sync_seen(e, ids, pos))) return r; }
    if ((r = launch_token(e))) return r;
    uint32_t *out_dev = nullptr;
    CK(sample_top_p_launch(e->samp_ws, e->samp_cub, e->logits, e->d.V, temperature, top_p, coin, e->st, &out_dev, e->stream));
    e->launches += 3;
    CK(cudaMemcpyAsync(e->samp_host, out_dev, 32, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    *next = e->samp_host[0];
    if (top6) for (int i = 0; i < 6; i++) top6[i] = e->samp_host[1 + i];
    return 0;
}

int nb200_decode_greedy(nb200_engine *e, uint32_t *ids, uint32_t n_prompt, uint32_t n_total, float penalty,
                        float *prefill_ms, float *device_ms) {
    if (!e || !ids) return fail(NB200_EINVAL, "null argument");
    if (n_prompt < 1 || n_total < n_prompt || n_total > pos_limit(e->d) + 1) return fail(NB200_EINVAL, "bad n_prompt/n_total");
    for (uint32_t i = 0; i < n_prompt; i++) if (ids[i] >= e->d.V) return fail(NB200_EINVAL, "id out of range");
    CK(cudaSetDevice(e->device));
    int r;
    struct Events { cudaEvent_t ev[3] = {nullptr, nullptr, nullptr}; ~Events() { for (auto v : ev) if (v) cudaEventDestroy(v); } } evs;     // destroyed on every return path
    cudaEvent_t (&ev)[3] = evs.ev;
    for (auto &v : ev) CK(cudaEventCreate(&v));
    if ((r = push_state(e, 0, 1, n_prompt, 1, penalty, 0, 0))) return r;
    CK(cudaMemcpyAsync(e->ids_dev, ids, (size_t)n_prompt * 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemsetAsync(e->seen, 0, e->d.V, e->stream));
    e->seen_valid = false; e->seen_mirror.clear();
    CK(cudaEventRecord(ev[0], e->stream));
    if (e->use_stream) { if ((r = launch_stream(e, n_prompt - 1))) return r; }
    else for (uint32_t p = 0; p + 1 < n_prompt; p++) if ((r = launch_token(e))) return r;
    CK(cudaEventRecord(ev[1], e->stream));
    if (e->use_stream) { if ((r = launch_stream(e, n_total - n_prompt))) return r; }
    else for (uint32_t p = n_prompt - 1; p + 1 < n_total; p++) if ((r = launch_token(e))) return r;
    CK(cudaEventRecord(ev[2], e->stream));
    CK(cudaMemcpyAsync(ids, e->ids_dev, (size_t)n_total * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    float a = 0, b = 0;
    CK(cudaEventElapsedTime(&a, ev[0], ev[1]));
    CK(cudaEventElapsedTime(&b, ev[1], ev[2]));
    if (prefill_ms) *prefill_ms = a;
    if (device_ms) *device_ms = b;
    return tp_check(e);
}

int nb200_read_buffer(nb200_engine *e, int field, uint32_t layer, uint32_t pos, float *dst, uint32_t count) {
    if (!e || !dst) return fail(NB200_EINVAL, "null argument");
    CK(cudaSetDevice(e->device));
    CK(cudaStreamSynchronize(e->stream));
    const Dims &d = e->d;
    const float *src = nullptr; uint32_t avail = 0;
    if (e->tp_size > 1 && (field == NB200_F_X || field == NB200_F_XBA || field == NB200_F_HB))
        return fail(NB200_EINVAL, "tensor-parallel engines keep x/xba/hb as {value, epoch} words; read them from a single-GPU engine");
    switch (field) {
        case NB200_F_X: src = e->x; avail = d.E; break;
        case NB200_F_XBA: src = e->xba; avail = d.q_dim; break;
        case NB200_F_HB: src = e->hb; avail = d.F; break;
        case NB200_F_Q: src = e->q; avail = d.q_dim; break;
        case NB200_F_LOGITS: src = e->logits; avail = d.V; break;
        case NB200_F_ACT_SCALE: src = e->dump_scales; avail = count; break;
        case NB200_F_ACT_I8: {
            CK(cudaMemcpy(dst, e->dump_codes, count, cudaMemcpyDeviceToHost));   // count = bytes here
            return 0;
        }
        case NB200_F_KROW: case NB200_F_VROW: {
            if (layer >= d.L || pos >= d.max_seq || count != d.kv_dim) return fail(NB200_EINVAL, "bad KV row request");
            const float *base = (field == NB200_F_KROW ? e->kc : e->vc) + (size_t)layer * d.KV * d.max_seq * d.hd;
            for (uint32_t h = 0; h < d.KV; h++)
                CK(cudaMemcpy(dst + (size_t)h * d.hd, base + ((size_t)h * d.max_seq + pos) * d.hd, (size_t)d.hd * 4, cudaMemcpyDeviceToHost));
            return 0;
        }
        default: return fail(NB200_EINVAL, "unknown field %d", field);
    }
    if (count > avail) return fail(NB200_EINVAL, "count %u exceeds field size %u", count, avail);
    CK(cudaMemcpy(dst, src, (size_t)count * 4, cudaMemcpyDeviceToHost));
    return 0;
}

int nb200_write_x(nb200_engine *e, const float *x, uint32_t count) {
    if (!e || !x || count != e->d.E) return fail(NB200_EINVAL, "bad argument");
    if (e->tp_size > 1) return fail(NB200_EINVAL, "not available on tensor-parallel engines");
    CK(cudaSetDevice(e->device));
    CK(cudaStreamSynchronize(e->stream));
    CK(cudaMemcpy(e->x, x, (size_t)count * 4, cudaMemcpyHostToDevice));
    return 0;
}

int nb200_run_layer(nb200_engine *e, uint32_t layer, uint32_t pos, uint32_t is_causal) {
    if (!e || layer >= e->d.L || pos >= pos_limit(e->d)) return fail(NB200_EINVAL, "bad argument");
    if (e->tp_size > 1) return fail(NB200_EINVAL, "not available on tensor-parallel engines");
    CK(cudaSetDevice(e->device));
    int r;
    if ((r = push_state(e, pos, is_causal ? 1u : 0u, 0, 0, 1.0f, 0, 1))) return r;
    if ((r = run_layer(e, layer))) return r;
    CK(cudaStreamSynchronize(e->stream));
    return 0;
}

// Runs tokens ids[start..start+n) (teacher-forced, API mode) WITHOUT graph/PDL and with a CUDA-event pair
// around every kernel; accumulates device milliseconds and launch counts per kernel class:
// 0 embed, 1 qkv, 2 attention, 3 o-proj, 4 w1|w3, 5 w2, 6 classifier.
int nb200_profile_tokens(nb200_engine *e, const uint32_t *ids, uint32_t start, uint32_t n, float ms[7], uint32_t counts[7]) {
    if (!e || !ids || !ms || !counts) return fail(NB200_EINVAL, "null argument");
    if (n > pos_limit(e->d) || start > pos_limit(e->d) - n) return fail(NB200_EINVAL, "range exceeds min(max_seq_len, block_size)");
    CK(cudaSetDevice(e->device));
    const bool pdl = e->use_pdl;
    e->use_pdl = false; e->prof_on = true;
    int r = 0;
    for (uint32_t i = 0; i < n && !r; i++) {
        r = push_state(e, start + i, 1, 0, 0, 1.0f, ids[start + i], 1);
        if (!r) r = run_token(e);
    }
    e->prof_on = false; e->use_pdl = pdl;
    cudaStreamSynchronize(e->stream);
    for (int k = 0; k < 7; k++) { ms[k] = 0.0f; counts[k] = 0; }
    for (auto &p : e->prof) {
        float t = 0.0f;
        if (cudaEventElapsedTime(&t, p.a, p.b) == cudaSuccess && p.tag >= 0 && p.tag < 7) { ms[p.tag] += t; counts[p.tag]++; }
        cudaEventDestroy(p.a); cudaEventDestroy(p.b);
    }
    e->prof.clear();
    return r;
}

// Debug (NB200_ATTN_DBG=1 at engine creation): the 32 %globaltimer stamps (ns) of the last run of layer L/2's attention kernel.
int nb200_read_attn_trace(nb200_engine *e, unsigned long long *stamps32) {
    if (!e || !stamps32 || !e->attn_dbg) return fail(NB200_EINVAL, "attention trace not enabled (NB200_ATTN_DBG=1)");
    CK(cudaSetDevice(e->device));
    CK(cudaStreamSynchronize(e->stream));
    CK(cudaMemcpy(stamps32, e->attn_dbg, 32 * 8, cudaMemcpyDeviceToHost));
    return 0;
}

// Debug: per-barrier clock64() stamps of CTA 0 for one token through the persistent kernel (5L+3 stamps + 1).
int nb200_trace_token(nb200_engine *e, uint32_t token, uint32_t pos, unsigned long long *stamps, uint32_t cap, uint32_t *count) {
    if (!e || !stamps || !count) return fail(NB200_EINVAL, "null argument");
    if (!e->use_stream) return fail(NB200_EINVAL, "persistent kernel not active");
    if (pos >= pos_limit(e->d) || token >= e->d.V) return fail(NB200_EINVAL, "token/pos out of range");
    CK(cudaSetDevice(e->device));
    const uint32_t n = 1024 + 256;         // [0, 5L+2): per-barrier stamps; [1024, 1024+15): phase stamps of layer L/2; [1100, 1100+64): stamps inside its four matvec phases
    if (cap < n || 5 * e->d.L + 4 > 1024) return fail(NB200_EINVAL, "need room for %u stamps", n);
    unsigned long long *buf = nullptr;
    CK(cudaMalloc(&buf, (size_t)n * 8));
    CK(cudaMemset(buf, 0, (size_t)n * 8));
    e->trace_dev = buf;
    int r = push_state(e, pos, 1, 0, 0, 1.0f, token, 1);
    if (!r) r = launch_stream(e, 1);
    e->trace_dev = nullptr;
    cudaStreamSynchronize(e->stream);
    if (!r) { CK(cudaMemcpy(stamps, buf, (size_t)n * 8, cudaMemcpyDeviceToHost)); *count = n; }
    cudaFree(buf);
    return r;
}

uint64_t nb200_kernel_launches(const nb200_engine *e) { return e ? e->launches : 0; }
uint32_t nb200_launches_per_token(const nb200_engine *e) { return e ? e->launches_per_token : 0; }
uint64_t nb200_weight_bytes(const nb200_engine *e) { return e ? e->weight_bytes : 0; }

// ---------------------------------------------------------------------------------------------
// op-level entry points
// ---------------------------------------------------------------------------------------------
}  // extern "C"
namespace {
struct DevBuf {
    void *p = nullptr;
    ~DevBuf() { if (p) cudaFree(p); }
    int alloc(size_t b) { return cudaMalloc(&p, b ? b : 16) == cudaSuccess ? 0 : fail(NB200_ENOMEM, "cudaMalloc failed"); }
    template <typename T> T *as() { return static_cast<T *>(p); }
};
int need_device() {
    if (nb200_device_count() <= 0) return fail(NB200_ENODEV, "no CUDA device: nano_b200 has no CPU path");
    return 0;
}
int op_prep(uint32_t quant, const float *x, const float *gain, uint32_t n, uint32_t gs, uint32_t exact, float *out_f32,
            int8_t *codes_host, size_t codes_bytes, float *scales_host, size_t scales_count) {
    int r;
    if ((r = need_device())) return r;
    DevBuf dx, dg, dout, dcodes, dscales;
    if ((r = dx.alloc((size_t)n * 4)) || (r = dg.alloc((size_t)n * 4)) || (r = dout.alloc((size_t)n * 4)) ||
        (r = dcodes.alloc((size_t)n * 2 + 64)) || (r = dscales.alloc((size_t)n * 4 + 64))) return r;
    CK(cudaMemcpy(dx.p, x, (size_t)n * 4, cudaMemcpyHostToDevice));
    if (gain) CK(cudaMemcpy(dg.p, gain, (size_t)n * 4, cudaMemcpyHostToDevice));
    const uint32_t smem = act_smem_bytes(quant, n, gs ? gs : 1);
    if (smem > 40 * 1024) CK(cudaFuncSetAttribute((const void *)k_op_prep, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));   // + static red[32]: see launch()
    k_op_prep<<<1, kThreads, smem>>>(dx.as<float>(), gain ? dg.as<float>() : nullptr, n, gs, quant, exact, dout.as<float>(),
                                     dcodes.as<int8_t>(), dscales.as<float>());
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    if (out_f32) CK(cudaMemcpy(out_f32, dout.p, (size_t)n * 4, cudaMemcpyDeviceToHost));
    if (codes_host) CK(cudaMemcpy(codes_host, dcodes.p, codes_bytes, cudaMemcpyDeviceToHost));
    if (scales_host) CK(cudaMemcpy(scales_host, dscales.p, scales_count * 4, cudaMemcpyDeviceToHost));
    return 0;
}
int op_matvec(uint32_t quant, float *out, const float *x, const void *w, size_t wbytes, const void *aux, size_t auxbytes,
              uint32_t n, uint32_t d_rows, uint32_t gs, uint32_t exact, bool q4k_file_blocks) {
    int r;
    if ((r = need_device())) return r;
    DevBuf dx, dw, da, dout, dstage;
    if ((r = dx.alloc((size_t)n * 4)) || (r = dout.alloc((size_t)d_rows * 4))) return r;
    CK(cudaMemcpy(dx.p, x, (size_t)n * 4, cudaMemcpyHostToDevice));
    Mat m; m.rows = d_rows; m.n = n;
    if (q4k_file_blocks) {
        const uint64_t nblocks = (uint64_t)d_rows * (n / 256);
        if ((r = dstage.alloc(nblocks * 160)) || (r = dw.alloc((size_t)d_rows * n / 2 + 64)) || (r = da.alloc(nblocks * 20 + 64))) return r;
        CK(cudaMemcpy(dstage.p, w, nblocks * 160, cudaMemcpyHostToDevice));
        k_q4k_split<<<256, 256>>>(dstage.as<uint8_t>(), nblocks, n / 256, dw.as<uint8_t>(), da.as<uint8_t>(), 0, 1);
        CK(cudaGetLastError());
    } else {
        if ((r = dw.alloc(wbytes + 64))) return r;
        CK(cudaMemcpy(dw.p, w, wbytes, cudaMemcpyHostToDevice));
        if (aux) { if ((r = da.alloc(auxbytes + 64))) return r; CK(cudaMemcpy(da.p, aux, auxbytes, cudaMemcpyHostToDevice)); }
    }
    m.w = dw.p; m.aux = da.p;
    MatvecArgs a{};
    a.d.quant = quant; a.d.gs = gs; a.d.exact = exact; a.d.hd = 4; a.d.max_seq = 1;
    a.src = dx.as<float>(); a.gain = nullptr; a.out = dout.as<float>();
    int dev = 0, sms = 148;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if ((r = run_matvec(nullptr, EPI_STORE, m, a, false, sms))) return r;
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(out, dout.p, (size_t)d_rows * 4, cudaMemcpyDeviceToHost));
    return 0;
}
}  // namespace
extern "C" {

int nb200_op_rmsnorm(float *out, const float *x, const float *gain, uint32_t n, uint32_t exact) {
    if (!out || !x || !gain || !n) return fail(NB200_EINVAL, "bad argument");
    return op_prep(0x00u, x, gain, n, 1, exact, out, nullptr, 0, nullptr, 0);
}

int nb200_op_q80_quantize(int8_t *codes, float *scales, const float *x, uint32_t n, uint32_t gs) {
    if (!codes || !scales || !x || !n) return fail(NB200_EINVAL, "bad argument");
    if ((gs != 32 && gs != 64 && gs != 128 && gs != 256) || n % gs) return fail(NB200_EINVAL, "unsupported group size");
    return op_prep(0x80u, x, nullptr, n, gs, 0, nullptr, codes, n, scales, n / gs);
}

int nb200_op_q80_matvec(float *out, const float *x, const int8_t *wc, const float *wscales, uint32_t n, uint32_t d, uint32_t gs) {
    if (!out || !x || !wc || !wscales || !n || !d) return fail(NB200_EINVAL, "bad argument");
    if ((gs != 32 && gs != 64 && gs != 128 && gs != 256) || n % gs) return fail(NB200_EINVAL, "unsupported group size");
    return op_matvec(0x80u, out, x, wc, (size_t)d * n, wscales, (size_t)d * (n / gs) * 4, n, d, gs, 1, false);     // the operator is bit-exact: ordered group sum
}

int nb200_op_f32_matvec(float *out, const float *x, const float *w, uint32_t n, uint32_t d, uint32_t exact) {
    if (!out || !x || !w || !n || !d || n % 4) return fail(NB200_EINVAL, "bad argument (n %% 4 != 0?)");
    return op_matvec(0x00u, out, x, w, (size_t)d * n * 4, nullptr, 0, n, d, 1, exact, false);
}

int nb200_op_q4k_quantize(uint8_t *blocks, const float *x, uint32_t n) {
    if (!blocks || !x || !n || n % 256) return fail(NB200_EINVAL, "bad argument (n %% 256 != 0?)");
    std::vector<int8_t> codes((size_t)n + 2 * (n / 32));
    std::vector<float> sc(2 * (size_t)(n / 256));
    int r = op_prep(0x42u, x, nullptr, n, 32, 0, nullptr, codes.data(), codes.size(), sc.data(), sc.size());
    if (r) return r;
    const uint32_t nb = n / 256;
    memset(blocks, 0, (size_t)nb * 160);
    for (uint32_t b = 0; b < nb; b++) {          // re-pack into the file block layout (tensor.c:198-241)
        uint8_t *blk = blocks + (size_t)b * 160;
        const uint32_t tag = 0x42u, len = 256u;
        memcpy(blk, &tag, 4); memcpy(blk + 4, &len, 4);
        memcpy(blk + 12, &sc[b], 4); memcpy(blk + 16, &sc[nb + b], 4);
        const int8_t *s6 = codes.data() + n + b * 8, *b6 = codes.data() + n + n / 32 + b * 8;
        for (int g = 0; g < 4; g++) {
            blk[20 + g] = (uint8_t)(((s6[4 + g] & 0x30) << 2) | (s6[g] & 0x3f));
            blk[24 + g] = (uint8_t)(((b6[4 + g] & 0x30) << 2) | (b6[g] & 0x3f));
            blk[28 + g] = (uint8_t)(((b6[4 + g] & 0x0f) << 4) | (s6[4 + g] & 0x0f));
        }
        for (uint32_t i = 0; i < 256; i += 2)
            blk[32 + (i >> 1)] = (uint8_t)((codes[(size_t)b * 256 + i] & 0x0f) | (codes[(size_t)b * 256 + i + 1] << 4));
    }
    return 0;
}

int nb200_op_q4k_matvec(float *out, const float *x, const uint8_t *w_blocks, uint32_t n, uint32_t d) {
    if (!out || !x || !w_blocks || !n || !d || n % 256) return fail(NB200_EINVAL, "bad argument (n %% 256 != 0?)");
    return op_matvec(0x42u, out, x, w_blocks, 0, nullptr, 0, n, d, 32, 0, true);
}

// Whole-tensor Q4K quantisation (quantize_tensor_q4k_in_situ, tensor.c:281-310): `x` holds nblocks*256 floats whose rows
// are multiples of 256 long; `blocks` receives nblocks 160-byte reference blocks.  Streams through the GPU in chunks.
int nb200_op_q4k_quantize_blocks(uint8_t *blocks, const float *x, uint64_t nblocks) {
    if (!blocks || !x || !nblocks) return fail(NB200_EINVAL, "bad argument");
    int r;
    if ((r = need_device())) return r;
    const uint64_t chunk = 1ull << 16;         // 64 Ki blocks = 64 MB of floats per pass
    DevBuf dx, db;
    const uint64_t cap = nblocks < chunk ? nblocks : chunk;
    if ((r = dx.alloc(cap * 1024)) || (r = db.alloc(cap * 160))) return r;
    for (uint64_t b0 = 0; b0 < nblocks; b0 += chunk) {
        const uint64_t nb = (nblocks - b0 < chunk) ? nblocks - b0 : chunk;
        CK(cudaMemcpy(dx.p, x + b0 * 256, nb * 1024, cudaMemcpyHostToDevice));
        const uint32_t grid = (uint32_t)((nb + 7) / 8 > 4736 ? 4736 : (nb + 7) / 8);
        k_q4k_quantize_blocks<<<grid, 256>>>(dx.as<float>(), nb, db.as<uint8_t>());
        CK(cudaGetLastError());
        CK(cudaMemcpy(blocks + b0 * 160, db.p, nb * 160, cudaMemcpyDeviceToHost));
    }
    return 0;
}

// matmul_q4k (tensor.c:438-471) with BOTH operands in the reference block layout: x_blocks = n/256 blocks,
// w_blocks = d rows of n/256 blocks (the caller applies the layer offset).
int nb200_op_q4k_matvec_blocks(float *out, const uint8_t *x_blocks, const uint8_t *w_blocks, uint32_t n, uint32_t d) {
    if (!out || !x_blocks || !w_blocks || !n || !d || n % 256) return fail(NB200_EINVAL, "bad argument (n %% 256 != 0?)");
    int r;
    if ((r = need_device())) return r;
    const uint32_t bpr = n / 256;
    DevBuf dx, dw, dout;
    if ((r = dx.alloc((size_t)bpr * 160)) || (r = dw.alloc((size_t)d * bpr * 160)) || (r = dout.alloc((size_t)d * 4))) return r;
    CK(cudaMemcpy(dx.p, x_blocks, (size_t)bpr * 160, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dw.p, w_blocks, (size_t)d * bpr * 160, cudaMemcpyHostToDevice));
    k_q4k_matvec_blocks<<<(d + 7) / 8, 256>>>(dw.as<uint8_t>(), dx.as<uint8_t>(), d, bpr, dout.as<float>());
    CK(cudaGetLastError());
    CK(cudaMemcpy(out, dout.p, (size_t)d * 4, cudaMemcpyDeviceToHost));
    return 0;
}

// host-side evaluation of the exact-mode expf (no GPU needed): lets CPU tests pin it to libm
float nb200_host_expf_ref(float x) { return nb::expf_ref_impl(x); }
void nb200_host_expf_ref_array(float *dst, const float *src, uint64_t n) { for (uint64_t i = 0; i < n; i++) dst[i] = nb::expf_ref_impl(src[i]); }

}  // extern "C"
