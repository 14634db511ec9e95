// Attention on wgmma tensor cores for packed ragged sequences (sm_90a): softmax(Q K^T / sqrt(hd)) V per
// (sequence, head) - the encoder self-attention of PARSeq's ViT (timm Attention / F.scaled_dot_product_attention, no
// mask; reference models/layers/parseq_transformer.py:206-234) and the two attentions of the refinement pass
// (reference models/parseq.py:264-299: cross-attention over the encoder memory, and the masked self-attention over the
// content stream whose mask has rows 0 and 1 cleared, SURVEY.md Appendix A1).
//
// One persistent CTA per SM works through its list of units (sequence, head, 128-query tile); it owns a Q tile and a
// 2-stage K/V ring in shared memory:
//   warp 8   lane 0 : TMA producer - Q tile once per unit, K/V tiles of 64 keys (SWIZZLE_128B boxes)
//   warpgroups 0, 1 : 64 queries each.  S = Q K^T by wgmma (both operands K-major in shared memory) into registers,
//                     mask + running max (lazy rescale: the reference max moves only when it grows by > 2^8) + exp2 in
//                     the accumulator layout, P packed to fp16 A fragments in registers, O += P V by wgmma with A from
//                     registers and V as MN-major B operand (the tile is stored exactly as TMA delivers [keys][hd]
//                     rows); after the last key tile O / l -> global.
// While one warpgroup is on the CUDA cores (softmax) the tensor core works for the other.  The P V product always
// runs its four 16-key steps; steps past the last visible key read a zero tile instead of V.
#include <cuda.h>

#include "gemm_tc.h"
#include "parseq_ops.h"
#include "ptx.cuh"

namespace ytk {

namespace {

constexpr int kAtQ = 128;        // queries per unit (two warpgroups of 64)
constexpr int kAtKV = 64;        // keys per tile
constexpr int kAtThreads = 288;  // 2 consumer warpgroups, 1 producer warp
constexpr int kAtStages = 2;
constexpr float kRescaleThreshold = 8.f;  // log2 units: P stays <= 2^8, well inside fp16

struct alignas(64) AttnMaps {
    CUtensorMap q, k, v;
};

struct AttnArgs {
    const SeqDesc* seqs;
    int nseq, heads;
    long long ldkv;     // row pitch of K / V in elements (k_base / ldkv = first key row of a sequence)
    float scale_log2;
    op_t* O;
    long long ldo;
};

template <int HD>
struct AtCfg {
    static constexpr int NB = (HD + 63) / 64;                 // 64-element (128 B) column blocks per row
    static constexpr int NO = NB * 64;                        // columns of the O accumulator
    static constexpr int kQBytes = NB * kAtQ * 128;
    static constexpr int kKBytes = NB * kAtKV * 128;          // one K (or V) tile
    static constexpr int kStageBytes = 2 * kKBytes;
    static constexpr int kZeroBytes = NB * 2048;               // 16 zero V rows per column block
    static constexpr int kSmemBytes =
        kQBytes + kAtStages * kStageBytes + kZeroBytes + 256 /*barriers*/ + 1024 /*alignment slack*/;
};

struct Bars {
    uint64_t q_full, q_empty, kv_full[kAtStages], kv_empty[kAtStages];
};

struct Unit {
    int q_row;    // first query row of the tile in Q
    int o_row;    // first output row
    int rows;     // valid queries in the tile
    int q0;       // index of the tile's first query inside its sequence
    int k_row;    // first key row in K / V
    int k_end;    // keys this tile can see
    int k_len, kpad;
    int nt;       // key tiles
    int head;
};

template <int MASKED>
__device__ __forceinline__ Unit make_unit(const SeqDesc& sd, int head, int qt, long long ldkv) {
    Unit u;
    u.q0 = qt * kAtQ;
    u.q_row = sd.q_off + u.q0;
    u.o_row = sd.o_off + u.q0;
    u.rows = min(kAtQ, sd.q_len - u.q0);
    u.k_row = static_cast<int>(sd.k_base / ldkv);
    u.k_len = sd.k_len;
    u.kpad = sd.kpad;
    int k_end = sd.k_len;
    if (MASKED) {
        k_end = min(k_end, sd.kpad);
        if (u.q0 >= 2) k_end = min(k_end, u.q0 + kAtQ);  // causal rows stop at their own index
    }
    u.k_end = k_end;
    u.nt = (k_end + kAtKV - 1) / kAtKV;
    u.head = head;
    return u;
}

// The units of one CTA in processing order: the CTA owns the (sequence, head) pairs p = cta, cta + ncta, ...; inside a
// pair the query tiles in ascending order, back to back, so that the pair's K / V tiles are still in L2 for the second
// tile.  Every role of the CTA walks the same sequence.
template <int MASKED>
struct UnitIter {
    int p, qt, nqt, head, W, npairs;
    SeqDesc sd;
    Unit u;
    const AttnArgs* a;
    __device__ __forceinline__ void load_pair() {
        const int seq = p / a->heads;
        head = p - seq * a->heads;
        sd = a->seqs[seq];
        nqt = (sd.q_len + kAtQ - 1) / kAtQ;
    }
    // positions on the CTA's first unit; false when it has none
    __device__ __forceinline__ bool begin(const AttnArgs* args, int cta, int ncta, int npairs_) {
        a = args;
        W = ncta;
        npairs = npairs_;
        p = cta;
        qt = -1;
        if (p >= npairs) return false;
        load_pair();
        return next();
    }
    __device__ __forceinline__ bool next() {
        for (;;) {
            ++qt;
            while (qt >= nqt) {
                p += W;
                qt = 0;
                if (p >= npairs) return false;
                load_pair();
            }
            u = make_unit<MASKED>(sd, head, qt, a->ldkv);
            if (u.nt <= 0) continue;
            return true;
        }
    }
};

__device__ __forceinline__ float fast_exp2(float x) {
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

template <int HD, int MASKED>
__global__ void __launch_bounds__(kAtThreads, 1) attn_tc_kernel(const __grid_constant__ AttnMaps maps,
                                                                const AttnArgs args) {
    using Cfg = AtCfg<HD>;
    constexpr int NB = Cfg::NB;
    constexpr int NO = Cfg::NO;
    extern __shared__ uint8_t at_smem_raw[];
    const uint32_t raw_addr = smem_u32(at_smem_raw);
    uint8_t* smem = at_smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
    uint8_t* sQ = smem;
    uint8_t* sKV = smem + Cfg::kQBytes;
    uint8_t* sZero = sKV + kAtStages * Cfg::kStageBytes;
    Bars& b = *reinterpret_cast<Bars*>(sZero + Cfg::kZeroBytes);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        mbar_init(&b.q_full, 1);
        mbar_init(&b.q_empty, 8);   // one arrive per consumer warp
        for (int i = 0; i < kAtStages; ++i) {
            mbar_init(&b.kv_full[i], 1);
            mbar_init(&b.kv_empty[i], 8);
        }
        fence_mbar_init();
        tma_prefetch_desc(&maps.q);
        tma_prefetch_desc(&maps.k);
        tma_prefetch_desc(&maps.v);
    }
    for (int i = threadIdx.x; i < Cfg::kZeroBytes / 16; i += blockDim.x)
        reinterpret_cast<uint4*>(sZero)[i] = make_uint4(0u, 0u, 0u, 0u);
    fence_proxy_async_smem();   // the zero tile (generic-proxy stores) -> visible to the wgmma operand reads
    __syncthreads();

    const int npairs = args.nseq * args.heads;
    const int cta = static_cast<int>(blockIdx.x), ncta = static_cast<int>(gridDim.x);

    if (warp < 8) {
        // ------------------------------------------------------------------ MMA + softmax + epilogue, 64 queries
        const int wg = warp >> 2, wl = warp & 3;
        const int r_in = wg * 64 + wl * 16 + (lane >> 2);   // tile row of this thread's first row (second: + 8)
        const int cq = (lane & 3) * 2;                      // first of the thread's two columns in every 8-column block
        const uint32_t q_addr = smem_u32(sQ) + static_cast<uint32_t>(wg * 64 * 128);
        uint32_t nu = 0, ck = 0;
        UnitIter<MASKED> it;
        for (bool more = it.begin(&args, cta, ncta, npairs); more; more = it.next(), ++nu) {
            const Unit u = it.u;
            float m_ref[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
            float o[NO / 2];
#pragma unroll
            for (int i = 0; i < NO / 2; ++i) o[i] = 0.f;
            mbar_wait(&b.q_full, nu & 1u);
            for (int t = 0; t < u.nt; ++t, ++ck) {
                const uint32_t st = ck % kAtStages;
                mbar_wait(&b.kv_full[st], (ck / kAtStages) & 1u);
                const uint32_t k_addr = smem_u32(sKV + st * Cfg::kStageBytes);
                const uint32_t v_addr = k_addr + Cfg::kKBytes;
                // ---- S = Q K^T (64 queries x 64 keys)
                float s[32];
#pragma unroll
                for (int i = 0; i < 32; ++i) s[i] = 0.f;
                reg_fence(s);
                wgmma_fence();
#pragma unroll
                for (int j = 0; j < HD / 16; ++j) {
                    const uint64_t da = wgmma_desc_sw128(q_addr + (j >> 2) * (kAtQ * 128)) + static_cast<uint64_t>(2 * (j & 3));
                    const uint64_t db = wgmma_desc_sw128(k_addr + (j >> 2) * (kAtKV * 128)) + static_cast<uint64_t>(2 * (j & 3));
                    wgmma_ss<64>(s, da, db, j != 0 ? 1u : 0u);
                }
                wgmma_commit();
                wgmma_wait<0>();
                reg_fence(s);
                if (t == u.nt - 1) {   // the Q tile is consumed: the producer may load the next unit's
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&b.q_empty);
                }
                // ---- mask, scale, tile max of both rows (a row is spread over the 4 lanes of a quad)
                const int key0 = t * kAtKV;
                float mt[2] = {-INFINITY, -INFINITY};
#pragma unroll
                for (int i = 0; i < 32; ++i) {
                    const int h = (i >> 1) & 1;
                    const int key = key0 + (i >> 2) * 8 + cq + (i & 1);
                    const int qi = u.q0 + r_in + 8 * h;   // query index inside the sequence
                    bool vis = key < u.k_end;
                    if (MASKED) vis = vis && ((qi < 2) || (key <= qi));
                    const float v = vis ? s[i] * args.scale_log2 : -INFINITY;
                    s[i] = v;
                    mt[h] = fmaxf(mt[h], v);
                }
                float factor[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    mt[h] = fmaxf(mt[h], __shfl_xor_sync(0xffffffffu, mt[h], 1));
                    mt[h] = fmaxf(mt[h], __shfl_xor_sync(0xffffffffu, mt[h], 2));
                    // reference max: moves only when the tile max exceeds it by more than the threshold
                    factor[h] = 1.f;
                    if (mt[h] > m_ref[h] + kRescaleThreshold || (m_ref[h] == -INFINITY && mt[h] > -INFINITY)) {
                        factor[h] = (m_ref[h] == -INFINITY) ? 0.f : fast_exp2(m_ref[h] - mt[h]);
                        m_ref[h] = mt[h];
                        l_run[h] *= factor[h];
                    }
                }
                if (factor[0] != 1.f || factor[1] != 1.f) {
#pragma unroll
                    for (int i = 0; i < NO / 2; ++i) o[i] *= factor[(i >> 1) & 1];
                }
                // ---- P = exp2(S - m) as fp16 A fragments: k step ks covers keys 16 ks .. 16 ks + 15
                uint32_t pa[4][4];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const float m_use = (m_ref[h] == -INFINITY) ? 0.f : m_ref[h];
                    float ls = 0.f;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const float p0 = fast_exp2(s[4 * j + 2 * h] - m_use);  // exp2(-inf) = 0
                        const float p1 = fast_exp2(s[4 * j + 2 * h + 1] - m_use);
                        ls += p0 + p1;
                        pa[j >> 1][(j & 1) * 2 + h] = pack_op(p0, p1);
                    }
                    l_run[h] += ls;
                }
                // ---- O += P V.  All four 16-key steps are issued (a wgmma under a branch is serialised); a step past
                // the last visible key has P = 0 and reads the zero tile instead of V rows that belong to no sequence
                // of this unit (their contents need not be finite)
                const int ksteps = (min(kAtKV, u.k_end - key0) + 15) >> 4;
                reg_fence(o);
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < 4; ++ks) {
                    const bool live = ks < ksteps;
                    const uint64_t db = live ? wgmma_desc_sw128_mn(v_addr + ks * 2048, kAtKV * 128)
                                             : wgmma_desc_sw128_mn(smem_u32(sZero), 2048);
                    wgmma_rs<NO>(o, pa[ks], db, 1u);
                }
                wgmma_commit();
                wgmma_wait<0>();
                reg_fence(o);
                __syncwarp();
                if (lane == 0) mbar_arrive(&b.kv_empty[st]);   // K / V stage consumed
            }
            // ---- epilogue: O / l -> global
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
                l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
                const int r = r_in + 8 * h;
                if (r < u.rows) {
                    const float inv = l_run[h] > 0.f ? 1.f / l_run[h] : 0.f;
                    op_t* op = args.O + static_cast<long long>(u.o_row + r) * args.ldo + u.head * HD + cq;
#pragma unroll
                    for (int j = 0; j < HD / 8; ++j)
                        *reinterpret_cast<uint32_t*>(op + 8 * j) = pack_op(o[4 * j + 2 * h] * inv, o[4 * j + 2 * h + 1] * inv);
                }
            }
        }
    } else if (lane == 0) {
        // ------------------------------------------------------------------ TMA producer
        uint32_t nu = 0, ck = 0;
        UnitIter<MASKED> it, pf;     // pf runs one unit ahead: its tiles are pulled into L2 while `it` is being fed
        bool more = it.begin(&args, cta, ncta, npairs);
        bool pf_more = pf.begin(&args, cta, ncta, npairs);
        if (pf_more) pf_more = pf.next();
        while (more) {
            const Unit u = it.u;
            const int head = u.head;
            if (pf_more) {
                const Unit& n = pf.u;
#pragma unroll
                for (int blk = 0; blk < NB; ++blk) tma_prefetch_l2_4d(&maps.q, n.head * HD + blk * 64, n.q_row, 0, 0);
                if (n.q0 == 0) {      // the pair's first query tile brings its keys / values in (later tiles re-read them)
                    const int nt = min(n.nt, 6);
                    for (int t = 0; t < nt; ++t)
#pragma unroll
                        for (int blk = 0; blk < NB; ++blk) {
                            tma_prefetch_l2_4d(&maps.k, n.head * HD + blk * 64, n.k_row + t * kAtKV, 0, 0);
                            tma_prefetch_l2_4d(&maps.v, n.head * HD + blk * 64, n.k_row + t * kAtKV, 0, 0);
                        }
                }
                pf_more = pf.next();
            }
            mbar_wait(&b.q_empty, (nu & 1u) ^ 1u);
            mbar_expect_tx(&b.q_full, Cfg::kQBytes);
#pragma unroll
            for (int blk = 0; blk < NB; ++blk)
                tma_load_4d(sQ + blk * (kAtQ * 128), &maps.q, &b.q_full, head * HD + blk * 64, u.q_row, 0, 0);
            ++nu;
            for (int t = 0; t < u.nt; ++t, ++ck) {
                const uint32_t st = ck % kAtStages;
                mbar_wait(&b.kv_empty[st], ((ck / kAtStages) & 1u) ^ 1u);
                mbar_expect_tx(&b.kv_full[st], Cfg::kStageBytes);
                uint8_t* sK = sKV + st * Cfg::kStageBytes;
                uint8_t* sV = sK + Cfg::kKBytes;
#pragma unroll
                for (int blk = 0; blk < NB; ++blk) {
                    tma_load_4d(sK + blk * (kAtKV * 128), &maps.k, &b.kv_full[st], head * HD + blk * 64,
                                u.k_row + t * kAtKV, 0, 0);
                    tma_load_4d(sV + blk * (kAtKV * 128), &maps.v, &b.kv_full[st], head * HD + blk * 64,
                                u.k_row + t * kAtKV, 0, 0);
                }
            }
            more = it.next();
        }
    }
}

template <int HD, int MASKED>
int launch_attn(const AttnMaps& maps, const AttnArgs& a, int pairs, cudaStream_t st) {
    using Cfg = AtCfg<HD>;
    static unsigned long long attr_done = 0;   // per device
    auto kern = attn_tc_kernel<HD, MASKED>;
    if (first_launch_on_device(&attr_done)) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
        if (e != cudaSuccess) {
            set_error("attention: cudaFuncSetAttribute(smem=%d): %s", Cfg::kSmemBytes, cudaGetErrorString(e));
            return 1;
        }
    }
    const int grid = pairs < num_sms() ? pairs : num_sms();
    kern<<<grid, kAtThreads, Cfg::kSmemBytes, st>>>(maps, a);
    return 0;
}

}  // namespace

int launch_attention_tc(const void* Q, long long ldq, long long q_rows, const void* K, const void* V, long long ldkv,
                        long long kv_rows, void* O, long long ldo, const SeqDesc* seqs, int nseq, int heads,
                        int head_dim, int masked, cudaStream_t st) {
    if (nseq <= 0) return 0;
    if (head_dim != 32 && head_dim != 48 && head_dim != 64 && head_dim != 96) {
        set_error("attention: head_dim %d unsupported (32/48/64/96)", head_dim);
        return 1;
    }
    if ((ldq % 8) || (ldkv % 8) || (ldo % 8)) {
        set_error("attention: row pitches must keep rows 16-byte aligned (%lld, %lld, %lld)", ldq, ldkv, ldo);
        return 1;
    }
    AttnMaps maps;
    const uint64_t cols = static_cast<uint64_t>(heads) * head_dim;
    {
        // columns beyond heads*head_dim and rows beyond the matrix are zero-filled by TMA (the second 64-column block of
        // the last 96-wide head reads 32 such columns; key tiles read rows of the next sequence, masked in the softmax)
        uint64_t dims[4] = {cols, static_cast<uint64_t>(q_rows), 1, 1};
        uint64_t strides[3] = {static_cast<uint64_t>(ldq) * 2, static_cast<uint64_t>(ldq) * 2 * q_rows,
                               static_cast<uint64_t>(ldq) * 2 * q_rows};
        uint32_t box[4] = {64, static_cast<uint32_t>(kAtQ), 1, 1};
        if (make_tmap_op_4d(&maps.q, Q, dims, strides, box)) return 1;
    }
    {
        uint64_t dims[4] = {cols, static_cast<uint64_t>(kv_rows), 1, 1};
        uint64_t strides[3] = {static_cast<uint64_t>(ldkv) * 2, static_cast<uint64_t>(ldkv) * 2 * kv_rows,
                               static_cast<uint64_t>(ldkv) * 2 * kv_rows};
        uint32_t box[4] = {64, static_cast<uint32_t>(kAtKV), 1, 1};
        if (make_tmap_op_4d(&maps.k, K, dims, strides, box)) return 1;
        if (make_tmap_op_4d(&maps.v, V, dims, strides, box)) return 1;
    }
    AttnArgs a;
    a.seqs = seqs;
    a.nseq = nseq;
    a.heads = heads;
    a.ldkv = ldkv;
    a.scale_log2 = 1.4426950408889634f / sqrtf(static_cast<float>(head_dim));
    a.O = reinterpret_cast<op_t*>(O);
    a.ldo = ldo;
    const int pairs = nseq * heads;
    int rc = 0;
#define YTK_AT(HD_)                                                  \
    do {                                                             \
        if (masked) rc = launch_attn<HD_, 1>(maps, a, pairs, st);    \
        else rc = launch_attn<HD_, 0>(maps, a, pairs, st);           \
    } while (0)
    switch (head_dim) {
        case 32: YTK_AT(32); break;
        case 48: YTK_AT(48); break;
        case 64: YTK_AT(64); break;
        default: YTK_AT(96); break;
    }
#undef YTK_AT
    if (rc) return 1;
    count_launch();
    if (cudaGetLastError() != cudaSuccess) {
        set_error("attention kernel launch failed");
        return 1;
    }
    return 0;
}

}  // namespace ytk
