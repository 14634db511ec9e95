// Attention on wgmma tensor cores for packed ragged sequences (sm_90a): softmax(Q K^T / sqrt(hd)) V per
// (sequence, head) - the encoder self-attention of PARSeq's ViT (timm Attention / F.scaled_dot_product_attention, no
// mask; reference models/layers/parseq_transformer.py:206-234) and the two attentions of the refinement pass
// (reference models/parseq.py:264-299: cross-attention over the encoder memory, and the masked self-attention over the
// content stream whose mask has rows 0 and 1 cleared, SURVEY.md Appendix A1).
//
// One persistent CTA per SM works through its list of units (sequence, head, 64-query tile).  Every consumer
// warpgroup owns whole units: unit n of the CTA belongs to warpgroup n % 3, which has its own Q buffer and barrier
// phases and computes no rows outside its tile.  Up to three consecutive units of one (sequence, head) pair form a
// chunk; the chunk's K/V tiles are loaded once into a shared ring and read by every warpgroup of the chunk.
//   warp 12  lane 0 : TMA producer - per chunk the Q tile of each unit, then the K/V tiles of 64 keys (SWIZZLE_128B
//                     boxes).  Every consumer warp passes every K/V tile in order, also those it does not read (not in
//                     the chunk, or its causal range ends earlier).  The ring is deeper than a chunk at the bench's
//                     lengths: the next chunk's loads run while this one computes.
//   warpgroups 0-2  : 64 queries each.  S = Q K^T by wgmma (both operands K-major in shared memory) into registers,
//                     mask + running max (lazy rescale: the reference max moves only when it grows by > 2^8) + exp2 in
//                     the accumulator layout, P packed to fp16 A fragments in registers, O += P V by wgmma with A from
//                     registers and V as MN-major B operand (the tile is stored exactly as TMA delivers [keys][hd]
//                     rows); after the last key tile O / l -> global.  S of tile t is issued together with P V of tile
//                     t-1, and the softmax of tile t runs while that P V is on the tensor core (one S and one P register
//                     set: two S sets do not fit the 160 registers a thread of three consumer warpgroups gets).
// The P V product always runs its four 16-key steps; steps past the last visible key read a zero tile instead of V.
#include <cuda.h>

#include "gemm_tc.h"
#include "parseq_ops.h"
#include "ptx.cuh"

namespace ytk {

namespace {

constexpr int kAtQ = 64;         // queries per unit (one warpgroup)
constexpr int kAtKV = 64;        // keys per tile
constexpr int kAtWG = 3;         // consumer warpgroups
constexpr int kAtProducerWarp = 4 * kAtWG;
constexpr int kAtThreads = 128 * (kAtWG + 1);
constexpr int kAtMaxStages = 8;
constexpr int kAtMaxSmem = 227 * 1024;
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
    static constexpr int kQBytes = NB * kAtQ * 128;           // one warpgroup's Q tile
    static constexpr int kKBytes = NB * kAtKV * 128;          // one K (or V) tile
    static constexpr int kStageBytes = 2 * kKBytes;
    static constexpr int kZeroBytes = NB * 2048;               // 16 zero V rows per column block
    static constexpr int kFixedBytes = kAtWG * kQBytes + kZeroBytes + 256 /*barriers*/ + 1024 /*alignment slack*/;
    static constexpr int kStages = (kAtMaxSmem - kFixedBytes) / kStageBytes < kAtMaxStages
                                       ? (kAtMaxSmem - kFixedBytes) / kStageBytes
                                       : kAtMaxStages;
    static constexpr int kSmemBytes = kFixedBytes + kStages * kStageBytes;
    // a warpgroup holds K/V tile t-1 while it waits for t
    static_assert(kStages >= 2, "attention: K/V ring too shallow");
};

struct Unit {
    int q_row;    // first query row of the tile in Q
    int o_row;    // first output row
    int rows;     // valid queries in the tile
    int q0;       // index of the tile's first query inside its sequence
    int k_row;    // first key row in K / V
    int k_end;    // keys this tile can see
    int nt;       // key tiles
};

template <int MASKED>
__device__ __forceinline__ int pair_keys(const SeqDesc& sd) {
    return MASKED ? min(sd.k_len, sd.kpad) : sd.k_len;
}

template <int MASKED>
__device__ __forceinline__ Unit make_unit(const SeqDesc& sd, int qt, long long ldkv) {
    Unit u;
    u.q0 = qt * kAtQ;
    u.q_row = sd.q_off + u.q0;
    u.o_row = sd.o_off + u.q0;
    u.rows = min(kAtQ, sd.q_len - u.q0);
    u.k_row = static_cast<int>(sd.k_base / ldkv);
    int k_end = pair_keys<MASKED>(sd);
    if (MASKED && u.q0 >= 2) k_end = min(k_end, u.q0 + kAtQ);  // causal rows stop at their own index
    u.k_end = k_end;
    u.nt = (k_end + kAtKV - 1) / kAtKV;
    return u;
}

// The chunks of one CTA in processing order: the CTA owns the (sequence, head) pairs p = cta, cta + ncta, ...; a
// pair's query tiles are cut into chunks of up to kAtWG consecutive tiles, run back to back so that the pair's K / V
// is still in L2 for a second chunk.  Units are numbered across the CTA (n0 = number of the chunk's first unit);
// kc0 counts the K/V tiles the ring received before the chunk.  Every role of the CTA walks the same sequence.
template <int MASKED>
struct ChunkIter {
    int p, W, npairs, head, nqt, qt0, cnt, n0, ntiles;
    uint32_t kc0;
    SeqDesc sd;
    const AttnArgs* a;
    __device__ __forceinline__ bool begin(const AttnArgs* args, int cta, int ncta, int npairs_) {
        a = args;
        W = ncta;
        npairs = npairs_;
        p = cta - ncta;
        nqt = qt0 = cnt = n0 = ntiles = 0;
        kc0 = 0;
        return next();
    }
    __device__ __forceinline__ bool next() {
        n0 += cnt;
        kc0 += static_cast<uint32_t>(ntiles);
        qt0 += cnt;
        while (qt0 >= nqt) {
            p += W;
            if (p >= npairs) return false;
            const int seq = p / a->heads;
            head = p - seq * a->heads;
            sd = a->seqs[seq];
            nqt = (sd.q_len > 0 && pair_keys<MASKED>(sd) > 0) ? (sd.q_len + kAtQ - 1) / kAtQ : 0;
            qt0 = 0;
        }
        cnt = min(kAtWG, nqt - qt0);
        ntiles = 0;
        for (int i = 0; i < cnt; ++i) ntiles = max(ntiles, unit(i).nt);
        return true;
    }
    __device__ __forceinline__ Unit unit(int i) const { return make_unit<MASKED>(sd, qt0 + i, a->ldkv); }
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
    constexpr int S = Cfg::kStages;
    extern __shared__ uint8_t at_smem_raw[];
    const uint32_t raw_addr = smem_u32(at_smem_raw);
    uint8_t* smem = at_smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
    uint8_t* sQ = smem;
    uint8_t* sKV = smem + kAtWG * Cfg::kQBytes;
    uint8_t* sZero = sKV + S * Cfg::kStageBytes;
    uint64_t* q_full = reinterpret_cast<uint64_t*>(sZero + Cfg::kZeroBytes);
    uint64_t* q_empty = q_full + kAtWG;
    uint64_t* kv_full = q_empty + kAtWG;
    uint64_t* kv_empty = kv_full + S;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int i = 0; i < kAtWG; ++i) {
            mbar_init(&q_full[i], 1);
            mbar_init(&q_empty[i], 4);       // one arrive per warp of the owning warpgroup
        }
        for (int i = 0; i < S; ++i) {
            mbar_init(&kv_full[i], 1);
            mbar_init(&kv_empty[i], 4 * kAtWG);  // one arrive per consumer warp
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

    if (warp < kAtProducerWarp) {
        // ------------------------------------------------------------------ MMA + softmax + epilogue, 64 queries
        setmaxnreg_inc<160>();   // 3 x 128 x 160 + 128 x 32 = 64 K registers
        const int wg = warp >> 2, wl = warp & 3;
        const int r_in = wl * 16 + (lane >> 2);   // tile row of this thread's first row (second: + 8)
        const int cq = (lane & 3) * 2;            // first of the thread's two columns in every 8-column block
        const uint32_t q_addr = smem_u32(sQ + wg * Cfg::kQBytes);
        // K/V tiles of the chunk that this warpgroup does not read: it still observes every fill of every stage in
        // order (a phase-parity wait is only unambiguous when the waiter has seen the previous phase) and counts itself
        // done with the tile
        auto pass_tiles = [&](uint32_t c, uint32_t end) {
            for (; c < end; ++c) {
                mbar_wait(&kv_full[c % S], (c / S) & 1u);
                __syncwarp();
                if (lane == 0) mbar_arrive(&kv_empty[c % S]);
            }
        };
        ChunkIter<MASKED> it;
        for (bool more = it.begin(&args, cta, ncta, npairs); more; more = it.next()) {
            int i = wg - it.n0 % kAtWG;
            if (i < 0) i += kAtWG;
            if (i >= it.cnt) {
                pass_tiles(it.kc0, it.kc0 + it.ntiles);
                continue;
            }
            const int n = it.n0 + i;   // unit number inside the CTA
            const Unit u = it.unit(i);
            const uint32_t kc0 = it.kc0;
            float m_ref[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
            float o[NO / 2];
#pragma unroll
            for (int j = 0; j < NO / 2; ++j) o[j] = 0.f;
            float s[32];
            uint32_t pa[4][4];
            float factor[2];

            auto release_kv = [&](int t) {   // K / V tile t consumed by this warp
                __syncwarp();
                if (lane == 0) mbar_arrive(&kv_empty[(kc0 + t) % S]);
            };
            auto release_q = [&]() {         // the unit's last S is done: the Q tile may be replaced
                __syncwarp();
                if (lane == 0) mbar_arrive(&q_empty[wg]);
            };
            // ---- S = Q K^T (64 queries x 64 keys) of key tile t, one wgmma group
            auto issue_s = [&](int t) {
                const uint32_t c = kc0 + t, st = c % S;
                mbar_wait(&kv_full[st], (c / S) & 1u);
                const uint32_t k_addr = smem_u32(sKV + st * Cfg::kStageBytes);
                reg_fence(s);
                wgmma_fence();
#pragma unroll
                for (int j = 0; j < HD / 16; ++j) {
                    const uint64_t da = wgmma_desc_sw128(q_addr + (j >> 2) * (kAtQ * 128)) + static_cast<uint64_t>(2 * (j & 3));
                    const uint64_t db = wgmma_desc_sw128(k_addr + (j >> 2) * (kAtKV * 128)) + static_cast<uint64_t>(2 * (j & 3));
                    wgmma_ss<64>(s, da, db, j != 0 ? 1u : 0u);
                }
                wgmma_commit();
            };
            // ---- O += P V of key tile t, one wgmma group.  All four 16-key steps are issued (a wgmma under a branch
            // is serialised); a step past the last visible key has P = 0 and reads the zero tile instead of V rows that
            // belong to no sequence of this unit (their contents need not be finite)
            auto issue_pv = [&](int t) {
                const uint32_t v_addr = smem_u32(sKV + ((kc0 + t) % S) * Cfg::kStageBytes) + Cfg::kKBytes;
                const int ksteps = (min(kAtKV, u.k_end - t * kAtKV) + 15) >> 4;
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
            };
            // ---- softmax of key tile t on S: mask, scale, running max, l; S becomes P = exp2(S - m) in place.  O is
            // not touched (the previous P V may still be running): its rescale by `factor` follows the wait.
            auto softmax = [&](int t) {
                // tile max of both rows (a row is spread over the 4 lanes of a quad)
                const int key0 = t * kAtKV;
                float mt[2] = {-INFINITY, -INFINITY};
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    const int h = (j >> 1) & 1;
                    const int key = key0 + (j >> 2) * 8 + cq + (j & 1);
                    const int qi = u.q0 + r_in + 8 * h;   // query index inside the sequence
                    bool vis = key < u.k_end;
                    if (MASKED) vis = vis && ((qi < 2) || (key <= qi));
                    const float v = vis ? s[j] * args.scale_log2 : -INFINITY;
                    s[j] = v;
                    mt[h] = fmaxf(mt[h], v);
                }
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
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const float m_use = (m_ref[h] == -INFINITY) ? 0.f : m_ref[h];
                    float ls = 0.f;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const float p0 = fast_exp2(s[4 * j + 2 * h] - m_use);  // exp2(-inf) = 0
                        const float p1 = fast_exp2(s[4 * j + 2 * h + 1] - m_use);
                        ls += p0 + p1;
                        s[4 * j + 2 * h] = p0;
                        s[4 * j + 2 * h + 1] = p1;
                    }
                    l_run[h] += ls;
                }
            };
            // ---- P as fp16 A fragments (k step ks covers keys 16 ks .. 16 ks + 15), O rescaled to the new max
            auto pack_rescale = [&]() {
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int j = 0; j < 8; ++j) pa[j >> 1][(j & 1) * 2 + h] = pack_op(s[4 * j + 2 * h], s[4 * j + 2 * h + 1]);
                if (factor[0] != 1.f || factor[1] != 1.f) {
#pragma unroll
                    for (int j = 0; j < NO / 2; ++j) o[j] *= factor[(j >> 1) & 1];
                }
            };

            mbar_wait(&q_full[wg], (n / kAtWG) & 1u);
            issue_s(0);
            wgmma_wait<0>();
            reg_fence(s);
            if (u.nt == 1) release_q();
            softmax(0);
            pack_rescale();
            // key tile t: S(t) and P(t-1) V(t-1) go to the tensor core together; the softmax of tile t runs while
            // P(t-1) V(t-1) is still on it
            for (int t = 1; t < u.nt; ++t) {
                issue_s(t);
                issue_pv(t - 1);
                wgmma_wait<1>();
                reg_fence(s);
                if (t == u.nt - 1) release_q();
                softmax(t);
                wgmma_wait<0>();
                reg_fence(o);
                release_kv(t - 1);
                pack_rescale();
            }
            issue_pv(u.nt - 1);
            wgmma_wait<0>();
            reg_fence(o);
            release_kv(u.nt - 1);
            pass_tiles(kc0 + u.nt, kc0 + it.ntiles);   // masked: a later query tile of the chunk sees more keys
            // ---- epilogue: O / l -> global
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
                l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
                const int r = r_in + 8 * h;
                if (r < u.rows) {
                    const float inv = l_run[h] > 0.f ? 1.f / l_run[h] : 0.f;
                    op_t* op = args.O + static_cast<long long>(u.o_row + r) * args.ldo + it.head * HD + cq;
#pragma unroll
                    for (int j = 0; j < HD / 8; ++j)
                        *reinterpret_cast<uint32_t*>(op + 8 * j) = pack_op(o[4 * j + 2 * h] * inv, o[4 * j + 2 * h + 1] * inv);
                }
            }
        }
    } else {
        // ------------------------------------------------------------------ TMA producer
        setmaxnreg_dec<32>();
        if (warp == kAtProducerWarp && lane == 0) {
            ChunkIter<MASKED> it;
            for (bool more = it.begin(&args, cta, ncta, npairs); more; more = it.next()) {
                const int head = it.head;
#pragma unroll
                for (int i = 0; i < kAtWG; ++i) {
                    if (i < it.cnt) {
                        const int n = it.n0 + i;
                        const int w = n % kAtWG;
                        const Unit u = it.unit(i);
                        mbar_wait(&q_empty[w], ((n / kAtWG) & 1u) ^ 1u);
                        mbar_expect_tx(&q_full[w], Cfg::kQBytes);
#pragma unroll
                        for (int blk = 0; blk < NB; ++blk)
                            tma_load_4d(sQ + w * Cfg::kQBytes + blk * (kAtQ * 128), &maps.q, &q_full[w],
                                        head * HD + blk * 64, u.q_row, 0, 0);
                    }
                }
                const int k_row = static_cast<int>(it.sd.k_base / args.ldkv);
                for (int t = 0; t < it.ntiles; ++t) {
                    const uint32_t c = it.kc0 + t, st = c % S;
                    mbar_wait(&kv_empty[st], ((c / S) & 1u) ^ 1u);
                    mbar_expect_tx(&kv_full[st], Cfg::kStageBytes);
                    uint8_t* sK = sKV + st * Cfg::kStageBytes;
                    uint8_t* sV = sK + Cfg::kKBytes;
#pragma unroll
                    for (int blk = 0; blk < NB; ++blk) {
                        tma_load_4d(sK + blk * (kAtKV * 128), &maps.k, &kv_full[st], head * HD + blk * 64,
                                    k_row + t * kAtKV, 0, 0);
                        tma_load_4d(sV + blk * (kAtKV * 128), &maps.v, &kv_full[st], head * HD + blk * 64,
                                    k_row + t * kAtKV, 0, 0);
                    }
                }
            }
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
