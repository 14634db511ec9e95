// wgmma implicit-GEMM convolution / linear kernel for sm_90a.  See gemm_tc.h for the contract.
//
// Warp roles (384 threads, 1 CTA per SM, persistent over output tiles):
//   warp 8      : TMA producer  (one elected lane) - A patch box + W box per 64-wide K block, STAGES-deep ring; the
//                 producer warpgroup (warps 8..11) hands its registers to the consumers (setmaxnreg)
//   warps 0..7  : two consumer warpgroups          - each: 4 x wgmma (K=16) per K block into a 64 x BLOCK_N register
//                                                    accumulator (tile rows 64 wg ..), then the epilogue of those rows:
//                                                    bias/residual/activation -> TMA boxes (residual in by
//                                                    cp.async.bulk.tensor, result out by TMA store) or, for the plans
//                                                    the TMA path does not cover, staged per-thread global accesses
// Pipelines: smem full/empty mbarriers (TMA <-> MMA) and, in the TMA epilogue, one mbarrier per residual box of every
// epilogue warp's ring.  The producer runs ahead into the next tile's K blocks while the consumers store.
#include "gemm_tc.h"

#include <cstdarg>
#include <cstdlib>
#include <cstdio>
#include <cstring>
#include <atomic>
#include <mutex>
#include <vector>

#include "ptx.cuh"

namespace ytk {

// ------------------------------------------------------------------------------------------------ errors
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
const char* last_error() { return g_err; }

static std::atomic<long long> g_launches{0};
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
long long launch_count() { return g_launches.load(std::memory_order_relaxed); }

int pdl_launch_attr(cudaLaunchAttribute* attr) {
    // Opt-in (YTK_PDL=1): a dependent persistent GEMM CTA that becomes resident early takes its SM away from the
    // remaining waves of the multi-wave kernel before it, which can cost more than the overlapped prologue saves.  The kernels keep their griddepcontrol.wait (a no-op for a
    // normal launch) so that the experiment stays one environment variable away.
    static const bool on = getenv("YTK_PDL") != nullptr && getenv("YTK_NO_PDL") == nullptr;
    if (!on) return 0;
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    return 1;
}

bool first_launch_on_device(unsigned long long* mask) {
    int d = 0;
    cudaGetDevice(&d);
    const unsigned long long bit = 1ull << (d & 63);
    if (*mask & bit) return false;
    *mask |= bit;     // two threads racing here both set the attribute: harmless
    return true;
}

int num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
    }
    return n;
}

// ------------------------------------------------------------------------------------------------ kernel
constexpr int kBlockM = 128;
constexpr int kBlockK = 64;  // 64 16-bit elements = 128 B = one swizzle row
constexpr int kABytes = kBlockM * kBlockK * 2;
constexpr int kThreads = 384;       // warps 0..7: two consumer warpgroups (MMA + epilogue), warps 8..11: TMA producer
constexpr int kProducerWarp = 8;
constexpr int kStagePitch = 80;     // bytes per staged row: 64 B payload + 16 B pad (conflict-free 16 B accesses)
constexpr int kEpiStageBytes = 8 * 32 * kStagePitch;
// Accumulator hand-off: a warpgroup's 64 x BLOCK_N accumulator lives in its registers in the wgmma fragment layout, the
// epilogue works on one output row per thread.  64-column slices pass through a per-warpgroup buffer
// [64 rows][kAccPitch fp32] (pitch 68 words: the row-per-thread 16-byte reads are conflict-free).
constexpr int kAccPitch = 68;
constexpr int kAccBytes = 2 * 64 * kAccPitch * 4;

// TMA epilogue (DIRECT == 2): works on the accumulator fragments directly (no slice buffer).  Every epilogue warp owns
// a ring of kEpiTmaBufs 2 KB buffers (16 tile rows x 128 bytes, 128-byte swizzled = the layout a TMA box of that shape
// has in shared memory).  With a residual, the boxes of the next three passes are in flight (the first ones of a tile
// load while its MMAs run) while one is being stored; without one they buffer the TMA stores.  Four boxes per warp
// fit in the bytes the slice buffer used to take, so every tile width keeps its K stages.
constexpr int kEpiBufBytes = 16 * 128;
constexpr int kEpiTmaBufs = 4;
constexpr int kSmemLimit = 232448;  // 227 KB of dynamic shared memory per CTA
constexpr int kSmemFixed = 1024 /*final-conv weights*/ + 1024 /*align slack*/ + 512 /*barriers*/;

template <int BLOCK_N, int EPI_BYTES = kEpiStageBytes, int ACC_BYTES = kAccBytes>
struct TileCfg {
    static constexpr int kBBytes = BLOCK_N * kBlockK * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kAccB = ACC_BYTES;   // accumulator slice buffers (none in the TMA epilogue)
    static constexpr int kRingBudget = kSmemLimit - kSmemFixed - ACC_BYTES - EPI_BYTES;
    static constexpr int kStages = (kRingBudget / kStageBytes) > 8 ? 8 : (kRingBudget / kStageBytes);
    static constexpr int kRingBytes = kStages * kStageBytes;
    static constexpr int kSmemBytes = kRingBytes + ACC_BYTES + EPI_BYTES + kSmemFixed;
    static_assert(kStages >= 3, "K pipeline depth");
    static_assert(kSmemBytes <= kSmemLimit, "shared memory budget");
    static_assert((kRingBytes + ACC_BYTES) % 2048 == 0, "epilogue buffers must stay 2 KB aligned");
};

// 16-bit 8x8 matrix moves between shared memory and the mma fragment layout (thread t: row t / 4, columns 2 (t % 4),
// +1); lane l gives the row address of matrix l / 8
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
                 : "r"(addr)
                 : "memory");
}
__device__ __forceinline__ void stsm_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
    asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1),
                 "r"(r2), "r"(r3)
                 : "memory");
}

// ragged last columns of a row segment: element-wise copy (rare; kept out of line)
__device__ __noinline__ void copy_elems(void* dst, const void* src, int n, int esz) {
    if (esz == 4)
        for (int e = 0; e < n; ++e) reinterpret_cast<uint32_t*>(dst)[e] = reinterpret_cast<const uint32_t*>(src)[e];
    else
        for (int e = 0; e < n; ++e) reinterpret_cast<uint16_t*>(dst)[e] = reinterpret_cast<const uint16_t*>(src)[e];
}
// Exact (erf) GELU, fp32, max |error| 5e-7 (2.8e-7 for |x| < 3; the form it replaces, Abramowitz-Stegun 7.1.26, had
// 0.5 |x| 1.5e-7):
//     GELU(x) = max(x, 0) - 0.5 t erfc(t / sqrt 2),   t = min(|x|, 5.7),   erfc(t / sqrt 2) = 2 ^ (t P(t))
// P = degree-6 weighted minimax fit (experiments/gelu_fit.py).  One ex2 per element, no reciprocal: the fc1 epilogue is
// bound by instruction issue, this form needs about half the instructions of a rational erf.
__device__ __forceinline__ float gelu_fast(float x) {
    const float t = fminf(fabsf(x), 5.7f);
    float p = fmaf(4.278742836e-06f, t, -1.279820572e-05f);
    p = fmaf(p, t, -5.757861654e-04f);
    p = fmaf(p, t, 7.670783438e-03f);
    p = fmaf(p, t, -5.294856429e-02f);
    p = fmaf(p, t, -4.590439200e-01f);
    p = fmaf(p, t, -1.151126981e+00f);
    const float a = __fmul_rn(p, t);
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(a));
    return fmaf(__fmul_rn(t, -0.5f), e, fmaxf(x, 0.f));
}
__device__ __forceinline__ void gelu_fast2(float& x0, float& x1) {
    x0 = gelu_fast(x0);
    x1 = gelu_fast(x1);
}

struct TileCoord {
    int img, h0, w0, n0;
};
__device__ __forceinline__ TileCoord decode_tile(const GemmArgs& a, int tile, int block_n) {
    TileCoord t;
    int m_tile = tile / a.tiles_n;
    int n_tile = tile - m_tile * a.tiles_n;
    int tw = m_tile % a.tiles_w;
    int t2 = m_tile / a.tiles_w;
    int th = t2 % a.tiles_h;
    t.img = t2 / a.tiles_h;
    t.h0 = th * (kBlockM >> a.bw_log2);
    t.w0 = tw << a.bw_log2;
    t.n0 = n_tile * block_n;
    return t;
}

// Epilogue variants are compile-time (OUT_F32: fp32 vs 16-bit output; RESID: 0 none, 1 16-bit, 2 fp32; MODE: EpiMode)
// so that each instantiation carries only its own store path - one kernel with every path inlined thrashes the
// instruction cache.
template <int BLOCK_N, int RESID, int DIRECT>
using KernelCfg = TileCfg<BLOCK_N, DIRECT == 2 ? 8 * kEpiTmaBufs * kEpiBufBytes : kEpiStageBytes,
                          DIRECT == 2 ? 0 : kAccBytes>;

// DIRECT: 0 = staged epilogue (registers -> per-warp shared staging -> coalesced per-thread global accesses),
//         1 = row per thread straight to global memory (A/B aid, not dispatched),
//         2 = TMA epilogue (EPI_NORMAL only): residual boxes arrive by TMA, results leave by TMA store.
template <int BLOCK_N, int OUT_F32, int RESID, int MODE, int DIRECT>
__global__ void __launch_bounds__(kThreads, 1) gemm_tc_kernel(const __grid_constant__ GemmMaps maps,
                                                              const __grid_constant__ GemmArgs args) {
    using Cfg = KernelCfg<BLOCK_N, RESID, DIRECT>;
    constexpr int kEpiBytes = Cfg::kSmemBytes - Cfg::kRingBytes - Cfg::kAccB - kSmemFixed;
    constexpr int stage_bytes = Cfg::kStageBytes;
    constexpr int nstages = Cfg::kStages;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw_addr = smem_u32(smem_raw);
    uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);  // 1024 B alignment for SWIZZLE_128B
    const int worker = static_cast<int>(blockIdx.x);
    const int n_workers = static_cast<int>(gridDim.x);

    float* acc_smem = reinterpret_cast<float*>(smem + Cfg::kRingBytes);
    uint8_t* epi_stage = smem + Cfg::kRingBytes + Cfg::kAccB;
    float* fin_w = reinterpret_cast<float*>(epi_stage + kEpiBytes);  // [4][64] weights of the fused final conv
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(epi_stage + kEpiBytes + 1024);
    uint64_t* empty_bar = full_bar + 8;
    [[maybe_unused]] uint64_t* rbar_base = empty_bar + 8;  // TMA epilogue: [8 warps][4] residual-box barriers

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int i = 0; i < nstages; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 8);  // one arrive per consumer warp
        }
        if constexpr (DIRECT == 2 && RESID != 0) {
            for (int i = 0; i < 32; ++i) mbar_init(&rbar_base[i], 1);
        }
        fence_mbar_init();
        tma_prefetch_desc(&maps.a[0]);
        tma_prefetch_desc(&maps.b);
        if constexpr (DIRECT == 2) {
            tma_prefetch_desc(&maps.out);
            if constexpr (RESID != 0) {
                tma_prefetch_desc(&maps.resid);
                tma_prefetch_desc(&maps.resid_pf);
            }
        }
    }
    if constexpr (MODE == EPI_CONVT_FINAL) {
        if (threadIdx.x < 256) fin_w[threadIdx.x] = args.fin_w[threadIdx.x];
    }
    __syncthreads();
    // programmatic dependent launch: the prologue above overlapped the previous kernel's tail; operands, residuals and
    // the output buffer may only be touched from here on
    pdl_wait();
    pdl_launch_dependents();

    const int tiles_m = args.n_img * args.tiles_h * args.tiles_w;
    const int num_kb = args.ntaps * args.kpt;
    const int total_units = tiles_m * args.tiles_n;

    if (warp >= kProducerWarp) {
        // ------------------------------------------------------------------ TMA producer
        setmaxnreg_dec<40>();
        if (warp == kProducerWarp && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            // TMA epilogue with a residual: the rows of the NEXT tile's residual go to L2 as one whole-tile request, so
            // that the epilogue warps' 64-byte boxes hit L2 instead of fetching DRAM piecemeal
            [[maybe_unused]] auto prefetch_resid = [&](int u2) {
                if (u2 >= total_units) return;
                const TileCoord c2 = decode_tile(args, u2, BLOCK_N);
                tma_prefetch_l2_4d(&maps.resid_pf, c2.n0, c2.w0, c2.h0, c2.img);
            };
            if constexpr (DIRECT == 2 && RESID != 0) {
                if (args.epi_pf) prefetch_resid(worker);
            }
            for (int u = worker; u < total_units; u += n_workers) {
                const TileCoord tc = decode_tile(args, u, BLOCK_N);
                if constexpr (DIRECT == 2 && RESID != 0) {
                    if (args.epi_pf) prefetch_resid(u + n_workers);
                }
                int tap = 0, cb = 0;
                for (int kb = 0; kb < num_kb; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1u);
                    uint8_t* sa = smem + stage * stage_bytes;
                    uint8_t* sb = sa + kABytes;
                    const ConvTap tp = args.taps[tap];
                    mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
                    tma_load_4d(sa, &maps.a[tp.map], &full_bar[stage], cb * kBlockK, tc.w0 + tp.dw, tc.h0 + tp.dh,
                                tc.img);
                    tma_load_4d(sb, &maps.b, &full_bar[stage], kb * kBlockK, tc.n0, 0, 0);
                    if (++cb == args.kpt) {
                        cb = 0;
                        ++tap;
                    }
                    if (++stage == nstages) {
                        stage = 0;
                        phase ^= 1u;
                    }
                }
            }
        }
    } else {
        // ------------------------------------------------------------------ consumers (warps 0..7)
        // Warpgroup wg computes tile rows [64 wg, 64 wg + 64) with wgmma, then runs the epilogue on them.  The TMA
        // epilogue (DIRECT == 2, below) works on each warp's own 16 fragment rows.  The staged one: warp wl of the
        // warpgroup stores the 32 rows of quadrant q (row per thread) and, of every 64-column slice, the 32-column chunk
        // of its set (the CONVT_FINAL epilogue pairs chunks instead, see below).  Values go registers -> slice buffer ->
        // bias/residual/activation -> per-warp shared staging and coalesced 16-byte global accesses (4 lanes per 64-byte
        // row segment), so DRAM sees whole sectors.
        setmaxnreg_inc<232>();   // 2 x 128 x 232 + 128 x 40 <= 64 K registers
        const int wg = warp >> 2, wl = warp & 3;
        const int q = 2 * wg + (wl & 1);   // 32-row quadrant of the tile this warp stores
        const int wset = wl >> 1;          // 0 or 1
        float* acc_buf = acc_smem + wg * 64 * kAccPitch;
        const float* my_acc = acc_buf + ((wl & 1) * 32 + lane) * kAccPitch;
        float acc[BLOCK_N / 2];
#pragma unroll
        for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
        int ring_stage = 0;
        uint32_t ring_phase = 0;
        // the whole K loop of one tile: one wgmma group per K block, one group kept in flight; a stage is released
        // once the group after it has been issued and its own group has completed
        auto mma_tile = [&]() {
            const uint32_t a_off = static_cast<uint32_t>(wg * 64 * 128);
            int prev = -1;
            for (int kb = 0; kb < num_kb; ++kb) {
                mbar_wait(&full_bar[ring_stage], ring_phase);
                const uint32_t a_addr = smem_u32(smem + ring_stage * stage_bytes);
                const uint64_t da = wgmma_desc_sw128(a_addr + a_off);
                const uint64_t db = wgmma_desc_sw128(a_addr + kABytes);
                reg_fence(acc);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < kBlockK / 16; ++k)
                    // advance 16 elements = 32 B inside the 128 B swizzle row: +2 in the (addr >> 4) field
                    wgmma_ss<BLOCK_N>(acc, da + static_cast<uint64_t>(2 * k), db + static_cast<uint64_t>(2 * k),
                                      (kb | k) != 0 ? 1u : 0u);
                wgmma_commit();
                wgmma_wait<1>();
                reg_fence(acc);
                if (prev >= 0) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty_bar[prev]);
                }
                prev = ring_stage;
                if (++ring_stage == nstages) {
                    ring_stage = 0;
                    ring_phase ^= 1u;
                }
            }
            wgmma_wait<0>();
            reg_fence(acc);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[prev]);
        };
        // accumulator columns [64 s, 64 s + 64) -> the warpgroup's slice buffer, once every warp is done with the last
        // slice (register indices must be compile-time: the slice is selected by predicate)
        auto dump_slice = [&](int s) {
            named_bar_sync(1 + wg, 128);
            const int r0 = wl * 16 + (lane >> 2), c2 = (lane & 3) * 2;
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j) {
                if ((j >> 3) == s) {
                    float* p = acc_buf + r0 * kAccPitch + (j & 7) * 8 + c2;
                    *reinterpret_cast<float2*>(p) = make_float2(acc[4 * j], acc[4 * j + 1]);
                    *reinterpret_cast<float2*>(p + 8 * kAccPitch) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
                }
            }
            named_bar_sync(1 + wg, 128);
        };
        // this thread's row of 32-column chunk c (after dump_slice(c / 2))
        auto load_chunk = [&](int c, float (&f)[32]) {
            const float4* a4 = reinterpret_cast<const float4*>(my_acc + (c & 1) * 32);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float4 x = a4[j];
                f[4 * j + 0] = x.x;
                f[4 * j + 1] = x.y;
                f[4 * j + 2] = x.z;
                f[4 * j + 3] = x.w;
            }
        };
        if constexpr (DIRECT == 2) {
            // ---- TMA epilogue, straight from the wgmma fragments.  Warp w (= 4 wg + wl) holds tile rows 16 w + lane / 4
            // (+ 8) and, of every 8-column group j, columns 8 j + 2 (lane % 4) (+ 1).  A "pass" is 128 bytes of columns of
            // those 16 rows: one 2 KB box, 128-byte swizzled (16-byte chunk ^= row % 8), which the warp reads (residual)
            // and writes (result) in the fragment layout - ldmatrix / stmatrix for 16-bit boxes, float2 accesses for
            // fp32 ones, all conflict-free - before lane 0 hands it to a TMA store.  The warp's passes (units ->
            // passes) form one sequence that indexes a ring of NBUF boxes: residual boxes are loaded LOOK passes ahead
            // by lane 0 (the first ones of a tile while its MMAs run).  Rows / columns outside the tensor are
            // zero-filled on load and dropped on store by the hardware.  Per element: (acc + bias) + residual, then the
            // activation, then rounding - the order of the staged epilogue, so both give the same bits.
            static_assert(MODE == EPI_NORMAL, "TMA epilogue: plain stores only");
            static_assert(RESID == 0 || (RESID == 2) == (OUT_F32 != 0), "TMA epilogue: residual and output boxes match");
            constexpr int NBUF = kEpiTmaBufs;
            static_assert(NBUF <= 4, "residual barriers: 4 per warp");
            constexpr int LOOK = NBUF - 1;
            constexpr int CPB = OUT_F32 ? 32 : 64;   // columns per box (128 bytes)
            constexpr int JPB = CPB / 8;             // 8-column fragment groups per box
            constexpr int NPASS = BLOCK_N / CPB;
            const int tr0 = warp * 16;               // first tile row of the warp
            const int bw_mask = (1 << args.bw_log2) - 1;
            const int qw = tr0 & bw_mask;            // where the warp's 16 rows start inside the BH x BW patch
            const int qh = tr0 >> args.bw_log2;
            uint8_t* bufs = epi_stage + warp * (NBUF * kEpiBufBytes);
            [[maybe_unused]] uint64_t* rbar = rbar_base + warp * 4;
            const int swz = args.epi_swz ? 7 : 0;
            const int fr = lane >> 2;                // fragment row (and fr + 8)
            const int fc = (lane & 3) * 2;           // fragment column inside an 8-column group
            // fp32 box: byte offset of (row fr, column 8 jj + fc) is f32_off + (((2 jj) ^ row) << 4) with the low chunk
            // bit folded in below; row fr + 8 is 1024 bytes further (same swizzle phase)
            const int f32_sub = (lane >> 1) & 1, f32_byte = (lane & 1) * 8;
            // 16-bit box, ldmatrix / stmatrix x4 over groups (2 t, 2 t + 1): lane gives row mrow of 16-byte chunk
            // 2 t + mchunk (matrices: rows 0-7 / 8-15 of group 2 t, then of group 2 t + 1)
            const int mrow = ((lane >> 3) & 1) * 8 + (lane & 7), mchunk = lane >> 4;
            // residual prefetch cursor (lane 0 only): position (unit, pass) of the next box to load
            [[maybe_unused]] int pf_u = worker, pf_p = 0, pf_g = 0;
            [[maybe_unused]] TileCoord pf_tc{};
            [[maybe_unused]] auto pf_seek = [&]() {   // moves the cursor to the next existing pass at or after its position
                while (pf_u < total_units) {
                    pf_tc = decode_tile(args, pf_u, BLOCK_N);
                    if (pf_p < NPASS && pf_tc.n0 + pf_p * CPB < args.Cout) return;
                    pf_p = 0;          // nothing (left) in the unit
                    pf_u += n_workers;
                }
            };
            [[maybe_unused]] auto pf_step = [&]() {
                ++pf_p;
                pf_seek();
            };
            [[maybe_unused]] auto pf_issue = [&]() {
                const int b = pf_g % NBUF;
                mbar_expect_tx(&rbar[b], kEpiBufBytes);
                tma_load_4d(bufs + b * kEpiBufBytes, &maps.resid, &rbar[b], pf_tc.n0 + pf_p * CPB, pf_tc.w0 + qw,
                            pf_tc.h0 + qh, pf_tc.img);
                ++pf_g;
            };
            if constexpr (RESID != 0) {
                if (lane == 0) {
                    pf_seek();
                    for (int k = 0; k < LOOK && pf_u < total_units; ++k) {
                        pf_issue();
                        pf_step();
                    }
                }
            }
            int gc = 0;  // passes consumed so far (warp-uniform)
            for (int u = worker; u < total_units; u += n_workers) {
                const TileCoord tc = decode_tile(args, u, BLOCK_N);
                mma_tile();
                // passes are unrolled: the fragment registers of a pass must be compile-time indices
#pragma unroll
                for (int p = 0; p < NPASS; ++p) {
                    const int col0 = tc.n0 + p * CPB;
                    if (col0 >= args.Cout) break;   // warp-uniform; the cursor above skips the same passes
                    const int b = gc % NBUF;
                    uint8_t* box = bufs + b * kEpiBufBytes;
                    const uint32_t box_s = smem_u32(box);
                    float v[4 * JPB];
#pragma unroll
                    for (int i = 0; i < 4 * JPB; ++i) v[i] = acc[4 * JPB * p + i];
                    if (args.bias != nullptr) {
#pragma unroll
                        for (int jj = 0; jj < JPB; ++jj) {
                            const int col = col0 + 8 * jj + fc;   // Cout is even on this path: col < Cout covers col + 1
                            const float2 bb = col < args.Cout ? __ldg(reinterpret_cast<const float2*>(args.bias + col))
                                                              : make_float2(0.f, 0.f);
                            v[4 * jj + 0] += bb.x;
                            v[4 * jj + 1] += bb.y;
                            v[4 * jj + 2] += bb.x;
                            v[4 * jj + 3] += bb.y;
                        }
                    }
                    if constexpr (RESID != 0) {
                        mbar_wait(&rbar[b], static_cast<uint32_t>(gc / NBUF) & 1u);
                        if constexpr (RESID == 2) {
#pragma unroll
                            for (int jj = 0; jj < JPB; ++jj) {
                                const uint8_t* rp = box + fr * 128 + (((2 * jj + f32_sub) ^ (fr & swz)) << 4) + f32_byte;
                                const float2 r0 = *reinterpret_cast<const float2*>(rp);
                                const float2 r1 = *reinterpret_cast<const float2*>(rp + 1024);
                                v[4 * jj + 0] += r0.x;
                                v[4 * jj + 1] += r0.y;
                                v[4 * jj + 2] += r1.x;
                                v[4 * jj + 3] += r1.y;
                            }
                        } else {
#pragma unroll
                            for (int t = 0; t < JPB / 2; ++t) {
                                uint32_t r0, r1, r2, r3;
                                ldsm_x4(box_s + mrow * 128 + (((2 * t + mchunk) ^ (mrow & swz)) << 4), r0, r1, r2, r3);
                                v[8 * t + 0] += op_lo(r0); v[8 * t + 1] += op_hi(r0);
                                v[8 * t + 2] += op_lo(r1); v[8 * t + 3] += op_hi(r1);
                                v[8 * t + 4] += op_lo(r2); v[8 * t + 5] += op_hi(r2);
                                v[8 * t + 6] += op_lo(r3); v[8 * t + 7] += op_hi(r3);
                            }
                        }
                        __syncwarp();   // every lane has read the residual before the results overwrite the box
                    } else {
                        // the store that used this buffer NBUF passes ago must have read it
                        if (lane == 0) bulk_wait_read<NBUF - 1>();
                        __syncwarp();
                    }
                    if (args.act == ACT_RELU) {
#pragma unroll
                        for (int j = 0; j < 4 * JPB; ++j) v[j] = fmaxf(v[j], 0.f);
                    } else if (args.act == ACT_GELU) {
#pragma unroll
                        for (int j = 0; j < 4 * JPB; j += 2) gelu_fast2(v[j], v[j + 1]);
                    } else if (args.act == ACT_SIGMOID) {
#pragma unroll
                        for (int j = 0; j < 4 * JPB; ++j) v[j] = __fdividef(1.f, 1.f + __expf(-v[j]));
                    } else if (args.act == ACT_SILU) {
#pragma unroll
                        for (int j = 0; j < 4 * JPB; ++j) v[j] = __fdividef(v[j], 1.f + __expf(-v[j]));
                    }
                    if constexpr (OUT_F32) {
#pragma unroll
                        for (int jj = 0; jj < JPB; ++jj) {
                            uint8_t* wp = box + fr * 128 + (((2 * jj + f32_sub) ^ (fr & swz)) << 4) + f32_byte;
                            *reinterpret_cast<float2*>(wp) = make_float2(v[4 * jj + 0], v[4 * jj + 1]);
                            *reinterpret_cast<float2*>(wp + 1024) = make_float2(v[4 * jj + 2], v[4 * jj + 3]);
                        }
                    } else {
#pragma unroll
                        for (int t = 0; t < JPB / 2; ++t)
                            stsm_x4(box_s + mrow * 128 + (((2 * t + mchunk) ^ (mrow & swz)) << 4),
                                    pack_op(v[8 * t + 0], v[8 * t + 1]), pack_op(v[8 * t + 2], v[8 * t + 3]),
                                    pack_op(v[8 * t + 4], v[8 * t + 5]), pack_op(v[8 * t + 6], v[8 * t + 7]));
                    }
                    fence_proxy_async_smem();   // the box just written -> visible to the TMA store
                    __syncwarp();
                    if (lane == 0) {
                        tma_store_4d(&maps.out, box, col0, tc.w0 + qw, tc.h0 + qh, tc.img);
                        bulk_commit();
                        if constexpr (RESID != 0) {
                            if (pf_u < total_units) {
                                // the next box goes where pass gc - 1 was stored from: all but the store just
                                // committed must have read their source
                                bulk_wait_read<1>();
                                pf_issue();
                                pf_step();
                            }
                        }
                    }
                    ++gc;
                }
            }
            if (lane == 0) bulk_wait_read<0>();   // shared memory must outlive the last stores' reads
            __syncwarp();
        } else {
        constexpr bool kFin = (MODE == EPI_CONVT_FINAL);
        constexpr bool kWide = (OUT_F32 != 0) || (RESID == 2);  // 16 columns (64 B of fp32) per staging pass
        constexpr int CPP = kWide ? 16 : 32;
        constexpr int NPASS = 32 / CPP;
        constexpr int OESZ = OUT_F32 ? 4 : 2;
        constexpr int RESZ = (RESID == 2) ? 4 : 2;
        const int row = q * 32 + lane;
        const int bw_mask = (1 << args.bw_log2) - 1;
        uint8_t* stage = epi_stage + warp * (32 * kStagePitch);
        uint8_t* my_row = stage + lane * kStagePitch;
        const int piece = lane & 3;
        for (int u = worker; u < total_units; u += n_workers) {
            const TileCoord tc = decode_tile(args, u, BLOCK_N);
            const int hh = tc.h0 + (row >> args.bw_log2);
            const int ww = tc.w0 + (row & bw_mask);
            const bool row_ok = (hh < args.Ho) && (ww < args.Wo);
            // rows this lane moves in the coalesced phase: rr = it * 8 + lane / 4
            int c_h[4], c_w[4];
            bool c_ok[4];
#pragma unroll
            for (int it = 0; it < 4; ++it) {
                const int rr = q * 32 + it * 8 + (lane >> 2);
                c_h[it] = tc.h0 + (rr >> args.bw_log2);
                c_w[it] = tc.w0 + (rr & bw_mask);
                c_ok[it] = (c_h[it] < args.Ho) && (c_w[it] < args.Wo);
            }
            mma_tile();
            [[maybe_unused]] float dots[4] = {0.f, 0.f, 0.f, 0.f};
            [[maybe_unused]] float rm_m = -INFINITY, rm_s = 0.f;   // EPI_ROWMAX: running (max, sum exp, arg-max)
            [[maybe_unused]] int rm_i = 0x7fffffff;
#pragma unroll 1
            for (int c = 0; c < BLOCK_N / 32; ++c) {
                const int col0 = tc.n0 + c * 32;
                if ((c & 1) == 0) {
                    if (col0 >= args.Cout) break;  // warpgroup-uniform
                    dump_slice(c >> 1);
                }
                if (((kFin ? (c >> 1) : c) & 1) != wset) continue;  // chunk belongs to the other warp set
                if (col0 >= args.Cout) continue;
                // residual prefetch: issue the coalesced global loads of every pass of this chunk before reading the
                // accumulator so that their latency overlaps the accumulator load and the bias math
                // DIRECT variant: the thread's own row segment (32 columns) straight from / to global memory
                [[maybe_unused]] uint4 dres[RESID == 2 ? 8 : 4];
                if constexpr (RESID != 0 && !kFin && DIRECT == 1) {
                    const long long pixo = (static_cast<long long>(tc.img) * args.Ho + hh) * args.Wo + ww;
                    const bool fullc = row_ok && (col0 + 32 <= args.Cout);
                    const uint4* gp = reinterpret_cast<const uint4*>(reinterpret_cast<const char*>(args.resid) +
                                                                     (pixo * args.ldr + col0) * RESZ);
#pragma unroll
                    for (int j = 0; j < (RESID == 2 ? 8 : 4); ++j) dres[j] = fullc ? gp[j] : make_uint4(0, 0, 0, 0);
                }
                [[maybe_unused]] uint4 rres[NPASS][4];
                if constexpr (RESID != 0 && !kFin && DIRECT == 0) {
                    constexpr int per16r = 16 / RESZ;
                    int ocol_r = col0, sub_r = 0;
                    if constexpr (MODE == EPI_SHUFFLE2X) {
                        const int cq = args.Cout >> 2;
                        sub_r = col0 / cq;
                        ocol_r = col0 - sub_r * cq;
                    }
#pragma unroll
                    for (int p = 0; p < NPASS; ++p) {
                        const int validr = min(CPP, args.Cout - (col0 + p * CPP));
                        const int e0 = piece * per16r;
#pragma unroll
                        for (int it = 0; it < 4; ++it) {
                            rres[p][it] = make_uint4(0, 0, 0, 0);
                            if (c_ok[it] && e0 + per16r <= validr) {
                                const long long pixr =
                                    (static_cast<long long>(tc.img) * args.Ho + c_h[it]) * args.Wo + c_w[it];
                                const char* gp = reinterpret_cast<const char*>(args.resid) +
                                                 (pixr * args.ldr + ocol_r + p * CPP + e0) * RESZ;
                                rres[p][it] = *reinterpret_cast<const uint4*>(gp);
                            }
                        }
                    }
                }
                float f[32];
                load_chunk(c, f);
                if (args.bias != nullptr) {
                    if (col0 + 32 <= args.Cout) {
                        const float4* b4 = reinterpret_cast<const float4*>(args.bias + col0);
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            const float4 b = __ldg(b4 + j);
                            f[4 * j + 0] += b.x;
                            f[4 * j + 1] += b.y;
                            f[4 * j + 2] += b.z;
                            f[4 * j + 3] += b.w;
                        }
                    } else {
#pragma unroll
                        for (int j = 0; j < 32; ++j) f[j] += __ldg(args.bias + min(col0 + j, args.Cout - 1));
                    }
                }
                if constexpr (MODE == EPI_ROWMAX) {
                    // chunk statistics over the valid columns, then one merge into the running triple
                    const int nvalid = min(32, args.Cout - col0);
                    float cm = -INFINITY;
                    int ci = 0x7fffffff;
#pragma unroll
                    for (int j = 0; j < 32; ++j) {
                        const float v = j < nvalid ? f[j] : -INFINITY;
                        f[j] = v;
                        if (v > cm) {            // strict: the smallest index wins among equals (ascending j)
                            cm = v;
                            ci = col0 + j;
                        }
                    }
                    float cs = 0.f;
                    if (args.act != ACT_RELU) {
#pragma unroll
                        for (int j = 0; j < 32; ++j) cs += __expf(f[j] - cm);   // exp(-inf) = 0 for masked columns
                    }
                    if (cm > rm_m) {             // chunks arrive in ascending column order: ties keep the earlier index
                        rm_s = rm_s * __expf(rm_m - cm) + cs;
                        rm_m = cm;
                        rm_i = ci;
                    } else {
                        rm_s += cs * __expf(cm - rm_m);
                    }
                } else if constexpr (kFin) {
                    // fused ConvTranspose2d(64->1, 2, 2) + sigmoid: this chunk holds 32 of the 64 channels of output
                    // pixel (2h+i, 2w+j) of the first transposed conv (after BN+ReLU)
                    const int chan0 = (c & 1) * 32;
#pragma unroll
                    for (int j = 0; j < 32; ++j) {
                        const float x = fmaxf(f[j], 0.f);
#pragma unroll
                        for (int k = 0; k < 4; ++k) dots[k] += x * fin_w[k * 64 + chan0 + j];
                    }
                    if (c & 1) {
                        if (row_ok) {
                            const int sub = c >> 1;  // (i, j) of the first transposed conv
                            const long long oy = 2LL * (2 * hh + (sub >> 1)), ox = 2LL * (2 * ww + (sub & 1));
                            float* op = reinterpret_cast<float*>(args.out) +
                                        (static_cast<long long>(tc.img) * (4 * args.Ho) + oy) * (4LL * args.Wo) + ox;
                            float2 r0, r1;
                            r0.x = 1.f / (1.f + __expf(-(dots[0] + args.fin_b)));
                            r0.y = 1.f / (1.f + __expf(-(dots[1] + args.fin_b)));
                            r1.x = 1.f / (1.f + __expf(-(dots[2] + args.fin_b)));
                            r1.y = 1.f / (1.f + __expf(-(dots[3] + args.fin_b)));
                            *reinterpret_cast<float2*>(op) = r0;
                            *reinterpret_cast<float2*>(op + 4LL * args.Wo) = r1;
                        }
                        dots[0] = dots[1] = dots[2] = dots[3] = 0.f;
                    }
                } else if constexpr (DIRECT == 1) {
                    int ocol = col0, sub = 0;
                    long long opix = (static_cast<long long>(tc.img) * args.Ho + hh) * args.Wo + ww;
                    if constexpr (MODE == EPI_SHUFFLE2X) {
                        const int cq = args.Cout >> 2;
                        sub = col0 / cq;
                        ocol = col0 - sub * cq;
                        opix = (static_cast<long long>(tc.img) * (2 * args.Ho) + (2 * hh + (sub >> 1))) * (2LL * args.Wo) +
                               (2 * ww + (sub & 1));
                    }
                    const bool fullc = (col0 + 32 <= args.Cout);
                    if constexpr (RESID == 2) {
                        if (fullc) {
#pragma unroll
                            for (int j = 0; j < 8; ++j) {
                                f[4 * j + 0] += __uint_as_float(dres[j].x);
                                f[4 * j + 1] += __uint_as_float(dres[j].y);
                                f[4 * j + 2] += __uint_as_float(dres[j].z);
                                f[4 * j + 3] += __uint_as_float(dres[j].w);
                            }
                        } else if (row_ok) {
                            const float* rp = reinterpret_cast<const float*>(args.resid) + opix * args.ldr + ocol;
#pragma unroll
                            for (int j = 0; j < 32; ++j)
                                if (col0 + j < args.Cout) f[j] += rp[j];
                        }
                    } else if constexpr (RESID == 1) {
                        if (fullc) {
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                f[8 * j + 0] += op_lo(dres[j].x); f[8 * j + 1] += op_hi(dres[j].x);
                                f[8 * j + 2] += op_lo(dres[j].y); f[8 * j + 3] += op_hi(dres[j].y);
                                f[8 * j + 4] += op_lo(dres[j].z); f[8 * j + 5] += op_hi(dres[j].z);
                                f[8 * j + 6] += op_lo(dres[j].w); f[8 * j + 7] += op_hi(dres[j].w);
                            }
                        } else if (row_ok) {
                            const op_t* rp =
                                reinterpret_cast<const op_t*>(args.resid) + opix * args.ldr + ocol;
#pragma unroll
                            for (int j = 0; j < 32; ++j)
                                if (col0 + j < args.Cout) f[j] += op2f(rp[j]);
                        }
                    }
                    if (args.act == ACT_RELU) {
#pragma unroll
                        for (int j = 0; j < 32; ++j) f[j] = fmaxf(f[j], 0.f);
                    } else if (args.act == ACT_GELU) {
#pragma unroll
                        for (int j = 0; j < 32; j += 2) gelu_fast2(f[j], f[j + 1]);
                    } else if (args.act == ACT_SIGMOID) {
#pragma unroll
                        for (int j = 0; j < 32; ++j) f[j] = __fdividef(1.f, 1.f + __expf(-f[j]));
                    } else if (args.act == ACT_SILU) {
#pragma unroll
                        for (int j = 0; j < 32; ++j) f[j] = __fdividef(f[j], 1.f + __expf(-f[j]));
                    }
                    if (row_ok) {
                        if constexpr (OUT_F32) {
                            float* op = reinterpret_cast<float*>(args.out) + opix * args.ldc + ocol;
                            if (fullc) {
#pragma unroll
                                for (int j = 0; j < 8; ++j)
                                    reinterpret_cast<float4*>(op)[j] =
                                        make_float4(f[4 * j], f[4 * j + 1], f[4 * j + 2], f[4 * j + 3]);
                            } else {
#pragma unroll
                                for (int j = 0; j < 32; ++j)
                                    if (col0 + j < args.Cout) op[j] = f[j];
                            }
                        } else {
                            op_t* op = reinterpret_cast<op_t*>(args.out) + opix * args.ldc + ocol;
                            if (fullc) {
#pragma unroll
                                for (int j = 0; j < 4; ++j) {
                                    uint4 o;
                                    o.x = pack_op(f[8 * j + 0], f[8 * j + 1]);
                                    o.y = pack_op(f[8 * j + 2], f[8 * j + 3]);
                                    o.z = pack_op(f[8 * j + 4], f[8 * j + 5]);
                                    o.w = pack_op(f[8 * j + 6], f[8 * j + 7]);
                                    reinterpret_cast<uint4*>(op)[j] = o;
                                }
                            } else {
#pragma unroll
                                for (int j = 0; j < 32; ++j)
                                    if (col0 + j < args.Cout) op[j] = f2op(f[j]);
                            }
                        }
                    }
                } else {
                    // output location of this chunk (the pixel index is remapped by the pixel-shuffle mode)
                    int ocol = col0, sub = 0;
                    if constexpr (MODE == EPI_SHUFFLE2X) {
                        const int cq = args.Cout >> 2;
                        sub = col0 / cq;
                        ocol = col0 - sub * cq;
                    }
                    long long c_pix[4];
#pragma unroll
                    for (int it = 0; it < 4; ++it) {
                        if constexpr (MODE == EPI_SHUFFLE2X)
                            c_pix[it] = (static_cast<long long>(tc.img) * (2 * args.Ho) + (2 * c_h[it] + (sub >> 1))) *
                                            (2LL * args.Wo) +
                                        (2 * c_w[it] + (sub & 1));
                        else
                            c_pix[it] = (static_cast<long long>(tc.img) * args.Ho + c_h[it]) * args.Wo + c_w[it];
                    }
#pragma unroll
                    for (int p = 0; p < NPASS; ++p) {
                        const int pc0 = ocol + p * CPP;                             // first output column of the pass
                        const int valid = min(CPP, args.Cout - (col0 + p * CPP));   // valid columns (may be <= 0)
                        if (valid > 0) {
                            // ---- residual: coalesced global -> staging -> own row
                            if constexpr (RESID != 0) {
                                constexpr int per16 = 16 / RESZ;
                                const int e0 = piece * per16;
#pragma unroll
                                for (int it = 0; it < 4; ++it) {
                                    const int rr = it * 8 + (lane >> 2);
                                    uint8_t* sp = stage + rr * kStagePitch + piece * 16;
                                    *reinterpret_cast<uint4*>(sp) = rres[p][it];  // prefetched (zero when masked)
                                    if (c_ok[it] && e0 < valid && e0 + per16 > valid) {
                                        // ragged last columns: element-wise into the staging row
                                        const char* gp = reinterpret_cast<const char*>(args.resid) +
                                                         (c_pix[it] * args.ldr + pc0 + e0) * RESZ;
                                        copy_elems(sp, gp, valid - e0, RESZ);
                                    }
                                }
                                __syncwarp();
                                if constexpr (RESID == 2) {
                                    const float4* rp = reinterpret_cast<const float4*>(my_row);
#pragma unroll
                                    for (int j = 0; j < 4; ++j) {
                                        const float4 r = rp[j];
                                        f[p * 16 + 4 * j + 0] += r.x;
                                        f[p * 16 + 4 * j + 1] += r.y;
                                        f[p * 16 + 4 * j + 2] += r.z;
                                        f[p * 16 + 4 * j + 3] += r.w;
                                    }
                                } else {
                                    const uint4* rp = reinterpret_cast<const uint4*>(my_row);
#pragma unroll
                                    for (int j = 0; j < CPP / 8; ++j) {
                                        const uint4 r = rp[j];
                                        const int b = p * CPP + 8 * j;
                                        f[b + 0] += op_lo(r.x); f[b + 1] += op_hi(r.x);
                                        f[b + 2] += op_lo(r.y); f[b + 3] += op_hi(r.y);
                                        f[b + 4] += op_lo(r.z); f[b + 5] += op_hi(r.z);
                                        f[b + 6] += op_lo(r.w); f[b + 7] += op_hi(r.w);
                                    }
                                }
                                __syncwarp();
                            }
                            // ---- activation + pack into the staging row (own row only)
                            if (args.act == ACT_RELU) {
#pragma unroll
                                for (int j = 0; j < CPP; ++j) f[p * CPP + j] = fmaxf(f[p * CPP + j], 0.f);
                            } else if (args.act == ACT_GELU) {
#pragma unroll
                                for (int j = 0; j < CPP; j += 2) gelu_fast2(f[p * CPP + j], f[p * CPP + j + 1]);
                            } else if (args.act == ACT_SIGMOID) {
#pragma unroll
                                for (int j = 0; j < CPP; ++j)
                                    f[p * CPP + j] = __fdividef(1.f, 1.f + __expf(-f[p * CPP + j]));
                            } else if (args.act == ACT_SILU) {
#pragma unroll
                                for (int j = 0; j < CPP; ++j)
                                    f[p * CPP + j] = __fdividef(f[p * CPP + j], 1.f + __expf(-f[p * CPP + j]));
                            }
                            if constexpr (OUT_F32) {
                                float4* wp = reinterpret_cast<float4*>(my_row);
#pragma unroll
                                for (int j = 0; j < 4; ++j) {
                                    float4 o;
                                    o.x = f[p * 16 + 4 * j + 0];
                                    o.y = f[p * 16 + 4 * j + 1];
                                    o.z = f[p * 16 + 4 * j + 2];
                                    o.w = f[p * 16 + 4 * j + 3];
                                    wp[j] = o;
                                }
                            } else {
                                uint4* wp = reinterpret_cast<uint4*>(my_row);
#pragma unroll
                                for (int j = 0; j < CPP / 8; ++j) {
                                    const int b = p * CPP + 8 * j;
                                    uint4 o;
                                    o.x = pack_op(f[b + 0], f[b + 1]);
                                    o.y = pack_op(f[b + 2], f[b + 3]);
                                    o.z = pack_op(f[b + 4], f[b + 5]);
                                    o.w = pack_op(f[b + 6], f[b + 7]);
                                    wp[j] = o;
                                }
                            }
                            __syncwarp();
                            // ---- coalesced staging -> global
                            {
                                constexpr int per16 = 16 / OESZ;
                                constexpr int row_bytes = CPP * OESZ;
                                const int e0 = piece * per16;
                                if (piece * 16 < row_bytes && e0 < valid) {
#pragma unroll
                                    for (int it = 0; it < 4; ++it) {
                                        if (!c_ok[it]) continue;
                                        const int rr = it * 8 + (lane >> 2);
                                        const uint8_t* sp = stage + rr * kStagePitch + piece * 16;
                                        char* gp = reinterpret_cast<char*>(args.out) +
                                                   (c_pix[it] * args.ldc + pc0 + e0) * OESZ;
                                        if (e0 + per16 <= valid) {
                                            *reinterpret_cast<uint4*>(gp) = *reinterpret_cast<const uint4*>(sp);
                                        } else {
                                            copy_elems(gp, sp, valid - e0, OESZ);
                                        }
                                    }
                                }
                            }
                            __syncwarp();
                        }
                    }
                }
            }
            if constexpr (MODE == EPI_ROWMAX) {
                if (row_ok) {
                    const long long pixo = (static_cast<long long>(tc.img) * args.Ho + hh) * args.Wo + ww;
                    float4 o;
                    o.x = rm_m;
                    o.y = rm_s;
                    o.z = __int_as_float(rm_i);
                    o.w = 0.f;
                    reinterpret_cast<float4*>(args.out)[pixo * args.ldc + (tc.n0 / BLOCK_N) * 2 + wset] = o;
                }
            }
        }
        }  // legacy (DIRECT 0 / 1) epilogue
    }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, []() {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
        if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

int make_tmap_op_4d(CUtensorMap* m, const void* base, const uint64_t dims[4], const uint64_t strides_b[3],
                      const uint32_t box[4]) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) {
        set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
        return 1;
    }
    cuuint64_t gd[4] = {dims[0], dims[1], dims[2], dims[3]};
    cuuint64_t gs[3] = {strides_b[0], strides_b[1], strides_b[2]};
    cuuint32_t bx[4] = {box[0], box[1], box[2], box[3]};
    cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = fn(m, kOpFmt ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), gd, gs, bx, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d): dims=%llu,%llu,%llu,%llu strides=%llu,%llu,%llu box=%u,%u,%u,%u "
                  "base=%p",
                  (int)r, (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2],
                  (unsigned long long)dims[3], (unsigned long long)strides_b[0], (unsigned long long)strides_b[1],
                  (unsigned long long)strides_b[2], box[0], box[1], box[2], box[3], base);
        return 1;
    }
    return 0;
}

// Output / residual tensor [n_img][Ho][Wo][Cout] (row pitch ld elements) as a 4-D map whose box is one epilogue warp's
// pass: 128 bytes of columns x the warp's 16 tile rows (16 consecutive pixels of a row when the patch is at least 16
// wide, else 16 / BW full patch rows).
static int make_tmap_epi(CUtensorMap* m, const void* base, int f32, const GemmArgs& a, int Cout, long long ld, int swz,
                         int tile_cols = 0) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) {
        set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
        return 1;
    }
    const uint64_t es = f32 ? 4 : 2;
    const int bw = 1 << a.bw_log2;
    cuuint64_t gd[4] = {(cuuint64_t)Cout, (cuuint64_t)a.Wo, (cuuint64_t)a.Ho, (cuuint64_t)a.n_img};
    cuuint64_t gs[3] = {(cuuint64_t)ld * es, (cuuint64_t)ld * es * a.Wo, (cuuint64_t)ld * es * a.Wo * a.Ho};
    cuuint32_t bx[4] = {(cuuint32_t)(128 / es), (cuuint32_t)(bw < 16 ? bw : 16), (cuuint32_t)(bw < 16 ? 16 / bw : 1), 1};
    if (tile_cols > 0) {   // prefetch map: the whole BH x BW x BLOCK_N output tile
        bx[0] = (cuuint32_t)tile_cols;
        bx[1] = (cuuint32_t)bw;
        bx[2] = (cuuint32_t)(128 / bw);
        swz = 0;
    }
    // L2 promotion of the box fetches: 128 B by default; YTK_EPI_L2P=256 opts into 256 B
    static const bool l2_256 = getenv("YTK_EPI_L2P") != nullptr && getenv("YTK_EPI_L2P")[0] == '2';
    cuuint32_t est[4] = {1, 1, 1, 1};
    const CUtensorMapDataType dt = f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                       : (kOpFmt ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
    CUresult r = fn(m, dt, 4, const_cast<void*>(base), gd, gs, bx, est, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    swz ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                    l2_256 ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B : CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled (epilogue box) failed (%d): dims=%llu,%llu,%llu,%llu ld=%lld f32=%d base=%p",
                  (int)r, (unsigned long long)gd[0], (unsigned long long)gd[1], (unsigned long long)gd[2],
                  (unsigned long long)gd[3], ld, f32, base);
        return 1;
    }
    return 0;
}

// Epilogue path: YTK_EPI=staged keeps the per-thread global accesses everywhere (A/B aid); default = TMA where the
// plan allows it.  YTK_EPI_SWZ=0 builds unswizzled boxes (debugging aid: bank conflicts, same results).
static int epi_mode_env() {
    static int mode = -1;
    if (mode < 0) {
        const char* e = getenv("YTK_EPI");
        mode = (e && e[0] == 's') ? 0 : 2;
    }
    return mode;
}

static int pick_block_n(int Cout) {
    if (Cout <= 64) return 64;
    if (Cout <= 128) return 128;
    if (Cout % 256 == 0 || Cout > 512) return 256;
    if (Cout % 128 == 0) return 128;
    return 256;
}

// Choose the BH x BW patch (BH*BW = 128) that wastes the fewest pixels.
static int pick_bw_log2(int Ho, int Wo) {
    int best = 7;
    long long best_cost = -1;
    for (int l = 3; l <= 7; ++l) {
        int bw = 1 << l, bh = 128 >> l;
        long long cost = (long long)((Wo + bw - 1) / bw) * ((Ho + bh - 1) / bh);
        if (best_cost < 0 || cost < best_cost || (cost == best_cost && l > best)) {
            best_cost = cost;
            best = l;
        }
    }
    return best;
}

// Refuses an epilogue the kernel cannot store safely, before any CUDA call.  The staged epilogue moves 16-byte pieces
// (uint4 / float4) at base + (pixel * pitch + column) * element size and reads the bias as float4, so bases and pitches
// must keep those pieces 16-byte aligned; the TMA epilogue encodes a tensor of width Cout with row pitch ldc.
static int check_epilogue(int Cout, const Epilogue& e) {
    auto misaligned = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; };
    if (e.out == nullptr) {
        set_error("gemm plan: null output");
        return 1;
    }
    if (Cout < 1) {
        set_error("gemm plan: Cout=%d", Cout);
        return 1;
    }
    if (e.act < ACT_NONE || e.act > ACT_SILU) {
        set_error("gemm plan: act %d unknown (0..4)", e.act);
        return 1;
    }
    // the fused final conv stores float2 pairs: its probability map needs 8-byte alignment only
    if ((e.mode != EPI_CONVT_FINAL && misaligned(e.out)) || misaligned(e.resid) || misaligned(e.bias)) {
        set_error("gemm plan: output, residual and bias must be 16-byte aligned");
        return 1;
    }
    if (e.mode == EPI_ROWMAX) {
        if (e.resid != nullptr) {
            set_error("gemm plan: ROWMAX takes no residual");
            return 1;
        }
    } else if (e.mode == EPI_CONVT_FINAL) {
        if (Cout != 256 || e.fin_w == nullptr || !e.out_f32) {
            set_error("gemm plan: CONVT_FINAL needs Cout=256, fp32 output and the final conv weights");
            return 1;
        }
    } else {
        if ((e.out_f32 ? (e.ldc % 4) : (e.ldc % 8)) != 0) {
            set_error("gemm plan: ldc=%lld must keep rows 16-byte aligned", e.ldc);
            return 1;
        }
        // SHUFFLE2X: column block (i, j) of width Cout / 4 goes to its own output pixel
        const long long width = e.mode == EPI_SHUFFLE2X ? Cout / 4 : Cout;
        if (e.ldc < width) {
            set_error("gemm plan: ldc=%lld is less than the %lld columns of an output row", e.ldc, width);
            return 1;
        }
    }
    if (e.resid) {
        if ((e.resid_f32 ? (e.ldr % 4) : (e.ldr % 8)) != 0) {
            set_error("gemm plan: ldr=%lld must keep rows 16-byte aligned", e.ldr);
            return 1;
        }
        if (e.ldr < Cout) {
            set_error("gemm plan: ldr=%lld is less than Cout=%d", e.ldr, Cout);
            return 1;
        }
    }
    if (e.mode == EPI_SHUFFLE2X && ((Cout % 4) != 0 || ((Cout / 4) % 32) != 0)) {
        set_error("gemm plan: SHUFFLE2X needs Cout/4 to be a multiple of 32 (Cout=%d)", Cout);
        return 1;
    }
    return 0;
}

static int finish_plan(GemmPlan* plan, const void* w_packed, int Ktot, int Cout, const Epilogue& e) {
    GemmArgs& a = plan->args;
    plan->block_n = pick_block_n(Cout);
    static const bool no_shrink = getenv("YTK_NO_SHRINK") != nullptr;  // debugging aid
    // YTK_WAVE_MODEL=1: choose the N tile of few-wave problems by waves x relative tile time (experiment switch: the
    // relative tile times below are a model, not a measurement of this kernel).
    static const bool no_wave_model = getenv("YTK_WAVE_MODEL") == nullptr;
    if (e.mode != EPI_CONVT_FINAL && !no_shrink) {
        const int m_tiles = a.n_img * a.tiles_h * a.tiles_w;
        const int sms = num_sms();
        auto tiles_at = [&](int bn) { return (long long)m_tiles * ((Cout + bn - 1) / bn); };
        if (no_wave_model || (tiles_at(plan->block_n) + sms - 1) / sms > 6) {
            // small problems (decode steps, coarse feature maps): shrink the N tile until the persistent grid fills the SMs
            while (plan->block_n > 64 && tiles_at(plan->block_n) < sms) plan->block_n >>= 1;
        } else {
            // a handful of waves: the last, partly filled wave costs as much as a full one (3200 decode rows x 768
            // columns = 150 tiles of 128 columns on 132 SMs = two waves).  Pick the N tile with the smallest
            // waves x (relative time of one tile of that width); ties go to the wider tile.
            int best = plan->block_n;
            double best_cost = 1e30;
            for (int bn = plan->block_n; bn >= 64; bn >>= 1) {
                const double w = bn == 256 ? 1.9 : bn == 128 ? 1.0 : 0.56;
                const double cost = (double)((tiles_at(bn) + sms - 1) / sms) * w;
                if (cost < best_cost - 1e-9) {
                    best_cost = cost;
                    best = bn;
                }
            }
            plan->block_n = best;
        }
    }
    a.tiles_n = (Cout + plan->block_n - 1) / plan->block_n;
    a.Cout = Cout;
    a.bias = e.bias;
    a.resid = e.resid;
    a.resid_f32 = e.resid_f32;
    a.ldr = e.ldr;
    a.out = e.out;
    a.out_f32 = e.out_f32;
    a.ldc = e.ldc;
    a.act = e.act;
    a.mode = e.mode;
    a.fin_w = e.fin_w;
    a.fin_b = e.fin_b;
    if (e.mode == EPI_ROWMAX) {
        a.out_f32 = 1;
        a.ldc = 2LL * a.tiles_n;   // float4 partials per row
    }
    const int tiles = a.n_img * a.tiles_h * a.tiles_w * a.tiles_n;
    // TMA epilogue: plain stores whose residual (if any) has the output's element size and rows whose extent is a
    // multiple of 16 bytes: a TMA store clips the box at the tensor's inner extent in 16-byte units (Cout = 7119 fp32
    // columns: column 7119 of a 7120-wide buffer was written).  Bases and pitches are 16-byte aligned (check_epilogue).
    a.epi_tma = 0;
    a.epi_swz = 0;
    a.epi_pf = 0;
    if (epi_mode_env() == 2 && e.mode == EPI_NORMAL && (e.resid == nullptr || (e.resid_f32 != 0) == (e.out_f32 != 0)) &&
        ((long long)Cout * (e.out_f32 ? 4 : 2)) % 16 == 0) {
        static const bool no_swz = getenv("YTK_EPI_SWZ") != nullptr && getenv("YTK_EPI_SWZ")[0] == '0';
        // whole-tile L2 prefetch of the residual one tile ahead: opt-in (YTK_EPI_PF=1).
        static const bool no_pf = !(getenv("YTK_EPI_PF") != nullptr && getenv("YTK_EPI_PF")[0] == '1');
        a.epi_tma = 1;
        a.epi_swz = no_swz ? 0 : 1;
        if (make_tmap_epi(&plan->maps.out, e.out, e.out_f32, a, Cout, e.ldc, a.epi_swz)) return 1;
        if (e.resid != nullptr) {
            if (make_tmap_epi(&plan->maps.resid, e.resid, e.resid_f32, a, Cout, e.ldr, a.epi_swz)) return 1;
            if (make_tmap_epi(&plan->maps.resid_pf, e.resid, e.resid_f32, a, Cout, e.ldr, 0, plan->block_n)) return 1;
            a.epi_pf = no_pf ? 0 : 1;
        } else {
            plan->maps.resid = plan->maps.out;
            plan->maps.resid_pf = plan->maps.out;
        }
    }
    // weights: [Cout][Ktot] 16-bit, K-major
    uint64_t dims[4] = {(uint64_t)Ktot, (uint64_t)Cout, 1, 1};
    uint64_t strides[3] = {(uint64_t)Ktot * 2, (uint64_t)Ktot * 2 * Cout, (uint64_t)Ktot * 2 * Cout};
    uint32_t box[4] = {(uint32_t)kBlockK, (uint32_t)plan->block_n, 1, 1};
    if (make_tmap_op_4d(&plan->maps.b, w_packed, dims, strides, box)) return 1;
    plan->grid = tiles < num_sms() ? tiles : num_sms();
    if (plan->grid < 1) plan->grid = 1;
    return 0;
}

int conv_plan_create(GemmPlan* plan, const void* in, const ConvGeom& g, const void* w_packed, const Epilogue& e) {
    memset(plan, 0, sizeof(*plan));
    GemmArgs& a = plan->args;
    if (g.Cin % kBlockK != 0) {
        set_error("conv plan: Cin=%d must be a multiple of %d", g.Cin, kBlockK);
        return 1;
    }
    if (g.stride != 1 && g.stride != 2) {
        set_error("conv plan: stride %d unsupported", g.stride);
        return 1;
    }
    if (g.kh * g.kw > kMaxTaps) {
        set_error("conv plan: %dx%d filter exceeds %d taps", g.kh, g.kw, kMaxTaps);
        return 1;
    }
    if (check_epilogue(g.Cout, e)) return 1;
    const int Ho = (g.H + 2 * g.pad - g.dil * (g.kh - 1) - 1) / g.stride + 1;
    const int Wo = (g.W + 2 * g.pad - g.dil * (g.kw - 1) - 1) / g.stride + 1;
    a.Ho = Ho;
    a.Wo = Wo;
    a.n_img = g.N;
    a.bw_log2 = pick_bw_log2(Ho, Wo);
    const int bw = 1 << a.bw_log2, bh = 128 >> a.bw_log2;
    a.tiles_w = (Wo + bw - 1) / bw;
    a.tiles_h = (Ho + bh - 1) / bh;
    a.kpt = g.Cin / kBlockK;
    a.ntaps = g.kh * g.kw;
    const uint64_t es = 2;
    const uint32_t box[4] = {(uint32_t)kBlockK, (uint32_t)bw, (uint32_t)bh, 1};
    const char* base = reinterpret_cast<const char*>(in);
    if (g.stride == 1) {
        uint64_t dims[4] = {(uint64_t)g.Cin, (uint64_t)g.W, (uint64_t)g.H, (uint64_t)g.N};
        uint64_t strides[3] = {(uint64_t)g.in_ld * es, (uint64_t)g.in_ld * es * g.W, (uint64_t)g.in_ld * es * g.W * g.H};
        if (make_tmap_op_4d(&plan->maps.a[0], base, dims, strides, box)) return 1;
        for (int i = 1; i < 4; ++i) plan->maps.a[i] = plan->maps.a[0];
        int t = 0;
        for (int r = 0; r < g.kh; ++r)
            for (int s = 0; s < g.kw; ++s, ++t) {
                a.taps[t].map = 0;
                a.taps[t].dh = r * g.dil - g.pad;
                a.taps[t].dw = s * g.dil - g.pad;
            }
    } else {
        // stride 2: input row 2*ho + (r*dil - pad) = 2*(ho + floor(o/2)) + (o mod 2): phase map (o mod 2), shift floor(o/2)
        bool used[4] = {false, false, false, false};
        int t = 0;
        for (int r = 0; r < g.kh; ++r)
            for (int s = 0; s < g.kw; ++s, ++t) {
                const int oh = r * g.dil - g.pad, ow = s * g.dil - g.pad;
                const int ph = ((oh % 2) + 2) % 2, pw = ((ow % 2) + 2) % 2;
                a.taps[t].map = ph * 2 + pw;
                a.taps[t].dh = (oh - ph) / 2;
                a.taps[t].dw = (ow - pw) / 2;
                used[ph * 2 + pw] = true;
            }
        int first = -1;
        for (int p = 0; p < 4; ++p) {
            if (!used[p]) continue;
            const int ph = p >> 1, pw = p & 1;
            const int hp = (g.H - ph + 1) / 2, wp = (g.W - pw + 1) / 2;
            if (hp <= 0 || wp <= 0) {
                set_error("conv plan: degenerate stride-2 phase");
                return 1;
            }
            uint64_t dims[4] = {(uint64_t)g.Cin, (uint64_t)wp, (uint64_t)hp, (uint64_t)g.N};
            uint64_t strides[3] = {(uint64_t)g.in_ld * es * 2, (uint64_t)g.in_ld * es * g.W * 2,
                                   (uint64_t)g.in_ld * es * g.W * g.H};
            const char* pbase = base + ((size_t)ph * g.W + pw) * g.in_ld * es;
            if (make_tmap_op_4d(&plan->maps.a[p], pbase, dims, strides, box)) return 1;
            if (first < 0) first = p;
        }
        for (int p = 0; p < 4; ++p)
            if (!used[p]) plan->maps.a[p] = plan->maps.a[first];
    }
    plan->flops = 2.0 * g.N * Ho * Wo * (double)g.Cout * g.Cin * g.kh * g.kw;
    return finish_plan(plan, w_packed, g.kh * g.kw * g.Cin, g.Cout, e);
}

int gemm_plan_create(GemmPlan* plan, const void* A, long long lda, int M, int K, const void* Wt, int N,
                     const Epilogue& e) {
    memset(plan, 0, sizeof(*plan));
    GemmArgs& a = plan->args;
    if (K % kBlockK != 0) {
        set_error("gemm plan: K=%d must be a multiple of %d", K, kBlockK);
        return 1;
    }
    if (M < 1) {
        set_error("gemm plan: M=%d", M);
        return 1;
    }
    if (lda < K || lda % 8 != 0) {
        set_error("gemm plan: lda=%lld must be >= K=%d and a multiple of 8", lda, K);
        return 1;
    }
    if (check_epilogue(N, e)) return 1;
    a.Ho = 1;
    a.Wo = M;
    a.n_img = 1;
    a.bw_log2 = 7;
    a.tiles_w = (M + 127) / 128;
    a.tiles_h = 1;
    a.kpt = K / kBlockK;
    a.ntaps = 1;
    a.taps[0].map = 0;
    a.taps[0].dh = 0;
    a.taps[0].dw = 0;
    uint64_t dims[4] = {(uint64_t)K, (uint64_t)M, 1, 1};
    uint64_t strides[3] = {(uint64_t)lda * 2, (uint64_t)lda * 2 * M, (uint64_t)lda * 2 * M};
    uint32_t box[4] = {(uint32_t)kBlockK, 128, 1, 1};
    if (make_tmap_op_4d(&plan->maps.a[0], A, dims, strides, box)) return 1;
    for (int i = 1; i < 4; ++i) plan->maps.a[i] = plan->maps.a[0];
    plan->flops = 2.0 * M * (double)N * K;
    return finish_plan(plan, Wt, K, N, e);
}

int stem_plan_create(GemmPlan* plan, const void* in_padded, int N, int Hn, int Wn, const void* w_packed,
                     const Epilogue& e) {
    memset(plan, 0, sizeof(*plan));
    if (check_epilogue(64, e)) return 1;
    GemmArgs& a = plan->args;
    const int Ho = Hn / 2, Wo = Wn / 2, Hp = Hn + 6, Wp = Wn + 8;
    a.Ho = Ho;
    a.Wo = Wo;
    a.n_img = N;
    a.bw_log2 = pick_bw_log2(Ho, Wo);
    const int bw = 1 << a.bw_log2, bh = 128 >> a.bw_log2;
    a.tiles_w = (Wo + bw - 1) / bw;
    a.tiles_h = (Ho + bh - 1) / bh;
    a.kpt = 1;
    a.ntaps = 7;
    const uint32_t box[4] = {(uint32_t)kBlockK, (uint32_t)bw, (uint32_t)bh, 1};
    const char* base = reinterpret_cast<const char*>(in_padded);
    const uint64_t row_b = (uint64_t)Wp * 8 * 2;
    for (int p = 0; p < 2; ++p) {
        // input row 2*ho + r = 2*(ho + r/2) + (r & 1): phase p = r & 1 starts at padded row p, steps 2 rows
        uint64_t dims[4] = {64, (uint64_t)Wo, (uint64_t)((Hp - p + 1) / 2), (uint64_t)N};
        uint64_t strides[3] = {32, 2 * row_b, (uint64_t)Hp * row_b};
        if (make_tmap_op_4d(&plan->maps.a[p], base + p * row_b, dims, strides, box)) return 1;
    }
    plan->maps.a[2] = plan->maps.a[0];
    plan->maps.a[3] = plan->maps.a[1];
    for (int r = 0; r < 7; ++r) {
        a.taps[r].map = r & 1;
        a.taps[r].dh = r >> 1;
        a.taps[r].dw = 0;
    }
    plan->flops = 2.0 * N * Ho * Wo * 64.0 * 448.0;
    return finish_plan(plan, w_packed, 7 * 64, 64, e);
}

int gemm_plan_set_out(GemmPlan* plan, void* out) {
    GemmArgs& a = plan->args;
    if ((reinterpret_cast<uintptr_t>(out) & 15) != 0) {
        set_error("gemm_plan_set_out: output must be 16-byte aligned");
        return 1;
    }
    a.out = out;
    if (!a.epi_tma) return 0;
    return make_tmap_epi(&plan->maps.out, out, a.out_f32, a, a.Cout, a.ldc, a.epi_swz);
}

template <int BLOCK_N, int OUT_F32, int RESID, int MODE, int DIRECT>
static int launch_variant2(const GemmPlan* plan, cudaStream_t stream) {
    using Cfg = KernelCfg<BLOCK_N, RESID, DIRECT>;
    static unsigned long long attr_done = 0;   // per device (a process may hold handles on several GPUs)
    auto kern = gemm_tc_kernel<BLOCK_N, OUT_F32, RESID, MODE, DIRECT>;
    if (first_launch_on_device(&attr_done)) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
        if (e != cudaSuccess) {
            set_error("cudaFuncSetAttribute(smem=%d): %s", Cfg::kSmemBytes, cudaGetErrorString(e));
            return 1;
        }
    }
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    cfg.gridDim = dim3(plan->grid);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = Cfg::kSmemBytes;
    cfg.stream = stream;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_launch_attr(attr);
    cudaError_t e = cudaLaunchKernelEx(&cfg, kern, plan->maps, plan->args);
    count_launch();
    if (e != cudaSuccess) {
        set_error("gemm_tc_kernel<%d,%d,%d,%d,%d> launch: %s", BLOCK_N, OUT_F32, RESID, MODE, DIRECT,
                  cudaGetErrorString(e));
        return 1;
    }
    return 0;
}

// Epilogue path per plan: the TMA epilogue (args.epi_tma, set by finish_plan) or the staged one.
template <int BLOCK_N, int OUT_F32, int RESID, int MODE>
static int launch_variant(const GemmPlan* plan, cudaStream_t stream) {
    if constexpr (MODE == EPI_NORMAL && (RESID == 0 || (RESID == 2) == (OUT_F32 != 0))) {
        if (plan->args.epi_tma) return launch_variant2<BLOCK_N, OUT_F32, RESID, MODE, 2>(plan, stream);
    }
    return launch_variant2<BLOCK_N, OUT_F32, RESID, MODE, 0>(plan, stream);
}

template <int BLOCK_N>
static int launch_bn(const GemmPlan* plan, cudaStream_t stream) {
    const GemmArgs& a = plan->args;
    const int resid = a.resid == nullptr ? 0 : (a.resid_f32 ? 2 : 1);
    if (a.mode == EPI_CONVT_FINAL) {
        if constexpr (BLOCK_N == 256) return launch_variant<256, 1, 0, EPI_CONVT_FINAL>(plan, stream);
        set_error("CONVT_FINAL needs BLOCK_N = 256");
        return 1;
    }
    if (a.mode == EPI_ROWMAX) return launch_variant2<BLOCK_N, 1, 0, EPI_ROWMAX, 0>(plan, stream);
    if (a.mode == EPI_SHUFFLE2X) {
        if (resid == 0 && !a.out_f32) return launch_variant<BLOCK_N, 0, 0, EPI_SHUFFLE2X>(plan, stream);
        if (resid == 0 && a.out_f32) return launch_variant<BLOCK_N, 1, 0, EPI_SHUFFLE2X>(plan, stream);
        set_error("SHUFFLE2X epilogue does not take a residual");
        return 1;
    }
    if (!a.out_f32) {
        if (resid == 0) return launch_variant<BLOCK_N, 0, 0, EPI_NORMAL>(plan, stream);
        if (resid == 1) return launch_variant<BLOCK_N, 0, 1, EPI_NORMAL>(plan, stream);
        return launch_variant<BLOCK_N, 0, 2, EPI_NORMAL>(plan, stream);
    }
    if (resid == 0) return launch_variant<BLOCK_N, 1, 0, EPI_NORMAL>(plan, stream);
    if (resid == 1) return launch_variant<BLOCK_N, 1, 1, EPI_NORMAL>(plan, stream);
    return launch_variant<BLOCK_N, 1, 2, EPI_NORMAL>(plan, stream);
}

// ---- per-launch timing of gemm_tc_kernel (bench.py roofline): CUDA events on the launching stream around every launch
namespace {
struct ProfRec {
    cudaEvent_t a, b;
    double flops;
    int pixels, cout, k, block_n, mode, act, resid, out_f32, ntaps;   // shape of the launch (YTK_GEMM_DUMP)
    int epi, bw_log2;   // epilogue path (1 = TMA, 0 = staged) and tile patch (BW = 1 << bw_log2)
};
std::mutex g_prof_mu;
bool g_prof_on = false;
std::vector<ProfRec> g_prof;        // records of the current window
std::vector<cudaEvent_t> g_prof_pool;  // recycled events
cudaEvent_t prof_event() {
    if (!g_prof_pool.empty()) {
        cudaEvent_t e = g_prof_pool.back();
        g_prof_pool.pop_back();
        return e;
    }
    cudaEvent_t e = nullptr;
    cudaEventCreate(&e);
    return e;
}
}  // namespace

void gemm_profile_begin() {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    for (ProfRec& r : g_prof) {
        g_prof_pool.push_back(r.a);
        g_prof_pool.push_back(r.b);
    }
    g_prof.clear();
    g_prof_on = true;
}

int gemm_profile_end(double* flops, double* ms, long long* launches) {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    g_prof_on = false;
    double f = 0, t = 0;
    for (ProfRec& r : g_prof) {
        if (cudaEventSynchronize(r.b) != cudaSuccess) {
            set_error("gemm_profile_end: event synchronize failed");
            return 1;
        }
        float e = 0.f;
        cudaEventElapsedTime(&e, r.a, r.b);
        t += e;
        f += r.flops;
    }
    if (flops) *flops = f;
    if (ms) *ms = t;
    if (launches) *launches = (long long)g_prof.size();
    if (const char* path = getenv("YTK_GEMM_DUMP")) {      // per-launch table of the window for shape-level analysis
        if (FILE* fp = fopen(path, "a")) {
            fprintf(fp, "pixels,cout,k,ntaps,block_n,mode,act,resid,out_f32,flops,ms,epi,bw_log2\n");
            for (ProfRec& r : g_prof) {
                float e = 0.f;
                cudaEventElapsedTime(&e, r.a, r.b);
                fprintf(fp, "%d,%d,%d,%d,%d,%d,%d,%d,%d,%.0f,%.6f,%d,%d\n", r.pixels, r.cout, r.k, r.ntaps, r.block_n,
                        r.mode, r.act, r.resid, r.out_f32, r.flops, e, r.epi, r.bw_log2);
            }
            fclose(fp);
        }
    }
    return 0;
}

int gemm_plan_launch(const GemmPlan* plan, cudaStream_t stream) {
    ProfRec rec{};
    bool prof = false;
    if (g_prof_on) {
        std::lock_guard<std::mutex> lk(g_prof_mu);
        if (g_prof_on) {
            rec.a = prof_event();
            rec.b = prof_event();
            rec.flops = plan->flops;
            const GemmArgs& g = plan->args;
            rec.pixels = g.Ho * g.Wo * g.n_img;
            rec.cout = g.Cout;
            rec.k = g.kpt * 64;
            rec.ntaps = g.ntaps;
            rec.block_n = plan->block_n;
            rec.mode = g.mode;
            rec.act = g.act;
            rec.resid = g.resid ? (g.resid_f32 ? 2 : 1) : 0;
            rec.out_f32 = g.out_f32;
            rec.epi = g.epi_tma;
            rec.bw_log2 = g.bw_log2;
            prof = true;
        }
    }
    if (prof) cudaEventRecord(rec.a, stream);
    int rc;
    switch (plan->block_n) {
        case 64: rc = launch_bn<64>(plan, stream); break;
        case 128: rc = launch_bn<128>(plan, stream); break;
        case 256: rc = launch_bn<256>(plan, stream); break;
        default: set_error("bad block_n %d", plan->block_n); rc = 1;
    }
    if (prof) {
        cudaEventRecord(rec.b, stream);
        std::lock_guard<std::mutex> lk(g_prof_mu);
        g_prof.push_back(rec);
    }
    return rc;
}

}  // namespace ytk
