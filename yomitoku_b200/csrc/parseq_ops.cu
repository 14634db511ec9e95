// Non-GEMM kernels of the PARSeq recognizer (sm_90a): patchify, LayerNorm, flash attention over packed ragged
// sequences, the decoder's small attention kernels and the device-side greedy / EOS / repetition control logic that
// removes every host sync from the AR loop.  Reference: models/parseq.py:133-311, models/layers/parseq_transformer.py.
#include "parseq_ops.h"

#include <cfloat>
#include <cstdlib>

#include "gemm_tc.h"
#include "ptx.cuh"

namespace ytk {

// Launch with programmatic stream serialization (kernels below that start with pdl_wait(): the chain of an AR step).
template <typename... KArgs, typename... Args>
static cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_launch_attr(attr);
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// =================================================================================================== patchify
// Replaces timm PatchEmbed.proj's im2col (reference parseq_transformer.py:220-227): the conv itself is a wgmma GEMM;
// this kernel writes its A operand and seeds the fp32 residual stream with the cropped positional embedding.
// Normalisation = ToTensor + Normalize(0.5, 0.5) (data/dataset.py:57-62); pixels right of the stored canvas are the
// collate padding value -1.0 (text_recognizer.py:146-156).
__global__ void patchify_u8_kernel(const uint8_t* __restrict__ crops, const CropDesc* __restrict__ descs, int ph,
                                   int pw, int Kpad, const float* __restrict__ pos_embed, int full_gw, int D,
                                   op_t* __restrict__ A, float* __restrict__ x) {
    const CropDesc d = descs[blockIdx.y];
    const int gw = d.wp / pw;
    const int K = 3 * ph * pw;
    for (int t = blockIdx.x; t < d.ntok; t += gridDim.x) {
        const int gy = t / gw, gx = t - gy * gw;
        const long long row = (long long)d.tok_off + t;
        for (int k = threadIdx.x; k < Kpad; k += blockDim.x) {
            float v = 0.f;
            if (k < K) {
                const int c = k / (ph * pw);
                const int r = k - c * ph * pw;
                const int py = r / pw, px = r - py * pw;
                const int yy = gy * ph + py, xx = gx * pw + px;
                v = -1.f;
                if (xx < d.w) {
                    const float u = (float)crops[d.pix_off + ((long long)yy * d.w + xx) * 3 + c];
                    v = (u / 255.f - 0.5f) / 0.5f;
                }
            }
            A[row * Kpad + k] = f2op(v);
        }
        const float* pe = pos_embed + ((long long)gy * full_gw + gx) * D;
        for (int j = threadIdx.x; j < D; j += blockDim.x) x[row * D + j] = pe[j];
    }
}

int launch_patchify_u8(const uint8_t* crops, const CropDesc* descs, int ncrops, int ph, int pw, int Kpad,
                       const float* pos_embed, int full_gw, int D, void* A, float* x, int T, cudaStream_t st) {
    (void)T;
    dim3 grid(64, ncrops);
    patchify_u8_kernel<<<grid, 128, 0, st>>>(crops, descs, ph, pw, Kpad, pos_embed, full_gw, D,
                                             reinterpret_cast<op_t*>(A), x);
    count_launch();
    return cudaGetLastError() != cudaSuccess;
}

__global__ void patchify_f32_kernel(const float* __restrict__ img, int W, int ph, int pw, int Kpad,
                                    const float* __restrict__ pos_embed, int full_gw, int D,
                                    op_t* __restrict__ A, float* __restrict__ x) {
    const int b = blockIdx.y;
    const int gw = W / pw, gh = 32 / ph;
    const int ntok = gh * gw;
    const int K = 3 * ph * pw;
    for (int t = blockIdx.x; t < ntok; t += gridDim.x) {
        const int gy = t / gw, gx = t - gy * gw;
        const long long row = (long long)b * ntok + t;
        for (int k = threadIdx.x; k < Kpad; k += blockDim.x) {
            float v = 0.f;
            if (k < K) {
                const int c = k / (ph * pw);
                const int r = k - c * ph * pw;
                const int py = r / pw, px = r - py * pw;
                v = img[(((long long)b * 3 + c) * 32 + gy * ph + py) * W + gx * pw + px];
            }
            A[row * Kpad + k] = f2op(v);
        }
        const float* pe = pos_embed + ((long long)gy * full_gw + gx) * D;
        for (int j = threadIdx.x; j < D; j += blockDim.x) x[row * D + j] = pe[j];
    }
}

int launch_patchify_f32(const float* images, int B, int W, int ph, int pw, int Kpad, const float* pos_embed,
                        int full_gw, int D, void* A, float* x, cudaStream_t st) {
    dim3 grid(64, B);
    patchify_f32_kernel<<<grid, 128, 0, st>>>(images, W, ph, pw, Kpad, pos_embed, full_gw, D,
                                              reinterpret_cast<op_t*>(A), x);
    count_launch();
    return cudaGetLastError() != cudaSuccess;
}

// =================================================================================================== LayerNorm
// One warp per row, fp32 statistics (two-pass over registers), bf16 (and optional fp32) output.
constexpr int kLnVec = 8;  // float4 per lane: D <= 1024, D % 4 == 0

__global__ void __launch_bounds__(256) layernorm_kernel(float* __restrict__ x, int M, int D, int d_real,
                                                        const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, float eps,
                                                        op_t* __restrict__ out_bf16,
                                                        float* __restrict__ out_f32, const float* __restrict__ addvec,
                                                        int period, const int* __restrict__ add_row0_dev,
                                                        int add_row0, int writeback) {
    pdl_wait();   // (no early launch_dependents: this grid runs in many waves and a dependent persistent GEMM CTA that
                  // becomes resident early takes its SM away from the remaining waves)
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= M) return;
    const int nvec = D >> 2;
    float4* xr = reinterpret_cast<float4*>(x + (long long)warp * D);
    float4 v[kLnVec];
    // phase 1: all loads in flight at once (16 B per lane, 512 B contiguous per warp instruction)
#pragma unroll
    for (int i = 0; i < kLnVec; ++i) {
        const int j = lane + 32 * i;
        v[i] = (j < nvec) ? xr[j] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (addvec != nullptr) {
        const int r0 = add_row0_dev ? *add_row0_dev : add_row0;
        const float4* av = reinterpret_cast<const float4*>(addvec + (long long)((warp % period) + r0) * D);
#pragma unroll
        for (int i = 0; i < kLnVec; ++i) {
            const int j = lane + 32 * i;
            if (j < nvec) {
                const float4 a = __ldg(av + j);
                v[i].x += a.x; v[i].y += a.y; v[i].z += a.z; v[i].w += a.w;
                if (writeback) xr[j] = v[i];
            }
        }
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < kLnVec; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    // statistics over the d_real leading features; columns d_real..D are zero padding (zero in, zero gamma/beta)
    const float mean = s / (float)d_real;
    const int nvec_real = d_real >> 2;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < kLnVec; ++i) {
        const int j = lane + 32 * i;
        if (j < nvec_real) {
            const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
            q += (a * a + b * b) + (c * c + d * d);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = rsqrtf(q / (float)d_real + eps);
    const float4* g4 = reinterpret_cast<const float4*>(gamma);
    const float4* b4 = reinterpret_cast<const float4*>(beta);
#pragma unroll
    for (int i = 0; i < kLnVec; ++i) {
        const int j = lane + 32 * i;
        if (j < nvec) {
            const float4 g = __ldg(g4 + j), b = __ldg(b4 + j);
            float4 y;
            y.x = (v[i].x - mean) * rstd * g.x + b.x;
            y.y = (v[i].y - mean) * rstd * g.y + b.y;
            y.z = (v[i].z - mean) * rstd * g.z + b.z;
            y.w = (v[i].w - mean) * rstd * g.w + b.w;
            if (out_bf16) {
                uint2 o;
                o.x = pack_op(y.x, y.y);
                o.y = pack_op(y.z, y.w);
                reinterpret_cast<uint2*>(out_bf16 + (long long)warp * D)[j] = o;
            }
            if (out_f32) reinterpret_cast<float4*>(out_f32 + (long long)warp * D)[j] = y;
        }
    }
}

int launch_layernorm(float* x, int M, int D, int d_real, const float* gamma, const float* beta, float eps,
                     void* out_bf16, float* out_f32, const float* addvec, int period, const int* add_row0_dev,
                     int add_row0, int writeback, cudaStream_t st) {
    if (D > 128 * kLnVec || (D & 3) != 0 || (d_real & 3) != 0 || d_real > D || d_real <= 0) {
        set_error("layernorm: D=%d / d_real=%d unsupported (multiples of 4, 0 < d_real <= D <= %d)", D, d_real,
                  128 * kLnVec);
        return 1;
    }
    if (M <= 0) return 0;
    const int warps_per_block = 8;
    const cudaError_t e = launch_pdl(layernorm_kernel, dim3((M + warps_per_block - 1) / warps_per_block),
                                     dim3(warps_per_block * 32), 0, st, x, M, D, d_real, gamma, beta, eps,
                                     reinterpret_cast<op_t*>(out_bf16), out_f32, addvec, period > 0 ? period : 1,
                                     add_row0_dev, add_row0, writeback);
    count_launch();
    return e != cudaSuccess;
}

// =================================================================================================== flash attention
// softmax(Q K^T / sqrt(hd)) V over packed ragged sequences (encoder self-attention: timm Attention /
// F.scaled_dot_product_attention without mask, and the refinement cross-attention).  Tensor-core path: mma.sync
// m16n8k16 bf16 with fp32 accumulation; 64 queries per CTA (4 warps x 16), 64-key tiles staged with cp.async.
// HD = head dim (multiple of 16, <= 96).
__device__ __forceinline__ void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
                 : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3,
                                                  uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
                 : "r"(addr));
}
__device__ __forceinline__ void mma_bf16_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                               uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32." YTK_OPERAND_NAME "." YTK_OPERAND_NAME ".f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
    const int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait_group() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

template <int HD, int MASKED, int QT>
__global__ void __launch_bounds__(QT * 2, QT == 128 ? 2 : 3) flash_attn_kernel(const op_t* __restrict__ Q, long long ldq,
                                                            const op_t* __restrict__ K,
                                                            const op_t* __restrict__ V, long long ldkv,
                                                            op_t* __restrict__ O, long long ldo,
                                                            const SeqDesc* __restrict__ seqs, float scale_log2) {
    // QT queries per CTA (one warp per 16), 64-key tiles double-buffered with cp.async.  Warps whose 16 queries lie
    // beyond q_len only help loading; the MMA loops stop at the last 16-key group that holds a valid key.
    constexpr int LDS = HD + 8;  // padded row (bf16 elements): 16 B aligned rows, conflict-free ldmatrix
    constexpr int NT = QT * 2;   // threads
    extern __shared__ __align__(16) unsigned char fa_smem[];
    op_t* sQ = reinterpret_cast<op_t*>(fa_smem);  // [QT][LDS]
    op_t* sK = sQ + QT * LDS;                               // [2][64][LDS]
    op_t* sV = sK + 2 * 64 * LDS;                           // [2][64][LDS]
    const SeqDesc sd = seqs[blockIdx.z];
    const int q0 = blockIdx.x * QT;
    if (q0 >= sd.q_len) return;
    const int head = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool active = q0 + warp * 16 < sd.q_len;
    constexpr int CH = HD / 8;  // 16-byte chunks per row
    // keys this CTA can ever see (causal rows stop at their own index, rows 0/1 and the unmasked kernel see them all)
    int k_end = sd.k_len;
    if (MASKED) k_end = min(k_end, sd.kpad);
    if (MASKED && q0 >= 2) k_end = min(k_end, q0 + QT);
    const int ntiles = (k_end + 63) / 64;
    auto load_kv = [&](int t, int buf) {
        const int k0 = t * 64;
        op_t* dK = sK + buf * 64 * LDS;
        op_t* dV = sV + buf * 64 * LDS;
        const int rows = min(64, ((k_end - k0 + 15) >> 4) << 4);  // only 16-key groups that are used
        for (int i = threadIdx.x; i < rows * CH; i += NT) {
            const int r = i / CH, c = i - r * CH;
            const bool ok = (k0 + r) < sd.k_len;
            const long long rowi = sd.k_base + (long long)(ok ? k0 + r : 0) * ldkv + head * HD + c * 8;
            cp_async16(smem_u32(&dK[r * LDS + c * 8]), K + rowi, ok);
            cp_async16(smem_u32(&dV[r * LDS + c * 8]), V + rowi, ok);
        }
    };
    // ---- Q tile + first K/V tile
    {
        const int qrows = min(QT, ((sd.q_len - q0 + 15) >> 4) << 4);
        for (int i = threadIdx.x; i < qrows * CH; i += NT) {
            const int r = i / CH, c = i - r * CH;
            const bool ok = (q0 + r) < sd.q_len;
            const op_t* src = Q + (long long)(sd.q_off + (ok ? q0 + r : 0)) * ldq + head * HD + c * 8;
            cp_async16(smem_u32(&sQ[r * LDS + c * 8]), src, ok);
        }
    }
    if (ntiles > 0) load_kv(0, 0);
    cp_async_commit();
    float o[HD / 8][4];
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    uint32_t qf[HD / 16][4];
    for (int t = 0; t < ntiles; ++t) {
        const int k0 = t * 64, buf = t & 1;
        if (t + 1 < ntiles) load_kv(t + 1, buf ^ 1);  // buffer buf^1 was released by the barrier ending tile t-1
        cp_async_commit();
        cp_async_wait_group<1>();  // tile t (and Q) landed; tile t+1 may still be in flight
        __syncthreads();
        if (active) {
            const op_t* tK = sK + buf * 64 * LDS;
            const op_t* tV = sV + buf * 64 * LDS;
            if (t == 0) {
#pragma unroll
                for (int kk = 0; kk < HD / 16; ++kk) {
                    const int r = warp * 16 + (lane & 15);
                    const int c = kk * 16 + (lane >> 4) * 8;
                    ldmatrix_x4(qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3], smem_u32(&sQ[r * LDS + c]));
                }
            }
            // 16-key groups of this tile this warp needs
            int kmax = k_end;
            if (MASKED && q0 + warp * 16 >= 2) kmax = min(kmax, q0 + warp * 16 + 16);
            const int ng = min(4, (kmax - k0 + 15) >> 4);
            if (ng > 0) {
                // ---- S = Q K^T for 16 queries x 64 keys
                float s[8][4];
#pragma unroll
                for (int n = 0; n < 8; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
#pragma unroll
                for (int kk = 0; kk < HD / 16; ++kk) {
#pragma unroll
                    for (int np = 0; np < 4; ++np) {  // pairs of 8-key groups
                        if (np < ng) {
                            uint32_t b0, b1, b2, b3;
                            const int r = np * 16 + (lane & 7) + ((lane >> 4) << 3);
                            const int c = kk * 16 + ((lane >> 3) & 1) * 8;
                            ldmatrix_x4(b0, b1, b2, b3, smem_u32(&tK[r * LDS + c]));
                            mma_bf16_16816(s[2 * np], qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3], b0, b1);
                            mma_bf16_16816(s[2 * np + 1], qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3], b2, b3);
                        }
                    }
                }
                // ---- online softmax (rows lane/4 and lane/4 + 8 of this warp's 16 queries)
                float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
                for (int n = 0; n < 8; ++n) {
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int key = k0 + n * 8 + (lane & 3) * 2 + (e & 1);
                        bool vis = key < sd.k_len;
                        if (MASKED) {
                            const int qi = q0 + warp * 16 + (lane >> 2) + (e >> 1) * 8;
                            vis = vis && ((qi < 2) || (key <= qi)) && (key < sd.kpad);
                        }
                        const float val = vis ? s[n][e] * scale_log2 : -INFINITY;
                        s[n][e] = val;
                        mx[e >> 1] = fmaxf(mx[e >> 1], val);
                    }
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
                    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
                }
                float corr[2], m_new[2], m_use[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    m_new[h] = fmaxf(m_run[h], mx[h]);
                    // a row that has seen no visible key yet keeps m = -inf: use 0 as the exponent offset (p = 0)
                    m_use[h] = m_new[h] == -INFINITY ? 0.f : m_new[h];
                    corr[h] = exp2f(m_run[h] - m_use[h]);  // m_run = -inf before the first visible key -> 0
                    m_run[h] = m_new[h];
                    l_run[h] *= corr[h];
                }
#pragma unroll
                for (int i = 0; i < HD / 8; ++i) {
                    o[i][0] *= corr[0];
                    o[i][1] *= corr[0];
                    o[i][2] *= corr[1];
                    o[i][3] *= corr[1];
                }
                uint32_t pf[4][4];  // P as A fragments: 4 k-steps of 16 keys
                float ls[2] = {0.f, 0.f};
#pragma unroll
                for (int n = 0; n < 8; ++n) {
                    const float p0 = exp2f(s[n][0] - m_use[0]), p1 = exp2f(s[n][1] - m_use[0]);
                    const float p2 = exp2f(s[n][2] - m_use[1]), p3 = exp2f(s[n][3] - m_use[1]);
                    ls[0] += p0 + p1;
                    ls[1] += p2 + p3;
                    const int ks = n >> 1;
                    if ((n & 1) == 0) {
                        pf[ks][0] = pack_op(p0, p1);
                        pf[ks][1] = pack_op(p2, p3);
                    } else {
                        pf[ks][2] = pack_op(p0, p1);
                        pf[ks][3] = pack_op(p2, p3);
                    }
                }
                l_run[0] += ls[0];
                l_run[1] += ls[1];
                // ---- O += P V
#pragma unroll
                for (int ks = 0; ks < 4; ++ks) {
                    if (ks < ng) {
#pragma unroll
                        for (int dp = 0; dp < HD / 16; ++dp) {  // pairs of 8-wide output column groups
                            uint32_t b0, b1, b2, b3;
                            const int r = ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
                            const int c = dp * 16 + (lane >> 4) * 8;
                            ldmatrix_x4_trans(b0, b1, b2, b3, smem_u32(&tV[r * LDS + c]));
                            mma_bf16_16816(o[2 * dp], pf[ks][0], pf[ks][1], pf[ks][2], pf[ks][3], b0, b1);
                            mma_bf16_16816(o[2 * dp + 1], pf[ks][0], pf[ks][1], pf[ks][2], pf[ks][3], b2, b3);
                        }
                    }
                }
            }
        }
        __syncthreads();  // tile t fully consumed: its buffer may be refilled
    }
    cp_async_wait_all();
    if (!active) return;
    // ---- finalize
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
        l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
    }
    const int r0 = q0 + warp * 16 + (lane >> 2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int r = r0 + h * 8;
        if (r < sd.q_len) {
            const float inv = 1.f / l_run[h];
            op_t* op = O + (long long)(sd.o_off + r) * ldo + head * HD + (lane & 3) * 2;
#pragma unroll
            for (int i = 0; i < HD / 8; ++i) {
                *reinterpret_cast<uint32_t*>(op + i * 8) = pack_op(o[i][2 * h] * inv, o[i][2 * h + 1] * inv);
            }
        }
    }
}

template <int HD, int MASKED, int QT>
static int launch_fa(dim3 grid, const op_t* q, long long ldq, const op_t* k, const op_t* v,
                     long long ldkv, op_t* o, long long ldo, const SeqDesc* seqs, float scale_log2,
                     cudaStream_t st) {
    constexpr int smem = (QT + 4 * 64) * (HD + 8) * 2;
    static unsigned long long attr_done = 0;   // per device
    if (first_launch_on_device(&attr_done)) {
        if (cudaFuncSetAttribute(flash_attn_kernel<HD, MASKED, QT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) !=
            cudaSuccess) {
            set_error("flash attention: cannot reserve %d bytes of shared memory", smem);
            return 1;
        }
    }
    flash_attn_kernel<HD, MASKED, QT><<<grid, QT * 2, smem, st>>>(q, ldq, k, v, ldkv, o, ldo, seqs, scale_log2);
    return 0;
}

int launch_flash_attention(const void* Q, long long ldq, long long q_rows, const void* K, const void* V, long long ldkv,
                           long long kv_rows, void* O, long long ldo, const SeqDesc* seqs, int nseq, int max_q_len,
                           int heads, int head_dim, int masked, cudaStream_t st, int impl) {
    if (nseq <= 0) return 0;
    if (impl == 0) {
        // YTK_ATTN=legacy: the round-1 mma.sync kernel; default: the wgmma kernel
        static const int env_impl = [] {
            const char* e = getenv("YTK_ATTN");
            return (e && e[0] == 'l') ? 1 : 2;
        }();
        impl = env_impl;
    }
    if (impl != 1 && impl != 2) {
        set_error("flash attention: impl %d unknown (1 = mma.sync, 2 = wgmma)", impl);
        return 1;
    }
    if (impl == 2)
        return launch_attention_tc(Q, ldq, q_rows, K, V, ldkv, kv_rows, O, ldo, seqs, nseq, heads, head_dim, masked, st);
    // 128-query tiles (8 warps) halve the K/V re-reads of the typical 92..200-token crop; short sequences keep 64
    const int qt = max_q_len > 64 ? 128 : 64;
    dim3 grid((max_q_len + qt - 1) / qt, heads, nseq);
    const float scale_log2 = 1.4426950408889634f / sqrtf((float)head_dim);
    const op_t *q = reinterpret_cast<const op_t*>(Q), *k = reinterpret_cast<const op_t*>(K),
                        *v = reinterpret_cast<const op_t*>(V);
    op_t* o = reinterpret_cast<op_t*>(O);
    int rc = 0;
#define YTK_FA(HD_)                                                                                      \
    do {                                                                                                 \
        if (masked && qt == 128) rc = launch_fa<HD_, 1, 128>(grid, q, ldq, k, v, ldkv, o, ldo, seqs, scale_log2, st); \
        else if (masked) rc = launch_fa<HD_, 1, 64>(grid, q, ldq, k, v, ldkv, o, ldo, seqs, scale_log2, st);          \
        else if (qt == 128) rc = launch_fa<HD_, 0, 128>(grid, q, ldq, k, v, ldkv, o, ldo, seqs, scale_log2, st);      \
        else rc = launch_fa<HD_, 0, 64>(grid, q, ldq, k, v, ldkv, o, ldo, seqs, scale_log2, st);                      \
    } while (0)
    switch (head_dim) {
        case 32: YTK_FA(32); break;
        case 48: YTK_FA(48); break;
        case 64: YTK_FA(64); break;
        case 96: YTK_FA(96); break;
        default: set_error("flash attention: head_dim %d unsupported (32/48/64/96)", head_dim); return 1;
    }
#undef YTK_FA
    if (rc) return 1;
    count_launch();
    return cudaGetLastError() != cudaSuccess;
}

// =================================================================================================== decoder attention
constexpr int kMaxS = 101;
constexpr int kMaxHd = 96;

// =================================================================================================== single-query attention
// Both attentions of an AR step have ONE query per (row, head) against a strided list of cached K/V rows:
//   mode 0  self : q = q_shared[step], keys = the row's content cache [row][pos][2D] (stride 2D), nk = step + 1
//   mode 1  cross: q = qc[row],        keys = the row's encoder memory K/V (stride 2D), nk = ntok
// One warp per (row, head), no block-level synchronisation.  LPK lanes share a key (each owns CPL 16-byte chunks of the
// head dim), 32/LPK key subsets run side by side, so every lane keeps several independent 16-byte loads in flight -
// the step is HBM-bound on exactly these reads.
template <int HD>
__global__ void __launch_bounds__(128) single_query_attn_kernel(int mode, const op_t* __restrict__ qsrc,
                                                                const op_t* __restrict__ kv, int B, int S,
                                                                int D, int heads, const int* __restrict__ step_dev,
                                                                const CropDesc* __restrict__ descs,
                                                                op_t* __restrict__ out) {
    constexpr int NCH = HD / 8;
    constexpr int LPK = (NCH % 4 == 0) ? 4 : 2;   // lanes per key
    constexpr int CPL = NCH / LPK;                // 16-byte chunks per lane
    constexpr int NSUB = 32 / LPK;                // key subsets
    __shared__ float sP[4][kMaxMem];
    pdl_wait();   // (no early launch_dependents: this grid runs in many waves and a dependent persistent GEMM CTA that
                  // becomes resident early takes its SM away from the remaining waves)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wid = blockIdx.x * 4 + warp;
    if (wid >= B * heads) return;
    const int row = wid / heads, head = wid - row * heads;
    const int part = lane % LPK, sub = lane / LPK;
    int nk;
    long long kstride;
    const op_t *qp, *kbase;
    if (mode == 0) {
        const int i = *step_dev;
        nk = i + 1;
        kstride = 2 * D;
        qp = qsrc + (long long)i * D + head * HD;
        kbase = kv + (long long)row * S * (2 * D) + head * HD;
    } else {
        const CropDesc d = descs[row];
        nk = d.ntok;
        kstride = 2 * D;
        qp = qsrc + (long long)row * D + head * HD;
        kbase = kv + (long long)d.tok_off * (2 * D) + head * HD;
    }
    // this lane's slice of the query in registers
    float q[8 * CPL];
#pragma unroll
    for (int c = 0; c < CPL; ++c) {
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(qp) + part * CPL + c);
        q[8 * c + 0] = op_lo(u.x); q[8 * c + 1] = op_hi(u.x); q[8 * c + 2] = op_lo(u.y); q[8 * c + 3] = op_hi(u.y);
        q[8 * c + 4] = op_lo(u.z); q[8 * c + 5] = op_hi(u.z); q[8 * c + 6] = op_lo(u.w); q[8 * c + 7] = op_hi(u.w);
    }
    const float scale = rsqrtf((float)HD);
    float* myP = sP[warp];
    // ---- scores
#pragma unroll 4
    for (int j0 = 0; j0 < nk; j0 += NSUB) {   // warp-uniform trip count: the shuffles below need every lane
        const int j = j0 + sub;
        const bool valid = j < nk;
        const uint4* kp = reinterpret_cast<const uint4*>(kbase + (long long)(valid ? j : 0) * kstride) + part * CPL;
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < CPL; ++c) {
            const uint4 u = valid ? __ldg(kp + c) : make_uint4(0, 0, 0, 0);
            s += q[8 * c + 0] * op_lo(u.x) + q[8 * c + 1] * op_hi(u.x) + q[8 * c + 2] * op_lo(u.y) +
                 q[8 * c + 3] * op_hi(u.y) + q[8 * c + 4] * op_lo(u.z) + q[8 * c + 5] * op_hi(u.z) +
                 q[8 * c + 6] * op_lo(u.w) + q[8 * c + 7] * op_hi(u.w);
        }
#pragma unroll
        for (int o = 1; o < LPK; o <<= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (valid && part == 0) myP[j] = s * scale;
    }
    __syncwarp();
    float mx = -INFINITY;
    for (int j = lane; j < nk; j += 32) mx = fmaxf(mx, myP[j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int j = lane; j < nk; j += 32) {
        const float p = __expf(myP[j] - mx);
        myP[j] = p;
        sum += p;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    __syncwarp();
    // ---- weighted value sum
    float acc[8 * CPL];
#pragma unroll
    for (int e = 0; e < 8 * CPL; ++e) acc[e] = 0.f;
#pragma unroll 4
    for (int j = sub; j < nk; j += NSUB) {
        const float p = myP[j];
        const uint4* vp = reinterpret_cast<const uint4*>(kbase + (long long)j * kstride + D) + part * CPL;
#pragma unroll
        for (int c = 0; c < CPL; ++c) {
            const uint4 u = __ldg(vp + c);
            acc[8 * c + 0] += p * op_lo(u.x); acc[8 * c + 1] += p * op_hi(u.x);
            acc[8 * c + 2] += p * op_lo(u.y); acc[8 * c + 3] += p * op_hi(u.y);
            acc[8 * c + 4] += p * op_lo(u.z); acc[8 * c + 5] += p * op_hi(u.z);
            acc[8 * c + 6] += p * op_lo(u.w); acc[8 * c + 7] += p * op_hi(u.w);
        }
    }
#pragma unroll
    for (int o = LPK; o < 32; o <<= 1) {
#pragma unroll
        for (int e = 0; e < 8 * CPL; ++e) acc[e] += __shfl_xor_sync(0xffffffffu, acc[e], o);
    }
    if (sub == 0) {
        const float inv = 1.f / sum;
        uint4* op = reinterpret_cast<uint4*>(out + (long long)row * D + head * HD) + part * CPL;
#pragma unroll
        for (int c = 0; c < CPL; ++c) {
            uint4 o;
            o.x = pack_op(acc[8 * c + 0] * inv, acc[8 * c + 1] * inv);
            o.y = pack_op(acc[8 * c + 2] * inv, acc[8 * c + 3] * inv);
            o.z = pack_op(acc[8 * c + 4] * inv, acc[8 * c + 5] * inv);
            o.w = pack_op(acc[8 * c + 6] * inv, acc[8 * c + 7] * inv);
            op[c] = o;
        }
    }
}

static int launch_single_query_attn(int mode, const void* qsrc, const void* kv, int B, int S, int D, int heads,
                                    const int* step_dev, const CropDesc* descs, void* out, cudaStream_t st) {
    const int hd = D / heads;
    const unsigned grid = (B * heads + 3) / 4;
    const op_t *q = reinterpret_cast<const op_t*>(qsrc), *k = reinterpret_cast<const op_t*>(kv);
    op_t* o = reinterpret_cast<op_t*>(out);
    cudaError_t e;
    switch (hd) {
        case 32: e = launch_pdl(single_query_attn_kernel<32>, dim3(grid), dim3(128), 0, st, mode, q, k, B, S, D, heads, step_dev, descs, o); break;
        case 48: e = launch_pdl(single_query_attn_kernel<48>, dim3(grid), dim3(128), 0, st, mode, q, k, B, S, D, heads, step_dev, descs, o); break;
        case 64: e = launch_pdl(single_query_attn_kernel<64>, dim3(grid), dim3(128), 0, st, mode, q, k, B, S, D, heads, step_dev, descs, o); break;
        case 96: e = launch_pdl(single_query_attn_kernel<96>, dim3(grid), dim3(128), 0, st, mode, q, k, B, S, D, heads, step_dev, descs, o); break;
        default: set_error("single-query attention: head dim %d unsupported (32/48/64/96)", hd); return 1;
    }
    count_launch();
    return e != cudaSuccess;
}

// Query stream vs. content K/V cache (reference DecoderLayer.forward_stream self_attn, parseq_transformer.py:83-90):
// AR step i = *step_dev, one query (position i) per row, keys 0..i of the row's cache.
int launch_dec_self_attn(const void* q_shared, const void* ckv, int B, int S, int D, int heads, const int* step_dev,
                         void* out, cudaStream_t st) {
    return launch_single_query_attn(0, q_shared, ckv, B, S, D, heads, step_dev, nullptr, out, st);
}

// One query per row against the row's encoder memory (reference cross_attn, parseq_transformer.py:92).  The memory
// K/V were projected ONCE (the reference re-projects them every step, SURVEY.md R7).
int launch_dec_cross_attn(const void* qc, const void* memkv, const CropDesc* descs, int B, int D, int heads, void* out,
                          cudaStream_t st) {
    return launch_single_query_attn(1, qc, memkv, B, 0, D, heads, nullptr, descs, out, st);
}

// =================================================================================================== AR control
// Per row: arg-max of the step's logits, the reference's bookkeeping (parseq.py:220-250) and the embedding of the
// token that enters the context at position j = i + 1.  A second tiny kernel closes groups whose rows all hold an EOS.
__device__ __forceinline__ void warp_argmax(float& v, int& idx) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
        if (ov > v || (ov == v && oi < idx)) {
            v = ov;
            idx = oi;
        }
    }
}

__device__ int detect_repeat(const int* seq, int n, int period_max, int min_run_p1, int min_repeats, int* period) {
    // seq[0..n): emitted tokens; returns onset index or -1 (reference _detect_repeat_onset, parseq.py:108-128)
    for (int p = 1; p <= period_max; ++p) {
        if (n < 2 * p) continue;
        int reps = 1, start = n - p;
        while (start - p >= 0) {
            bool same = true;
            for (int t = 0; t < p; ++t)
                if (seq[start - p + t] != seq[n - p + t]) {
                    same = false;
                    break;
                }
            if (!same) break;
            ++reps;
            start -= p;
        }
        if (reps >= (p == 1 ? min_run_p1 : min_repeats)) {
            *period = p;
            return start;
        }
    }
    return -1;
}

__global__ void __launch_bounds__(256) ar_control_kernel(const float* __restrict__ logits, long long ldl, int C, int npart, int S,
                                                         const int* __restrict__ row_group, int g0, int ngroups,
                                                         ArState a, int eos_id, int rep_on, int rep_period_max, int rep_min_run_p1,
                                                         int rep_min_repeats, const float* __restrict__ embed,
                                                         const float* __restrict__ pos_q, int D, int d_real,
                                                         const float* __restrict__ g_c, const float* __restrict__ b_c,
                                                         op_t* __restrict__ cin) {
    __shared__ float sv[8];
    __shared__ int si[8];
    __shared__ int s_tok;
    __shared__ float s_stat[2];
    __shared__ float red[8];
    __shared__ int s_last;
    pdl_wait();   // (no early launch_dependents: this grid runs in many waves and a dependent persistent GEMM CTA that
                  // becomes resident early takes its SM away from the remaining waves)
    const int row = blockIdx.x;
    const int i = *a.step;
    const int j = i + 1;
    const int grp = row_group[row];
    const bool running = a.group_len[grp] == 0;  // finished group: nothing more happens to its rows
    if (running) {
        const float* lr = logits + (long long)row * ldl;
        float best = -INFINITY;
        int bi = 0x7fffffff;
        if (npart > 0) {
            // fused head epilogue (gemm_tc EPI_ROWMAX): `logits` holds float4 partials {max, sum, index, -}, ldl per row
            const float4* pr = reinterpret_cast<const float4*>(logits) + (long long)row * ldl;
            for (int v = threadIdx.x; v < npart; v += blockDim.x) {
                const float4 x = __ldg(pr + v);
                const int xi = __float_as_int(x.z);
                if (x.x > best || (x.x == best && xi < bi)) {
                    best = x.x;
                    bi = xi;
                }
            }
        } else {
            const int nvec = C >> 2;
            const float4* l4 = reinterpret_cast<const float4*>(lr);
            for (int v = threadIdx.x; v < nvec; v += blockDim.x) {   // strict '>' keeps the smallest index (ascending)
                const float4 x = __ldg(l4 + v);
                if (x.x > best) { best = x.x; bi = 4 * v; }
                if (x.y > best) { best = x.y; bi = 4 * v + 1; }
                if (x.z > best) { best = x.z; bi = 4 * v + 2; }
                if (x.w > best) { best = x.w; bi = 4 * v + 3; }
            }
            for (int c = 4 * nvec + threadIdx.x; c < C; c += blockDim.x) {
                const float v = lr[c];
                if (v > best) { best = v; bi = c; }
            }
        }
        warp_argmax(best, bi);
        if ((threadIdx.x & 31) == 0) {
            sv[threadIdx.x >> 5] = best;
            si[threadIdx.x >> 5] = bi;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            float v = sv[0];
            int id = si[0];
            for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
                if (sv[w] > v || (sv[w] == v && si[w] < id)) {
                    v = sv[w];
                    id = si[w];
                }
            a.raw[row * S + i] = id;
            int tok = id;
            int has = a.has_eos[row];
            if (j < S) {
                a.tgt[row * S + j] = id;
                if (rep_on && !a.rep_done[row] && id != eos_id) {
                    int period = 0;
                    const int onset = detect_repeat(a.tgt + row * S + 1, j, rep_period_max, rep_min_run_p1,
                                                    rep_min_repeats, &period);
                    if (onset >= 0) {
                        a.rep_cut[row] = onset + period;
                        a.rep_done[row] = 1;
                        a.tgt[row * S + j] = eos_id;
                        tok = eos_id;
                    }
                }
                if (tok == eos_id) {
                    a.has_eos[row] = 1;
                    has = 1;
                }
            }
            if (!has) atomicAdd(&a.open_rows[grp], 1);
            s_tok = tok;
        }
        __syncthreads();
        if (j < S) {
            // content embedding of position j: pos_queries[j-1] + sqrt(D) * E[tok], then LN_c (eps 1e-5)
            const int tok = s_tok;
            const float sq = sqrtf((float)D);
            float loc[4];  // D <= 1024 with 256 threads
            float s = 0.f;
            for (int t = 0; t < 4; ++t) {
                const int d = threadIdx.x + t * 256;
                float v = 0.f;
                if (d < D) v = pos_q[(long long)(j - 1) * D + d] + sq * embed[(long long)tok * D + d];
                loc[t] = v;
                s += v;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
            __syncthreads();
            if (threadIdx.x == 0) {
                float t = 0.f;
                for (int w = 0; w < 8; ++w) t += red[w];
                s_stat[0] = t / (float)d_real;
            }
            __syncthreads();
            const float mean = s_stat[0];
            float q = 0.f;
            for (int t = 0; t < 4; ++t) {
                const int d = threadIdx.x + t * 256;
                if (d < d_real) q += (loc[t] - mean) * (loc[t] - mean);
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
            if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = q;
            __syncthreads();
            if (threadIdx.x == 0) {
                float t = 0.f;
                for (int w = 0; w < 8; ++w) t += red[w];
                s_stat[1] = rsqrtf(t / (float)d_real + 1e-5f);
            }
            __syncthreads();
            const float rstd = s_stat[1];
            for (int t = 0; t < 4; ++t) {
                const int d = threadIdx.x + t * 256;
                if (d < D) cin[(long long)row * D + d] = f2op((loc[t] - mean) * rstd * g_c[d] + b_c[d]);
            }
        }
    }
    // ---- the CTA that finishes last closes the step: a group ends after step i when every one of its rows holds an
    // EOS (parseq.py:245-250).  Every CTA read *a.step / group_len before taking its ticket, so the updates below
    // cannot be seen by this launch.
    if (threadIdx.x == 0) {
        __threadfence();
        s_last = atomicAdd(a.ticket, 1) == (int)gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    __shared__ int active;
    if (threadIdx.x == 0) active = 0;
    __syncthreads();
    for (int g = g0 + threadIdx.x; g < g0 + ngroups; g += blockDim.x) {  // the groups of this launch's rows
        if (a.group_len[g] == 0) {
            const int open = atomicExch(&a.open_rows[g], 0);
            if (j >= S) a.group_len[g] = S;          // ran all the steps
            else if (open == 0) a.group_len[g] = j;  // logits has j entries, tgt_in for refinement length j
            else atomicAdd(&active, 1);
        } else {
            a.open_rows[g] = 0;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        *a.n_active = active;
        *a.step = i + 1;
        *a.ticket = 0;
    }
}

int launch_ar_control(const float* logits, long long ldl, int C, int npart, int B, int S, const int* row_group, int g0,
                      int ngroups, ArState a, int eos_id, int rep_on, int rep_period_max, int rep_min_run_p1, int rep_min_repeats,
                      const float* embed, const float* pos_q, int D, int d_real, const float* g_c, const float* b_c,
                      void* cin, cudaStream_t st) {
    if (D > 1024) {
        set_error("ar_control: D=%d too large", D);
        return 1;
    }
    const cudaError_t e = launch_pdl(ar_control_kernel, dim3(B), dim3(256), 0, st, logits, ldl, C, npart, S, row_group, g0,
                                     ngroups, a, eos_id, rep_on, rep_period_max, rep_min_run_p1, rep_min_repeats, embed,
                                     pos_q, D, d_real, g_c, b_c, reinterpret_cast<op_t*>(cin));
    count_launch(1);
    return e != cudaSuccess;
}

// =================================================================================================== refinement embed
__global__ void __launch_bounds__(256) refine_embed_kernel(const int* __restrict__ raw,
                                                           const int* __restrict__ row_group,
                                                           const int* __restrict__ group_len, int S, int bos_id,
                                                           int eos_id, const float* __restrict__ embed,
                                                           const float* __restrict__ pos_q, int D, int d_real,
                                                           const float* __restrict__ g_c, const float* __restrict__ b_c,
                                                           op_t* __restrict__ cin, int* __restrict__ klen,
                                                           int* __restrict__ kpad) {
    // grid (S, B): content position `pos` of row `row`; tgt_in = [BOS, raw[0..L-2]] (parseq.py:286)
    const int pos = blockIdx.x, row = blockIdx.y;
    const int L = group_len[row_group[row]];
    if (pos == 0 && threadIdx.x == 0) {
        klen[row] = L;
        int first = L;  // first EOS in tgt_in -> keys at/after it are padding (parseq.py:288-290)
        for (int p = 1; p < L; ++p)
            if (raw[row * S + p - 1] == eos_id) {
                first = p;
                break;
            }
        kpad[row] = first;
    }
    __shared__ float red[8];
    __shared__ float s_stat[2];
    const float sq = sqrtf((float)D);
    const int tok = (pos == 0) ? bos_id : ((pos < L) ? raw[row * S + pos - 1] : eos_id);
    float loc[4];
    float s = 0.f;
    for (int t = 0; t < 4; ++t) {
        const int d = threadIdx.x + t * 256;
        float v = 0.f;
        if (d < D) v = sq * embed[(long long)tok * D + d] + (pos > 0 ? pos_q[(long long)(pos - 1) * D + d] : 0.f);
        loc[t] = v;
        s += v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int w = 0; w < 8; ++w) t += red[w];
        s_stat[0] = t / (float)d_real;   // padded features are zero: the sum is over the real ones
    }
    __syncthreads();
    const float mean = s_stat[0];
    float q = 0.f;
    for (int t = 0; t < 4; ++t) {
        const int d = threadIdx.x + t * 256;
        if (d < d_real) q += (loc[t] - mean) * (loc[t] - mean);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = q;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int w = 0; w < 8; ++w) t += red[w];
        s_stat[1] = rsqrtf(t / (float)d_real + 1e-5f);
    }
    __syncthreads();
    const float rstd = s_stat[1];
    // layout [row][pos][D]: the K/V GEMM output is the cache layout [row][pos][2D]
    const long long orow = (long long)row * S + pos;
    for (int t = 0; t < 4; ++t) {
        const int d = threadIdx.x + t * 256;
        if (d < D) cin[orow * D + d] = f2op((loc[t] - mean) * rstd * g_c[d] + b_c[d]);
    }
}

int launch_refine_embed(const int* raw, const int* row_group, const int* group_len, int B, int S, int bos_id, int eos_id,
                        const float* embed, const float* pos_q, int D, int d_real, const float* g_c, const float* b_c,
                        void* cin, int* klen, int* kpad, cudaStream_t st) {
    dim3 grid(S, B);
    refine_embed_kernel<<<grid, 256, 0, st>>>(raw, row_group, group_len, S, bos_id, eos_id, embed, pos_q, D, d_real, g_c, b_c,
                                              reinterpret_cast<op_t*>(cin), klen, kpad);
    count_launch();
    return cudaGetLastError() != cudaSuccess;
}

// =================================================================================================== softmax max
// Replaces `.softmax(-1)` + per-position max of the reference (text_recognizer.py:255, parseq_tokenizer.py:79-87):
// only (argmax id, max probability) leave the device.  One CTA per logits row.
// online (max, sum-exp, arg-max) triple: one pass over the row
struct SmStat {
    float m, s;
    int i;
};
__device__ __forceinline__ void sm_push(SmStat& a, float v, int idx) {
    if (v > a.m) {
        a.s = a.s * __expf(a.m - v) + 1.f;
        a.m = v;
        a.i = idx;
    } else {
        a.s += __expf(v - a.m);
    }
}
__device__ __forceinline__ void sm_merge(SmStat& a, const SmStat& b) {
    if (b.s == 0.f) return;  // empty partial (no elements seen)
    if (b.m > a.m || (b.m == a.m && b.i < a.i)) {
        a.s = a.s * __expf(a.m - b.m) + b.s;
        a.m = b.m;
        a.i = b.i;
    } else {
        a.s += b.s * __expf(b.m - a.m);
    }
}

__global__ void __launch_bounds__(256) softmax_max_kernel(const float* __restrict__ logits, long long ldl, int C, int S,
                                                          long long g_stride, long long g_off,
                                                          const int* __restrict__ rep_cut, int eos_id,
                                                          int* __restrict__ ids, float* __restrict__ probs) {
    const int r = blockIdx.x;  // local row in this logits buffer
    const long long g = (long long)r * g_stride + g_off;  // global (crop*S + position)
    const int crop = (int)(g / S), pos = (int)(g % S);
    if (rep_cut != nullptr && rep_cut[crop] == pos) {  // parseq.py:301-309: logits = -30 everywhere, +30 at EOS
        if (threadIdx.x == 0) {
            ids[g] = eos_id;
            probs[g] = 1.f / (1.f + (float)(C - 1) * expf(-60.f));
        }
        return;
    }
    const float* lr = logits + (long long)r * ldl;   // rows are 16-byte aligned (ldl % 4 == 0)
    SmStat st{-INFINITY, 0.f, 0x7fffffff};
    const int nvec = C >> 2;
    const float4* l4 = reinterpret_cast<const float4*>(lr);
    for (int v = threadIdx.x; v < nvec; v += 256) {
        const float4 x = __ldg(l4 + v);
        sm_push(st, x.x, 4 * v);
        sm_push(st, x.y, 4 * v + 1);
        sm_push(st, x.z, 4 * v + 2);
        sm_push(st, x.w, 4 * v + 3);
    }
    for (int c = 4 * nvec + threadIdx.x; c < C; c += 256) sm_push(st, lr[c], c);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        SmStat b;
        b.m = __shfl_xor_sync(0xffffffffu, st.m, o);
        b.s = __shfl_xor_sync(0xffffffffu, st.s, o);
        b.i = __shfl_xor_sync(0xffffffffu, st.i, o);
        sm_merge(st, b);
    }
    __shared__ SmStat sw[8];
    if ((threadIdx.x & 31) == 0) sw[threadIdx.x >> 5] = st;
    __syncthreads();
    if (threadIdx.x == 0) {
        SmStat a = sw[0];
        for (int w = 1; w < 8; ++w) sm_merge(a, sw[w]);
        ids[g] = a.i;
        probs[g] = 1.f / a.s;
    }
}

// Same result from the partials of the fused head epilogue (gemm_tc EPI_ROWMAX): one warp per row merges the
// 2 * tiles_n (max, sum exp, arg-max) triples.
__global__ void __launch_bounds__(256) rowmax_finalize_kernel(const float4* __restrict__ part, long long ldp, int npart,
                                                              int rows, int C, int S, long long g_stride, long long g_off,
                                                              const int* __restrict__ rep_cut, int eos_id,
                                                              int* __restrict__ ids, float* __restrict__ probs) {
    const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= rows) return;
    const long long g = (long long)r * g_stride + g_off;
    const int crop = (int)(g / S), pos = (int)(g % S);
    if (rep_cut != nullptr && rep_cut[crop] == pos) {
        if (lane == 0) {
            ids[g] = eos_id;
            probs[g] = 1.f / (1.f + (float)(C - 1) * expf(-60.f));
        }
        return;
    }
    SmStat st{-INFINITY, 0.f, 0x7fffffff};
    const float4* pr = part + (long long)r * ldp;
    for (int v = lane; v < npart; v += 32) {
        const float4 x = __ldg(pr + v);
        SmStat b{x.x, x.y, __float_as_int(x.z)};
        sm_merge(st, b);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        SmStat b;
        b.m = __shfl_xor_sync(0xffffffffu, st.m, o);
        b.s = __shfl_xor_sync(0xffffffffu, st.s, o);
        b.i = __shfl_xor_sync(0xffffffffu, st.i, o);
        sm_merge(st, b);
    }
    if (lane == 0) {
        ids[g] = st.i;
        probs[g] = 1.f / st.s;
    }
}

int launch_rowmax_finalize(const float* partials, long long ldp, int npart, int C, int rows, int S, long long g_stride,
                           long long g_off, const int* rep_cut, int eos_id, int* ids, float* probs, cudaStream_t st) {
    if (rows <= 0) return 0;
    rowmax_finalize_kernel<<<(rows * 32 + 255) / 256, 256, 0, st>>>(reinterpret_cast<const float4*>(partials), ldp, npart,
                                                                    rows, C, S, g_stride, g_off, rep_cut, eos_id, ids,
                                                                    probs);
    count_launch();
    return cudaGetLastError() != cudaSuccess;
}

int launch_softmax_max(const float* logits, long long ldl, int C, int rows, int S, long long g_stride, long long g_off,
                       const int* rep_cut, int eos_id, int* ids, float* probs, cudaStream_t st) {
    if (rows <= 0) return 0;
    softmax_max_kernel<<<rows, 256, 0, st>>>(logits, ldl, C, S, g_stride, g_off, rep_cut, eos_id, ids, probs);
    count_launch();
    return cudaGetLastError() != cudaSuccess;
}

// Broadcast one row to many (content K/V of the BOS position is identical for every crop).
__global__ void bcast_rows_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int vec_per_row,
                                  long long dst_stride_vec, long long total) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < total) dst[(i / vec_per_row) * dst_stride_vec + i % vec_per_row] = src[i % vec_per_row];
}
int launch_bcast_rows(const void* src, void* dst, int row_bytes, long long dst_stride_bytes, int rows,
                      cudaStream_t st) {
    const int vpr = row_bytes / 16;
    const long long total = (long long)vpr * rows;
    if (total <= 0) return 0;
    bcast_rows_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
        reinterpret_cast<const uint4*>(src), reinterpret_cast<uint4*>(dst), vpr, dst_stride_bytes / 16, total);
    count_launch();
    return cudaGetLastError() != cudaSuccess;
}

// refine_iters == 0: the AR logits are the output; apply the repetition patch after the loop (parseq.py:301-309).
__global__ void apply_rep_cut_kernel(const int* __restrict__ rep_cut, int B, int S, int C, int eos_id,
                                     int* __restrict__ ids, float* __restrict__ probs) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= B) return;
    const int cut = rep_cut[r];
    if (cut >= 0 && cut < S) {
        ids[r * S + cut] = eos_id;
        probs[r * S + cut] = 1.f / (1.f + (float)(C - 1) * expf(-60.f));
    }
}
int launch_apply_rep_cut(const int* rep_cut, int B, int S, int C, int eos_id, int* ids, float* probs,
                         cudaStream_t st) {
    apply_rep_cut_kernel<<<(B + 127) / 128, 128, 0, st>>>(rep_cut, B, S, C, eos_id, ids, probs);
    count_launch();
    return cudaGetLastError() != cudaSuccess;
}

// Per-row descriptors of the refinement self-attention: queries = the shared projected pos_queries (rows 0..S-1 of
// q_shared), keys = this row's content K/V cache (key j at ckv[(row*S + j) * 2D]), output rows row*S ...
__global__ void refine_seqs_kernel(const int* __restrict__ klen, const int* __restrict__ kpad, int B, int S, int D,
                                   SeqDesc* __restrict__ seqs) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= B) return;
    SeqDesc d;
    d.q_off = 0;
    d.q_len = S;
    d.o_off = r * S;
    d.k_len = klen[r];
    d.k_base = (long long)r * S * (2 * D);
    d.kpad = kpad[r];
    d.pad_ = 0;
    seqs[r] = d;
}
int launch_refine_seqs(const int* klen, const int* kpad, int B, int S, int D, SeqDesc* seqs, cudaStream_t st) {
    refine_seqs_kernel<<<(B + 127) / 128, 128, 0, st>>>(klen, kpad, B, S, D, seqs);
    count_launch();
    return cudaGetLastError() != cudaSuccess;
}

__global__ void fill_i32_kernel(int* p, int v, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}
int launch_fill_i32(int* p, int v, long long n, cudaStream_t st) {
    if (n <= 0) return 0;
    fill_i32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(p, v, n);
    return cudaGetLastError() != cudaSuccess;
}

}  // namespace ytk
