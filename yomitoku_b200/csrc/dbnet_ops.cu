// Memory-bound CUDA kernels around the wgmma convolutions of DBNet++ (all NHWC bf16, 8-channel = 16-byte vectors).
// Each kernel cites the reference op it replaces; they are HBM-bound by construction (no data reuse beyond a 3x3
// neighbourhood), so the design rule is: coalesced 16 B accesses, one pass, no intermediate tensors.
#include "dbnet_ops.h"

#include "gemm_tc.h"
#include "ptx.cuh"
#include "resample_math.h"

namespace ytk {

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
    f[0] = op_lo(u.x); f[1] = op_hi(u.x); f[2] = op_lo(u.y); f[3] = op_hi(u.y);
    f[4] = op_lo(u.z); f[5] = op_hi(u.z); f[6] = op_lo(u.w); f[7] = op_hi(u.w);
}
__device__ __forceinline__ uint4 pack8(const float* f) {
    uint4 u;
    u.x = pack_op(f[0], f[1]); u.y = pack_op(f[2], f[3]); u.z = pack_op(f[4], f[5]); u.w = pack_op(f[6], f[7]);
    return u;
}

// ------------------------------------------------------------------------------------------------------------------
// Detector pre-processing (reference text_detector.py:99-107, data/functions.py:196-264):
// BGR u8 page -> float -> cv2.resize(INTER_AREA) to (Hn, Wn) -> /255 -> (x - mean[c]) / std[c] applied positionally
// to the B,G,R planes (SURVEY.md Appendix A2) -> network input.  Output layout: zero-padded NHWC with 8 channels,
// pixel (h, w) at padded position (h + 3, w + 3) of a [Hn+6, Wn+8] canvas (the 7x7/stride-2 stem reads it through
// overlapping TMA boxes, see dbnet_engine.cu).  One kernel body; the resampler is the one OpenCV picks by the scales
// of each page: AreaSampler (ResizeArea tables) when both axes shrink or keep their size, AreaUpSampler (bilinear with
// "area-mode" coefficients) when some axis grows.  Both restate OpenCV's tables in fp32.  One page per blockIdx.y, so
// the choice is uniform in a block even when the pages of a launch have different sizes (a page table).
// ------------------------------------------------------------------------------------------------------------------
struct AreaTap { int lo; int hi; float w_lo; float w_mid; float w_hi; };  // src indices [lo, hi], edge weights

__device__ __forceinline__ AreaTap area_tap(int d, double scale, int ssize) {
    // OpenCV computeResizeAreaTab for destination index d
    const double fs1 = d * scale, fs2 = fs1 + scale;
    const double cell = fmin(scale, (double)ssize - fs1);
    int s1 = (int)ceil(fs1), s2 = (int)floor(fs2);
    s2 = min(s2, ssize - 1);
    s1 = min(s1, s2);
    AreaTap t;
    t.w_mid = (float)(1.0 / cell);
    t.lo = s1;
    t.w_lo = 0.f;
    if (s1 - fs1 > 1e-3) {
        t.lo = s1 - 1;
        t.w_lo = (float)((s1 - fs1) / cell);
    }
    t.hi = s2 - 1;
    t.w_hi = 0.f;
    if (fs2 - s2 > 1e-3) {
        t.hi = s2;
        t.w_hi = (float)(fmin(fmin(fs2 - s2, 1.0), cell) / cell);
    }
    return t;
}

// OpenCV's ResizeArea: pixel (h, w) of page img as fp32 B, G, R on the 0..255 scale
struct AreaSampler {
    __device__ __forceinline__ static void sample(const uint8_t* base, int H0, int W0, int Hn, int Wn, int h, int w,
                                                  float* acc) {
        const double sy = (double)H0 / Hn, sx = (double)W0 / Wn;
        const AreaTap ty = area_tap(h, sy, H0), tx = area_tap(w, sx, W0);
        acc[0] = acc[1] = acc[2] = 0.f;
        for (int y = ty.lo; y <= ty.hi; ++y) {
            const float wy = (y == ty.lo && ty.w_lo > 0.f) ? ty.w_lo : ((y == ty.hi && ty.w_hi > 0.f) ? ty.w_hi : ty.w_mid);
            float row[3] = {0.f, 0.f, 0.f};
            for (int x = tx.lo; x <= tx.hi; ++x) {
                const float wx =
                    (x == tx.lo && tx.w_lo > 0.f) ? tx.w_lo : ((x == tx.hi && tx.w_hi > 0.f) ? tx.w_hi : tx.w_mid);
                const uint8_t* p = base + ((size_t)y * W0 + x) * 3;
                row[0] += wx * p[0];
                row[1] += wx * p[1];
                row[2] += wx * p[2];
            }
            acc[0] += wy * row[0];
            acc[1] += wy * row[1];
            acc[2] += wy * row[2];
        }
    }
};

struct UpTap { int s0; int s1; float f; };  // value = S[s0] (1 - f) + S[s1] f

__device__ __forceinline__ UpTap area_up_tap(int d, int ssize, int dsize) {
    // OpenCV resize() with INTER_AREA when some axis grows, for destination index d of one axis (either axis: a
    // shrinking one is sampled the same way).  scale must be 1 / (dsize / ssize) as in OpenCV, not ssize / dsize: where
    // d * scale lands on an integer the two can floor to neighbouring pixels.  The products are rounded on their own
    // (no FMA), as OpenCV's host code computes them.
    const double inv = (double)dsize / ssize, scale = 1.0 / inv;
    int s = (int)floor(__dmul_rn((double)d, scale));          // >= 0: d >= 0
    float f = (float)((double)(d + 1) - __dmul_rn((double)(s + 1), inv));
    f = f <= 0.f ? 0.f : f - floorf(f);
    if (s >= ssize - 1) {
        s = ssize - 1;
        f = 0.f;
    }
    UpTap t;
    t.s0 = s;
    t.s1 = min(s + 1, ssize - 1);  // with f = 0 the second tap adds exactly 0
    t.f = f;
    return t;
}

// OpenCV's INTER_AREA up-scaling: a horizontal pass over two source rows, then a vertical one, in fp32
struct AreaUpSampler {
    __device__ __forceinline__ static void sample(const uint8_t* base, int H0, int W0, int Hn, int Wn, int h, int w,
                                                  float* acc) {
        const UpTap ty = area_up_tap(h, H0, Hn), tx = area_up_tap(w, W0, Wn);
        const uint8_t* r0 = base + (size_t)ty.s0 * W0 * 3;
        const uint8_t* r1 = base + (size_t)ty.s1 * W0 * 3;
        const float ax = 1.f - tx.f, ay = 1.f - ty.f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float v0 = r0[tx.s0 * 3 + c] * ax + r0[tx.s1 * 3 + c] * tx.f;
            const float v1 = r1[tx.s0 * 3 + c] * ax + r1[tx.s1 * 3 + c] * tx.f;
            acc[c] = v0 * ay + v1 * ty.f;
        }
    }
};

// Page img of the launch: from the page table when there is one, else page img of a same-size [n][H0][W0][3] batch.
__global__ void preprocess_kernel(const uint8_t* __restrict__ src, const RtSrc* __restrict__ table, int H0, int W0,
                                  int Hn, int Wn, op_t* __restrict__ dst) {
    const int Hp = Hn + 6, Wp = Wn + 8;
    const int img = blockIdx.y;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= Hp * Wp) return;
    const uint8_t* page = src + (size_t)img * H0 * W0 * 3;
    int H = H0, W = W0;
    if (table) {
        const RtSrc p = table[img];
        page = src + p.page_off;
        H = p.H;
        W = p.W;
    }
    const int wp = idx % Wp;
    const int hp = idx / Wp;
    float o[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const int h = hp - 3, w = wp - 3;
    if (h >= 0 && h < Hn && w >= 0 && w < Wn) {
        float acc[3];
        // OpenCV's rule: true area resampling only when neither axis grows
        if (Hn <= H && Wn <= W)
            AreaSampler::sample(page, H, W, Hn, Wn, h, w, acc);
        else
            AreaUpSampler::sample(page, H, W, Hn, Wn, h, w, acc);
        // channel order seen by the network is B,G,R with the ImageNet RGB mean/std applied positionally
        const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
#pragma unroll
        for (int c = 0; c < 3; ++c) o[c] = (float)(((double)acc[c] / 255.0 - (double)mean[c]) / (double)stdv[c]);
    }
    reinterpret_cast<uint4*>(dst)[(size_t)img * Hp * Wp + idx] = pack8(o);
}

static int preprocess(const uint8_t* src, const RtSrc* table, int n_img, int H0, int W0, int Hn, int Wn, void* dst,
                      cudaStream_t st) {
    if (n_img < 1 || n_img > 65535) return 1;  // one page per blockIdx.y
    const int threads = 256;
    const dim3 grid((unsigned)(((long long)(Hn + 6) * (Wn + 8) + threads - 1) / threads), (unsigned)n_img);
    preprocess_kernel<<<grid, threads, 0, st>>>(src, table, H0, W0, Hn, Wn, reinterpret_cast<op_t*>(dst));
    count_launch();
    return cudaGetLastError() != cudaSuccess;
}

int launch_preprocess(const uint8_t* src, int n_img, int H0, int W0, int Hn, int Wn, void* dst, cudaStream_t st) {
    return preprocess(src, nullptr, n_img, H0, W0, Hn, Wn, dst, st);
}

int launch_preprocess_table(const uint8_t* pages, const RtSrc* table_dev, int n_img, int Hn, int Wn, void* dst,
                            cudaStream_t st) {
    return preprocess(pages, table_dev, n_img, 0, 0, Hn, Wn, dst, st);
}

// Model-level seam: the reference hands DBNet a normalised (N,3,H,W) fp32 tensor (text_detector.py:127-129).  Repack
// it into the same zero-padded 8-channel NHWC bf16 canvas the fused u8 path writes.
__global__ void pack_nchw_kernel(const float* __restrict__ src, int n_img, int Hn, int Wn,
                                 op_t* __restrict__ dst) {
    const int Hp = Hn + 6, Wp = Wn + 8;
    const long long total = (long long)n_img * Hp * Wp;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int wp = (int)(idx % Wp);
    const int hp = (int)((idx / Wp) % Hp);
    const int img = (int)(idx / ((long long)Wp * Hp));
    float o[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const int h = hp - 3, w = wp - 3;
    if (h >= 0 && h < Hn && w >= 0 && w < Wn) {
#pragma unroll
        for (int c = 0; c < 3; ++c) o[c] = __ldg(src + (((size_t)img * 3 + c) * Hn + h) * Wn + w);
    }
    reinterpret_cast<uint4*>(dst)[idx] = pack8(o);
}

int launch_pack_nchw_f32(const float* src, int n_img, int Hn, int Wn, void* dst, cudaStream_t st) {
    const long long total = (long long)n_img * (Hn + 6) * (Wn + 8);
    pack_nchw_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(src, n_img, Hn, Wn,
                                                                       reinterpret_cast<op_t*>(dst));
    count_launch();
    return cudaGetLastError() != cudaSuccess;
}

// ------------------------------------------------------------------------------------------------------------------
// MaxPool2d(kernel 3, stride 2, padding 1) of the ResNet stem (torchvision resnet50.maxpool, reference
// dbnet_plus.py:34-37).  One thread per (output pixel, 8-channel group).
// ------------------------------------------------------------------------------------------------------------------
__global__ void maxpool3x3s2_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, int n_img, int H, int W,
                                    int C8, int Ho, int Wo) {
    const long long total = (long long)n_img * Ho * Wo * C8;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int c = (int)(idx % C8);
    const int wo = (int)((idx / C8) % Wo);
    const int ho = (int)((idx / ((long long)C8 * Wo)) % Ho);
    const int img = (int)(idx / ((long long)C8 * Wo * Ho));
    float m[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) m[j] = -INFINITY;
    for (int dy = 0; dy < 3; ++dy) {
        const int y = 2 * ho - 1 + dy;
        if (y < 0 || y >= H) continue;
        for (int dx = 0; dx < 3; ++dx) {
            const int x = 2 * wo - 1 + dx;
            if (x < 0 || x >= W) continue;
            float f[8];
            unpack8(__ldg(in + (((size_t)img * H + y) * W + x) * C8 + c), f);
#pragma unroll
            for (int j = 0; j < 8; ++j) m[j] = fmaxf(m[j], f[j]);
        }
    }
    out[idx] = pack8(m);
}

int launch_maxpool(const void* in, void* out, int n_img, int H, int W, int C, cudaStream_t st) {
    const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    const long long total = (long long)n_img * Ho * Wo * (C / 8);
    maxpool3x3s2_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
        reinterpret_cast<const uint4*>(in), reinterpret_cast<uint4*>(out), n_img, H, W, C / 8, Ho, Wo);
    count_launch();
    return cudaGetLastError() != cudaSuccess;
}

// ------------------------------------------------------------------------------------------------------------------
// Bilinear upsampling, align_corners=False (F.interpolate / nn.Upsample, reference dbnet_plus.py:65-67,82,92,102,
// 213-218).  dst[.., coff:coff+C] (= or +=) bilinear(src).  PyTorch's source index: (d + 0.5) * (in/out) - 0.5,
// clamped at 0; the upper neighbour is clamped to in-1.
// ------------------------------------------------------------------------------------------------------------------
__global__ void upsample_bilinear_kernel(const uint4* __restrict__ src, int n_img, int Hs, int Ws, int C8,
                                         op_t* __restrict__ dst, int Hd, int Wd, long long ldd, int coff,
                                         int accumulate) {
    const long long total = (long long)n_img * Hd * Wd * C8;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int c = (int)(idx % C8);
    const int wd = (int)((idx / C8) % Wd);
    const int hd = (int)((idx / ((long long)C8 * Wd)) % Hd);
    const int img = (int)(idx / ((long long)C8 * Wd * Hd));
    const float sh = (float)Hs / (float)Hd, sw = (float)Ws / (float)Wd;
    float fy = fmaxf((hd + 0.5f) * sh - 0.5f, 0.f), fx = fmaxf((wd + 0.5f) * sw - 0.5f, 0.f);
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = min(y0 + 1, Hs - 1), x1 = min(x0 + 1, Ws - 1);
    const float ly = fy - y0, lx = fx - x0;
    const size_t b = (size_t)img * Hs * Ws;
    float a00[8], a01[8], a10[8], a11[8], o[8];
    unpack8(__ldg(src + (b + (size_t)y0 * Ws + x0) * C8 + c), a00);
    unpack8(__ldg(src + (b + (size_t)y0 * Ws + x1) * C8 + c), a01);
    unpack8(__ldg(src + (b + (size_t)y1 * Ws + x0) * C8 + c), a10);
    unpack8(__ldg(src + (b + (size_t)y1 * Ws + x1) * C8 + c), a11);
    uint4* dp = reinterpret_cast<uint4*>(dst + (((size_t)img * Hd + hd) * Wd + wd) * ldd + coff + c * 8);
    if (accumulate) {
        unpack8(*dp, o);
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j)
        o[j] += (1.f - ly) * ((1.f - lx) * a00[j] + lx * a01[j]) + ly * ((1.f - lx) * a10[j] + lx * a11[j]);
    *dp = pack8(o);
}

int launch_upsample(const void* src, int n_img, int Hs, int Ws, int C, void* dst, int Hd, int Wd, long long ldd,
                    int coff, int accumulate, cudaStream_t st) {
    const long long total = (long long)n_img * Hd * Wd * (C / 8);
    upsample_bilinear_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
        reinterpret_cast<const uint4*>(src), n_img, Hs, Ws, C / 8, reinterpret_cast<op_t*>(dst), Hd, Wd, ldd,
        coff, accumulate);
    count_launch();
    return cudaGetLastError() != cudaSuccess;
}

// ------------------------------------------------------------------------------------------------------------------
// Adaptive Scale Fusion attention (reference dbnet_feature_attention.py:69-79 and :150-160) after its 3x3 conv.
//   pass 1  asf_pool:    per-image, per-chunk channel sums of a = conv(fuse) -> gsum[N,64 chunks,64] (AdaptiveAvgPool2d(1))
//   pass 2  asf_gate:    g = sigmoid(W2 relu(W1 mean))              -> gvec[N,64], gmean[N]
//   pass 3  asf_cmean:   m[h,w] = mean_c(a + g)                     -> m[N,H,W] fp32
//   pass 4  asf_apply:   s = sigmoid(w1x1 * relu(conv3x3(m))); z = s + a + g; score = sigmoid(Watt z) (4);
//                        fuse[:, 64*i : 64*i+64] *= score[i]        (in place)
// ------------------------------------------------------------------------------------------------------------------
__global__ void asf_pool_kernel(const uint4* __restrict__ a, int HW, float* __restrict__ gsum) {
    // grid (chunks, n_img); 256 threads: thread t handles channel group t%8, pixel lane t/8
    const int img = blockIdx.y;
    const int cg = threadIdx.x & 7, pl = threadIdx.x >> 3;  // 32 pixel lanes
    const int per = (HW + gridDim.x - 1) / gridDim.x;
    const int p0 = blockIdx.x * per, p1 = min(HW, p0 + per);
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int p = p0 + pl; p < p1; p += 32) {
        float f[8];
        unpack8(__ldg(a + ((size_t)img * HW + p) * 8 + cg), f);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += f[j];
    }
    __shared__ float red[32][64];
#pragma unroll
    for (int j = 0; j < 8; ++j) red[pl][cg * 8 + j] = acc[j];
    __syncthreads();
    if (threadIdx.x < 64) {
        float s = 0.f;
        for (int i = 0; i < 32; ++i) s += red[i][threadIdx.x];
        // one partial per (image, chunk): summed in a fixed order by asf_gate_kernel - the forward is deterministic
        gsum[((size_t)img * gridDim.x + blockIdx.x) * 64 + threadIdx.x] = s;
    }
}

__global__ void asf_gate_kernel(const float* __restrict__ gsum, int chunks, int HW, const float* __restrict__ w1 /*16x64*/,
                                const float* __restrict__ w2 /*64x16*/, float* __restrict__ gvec,
                                float* __restrict__ gmean) {
    const int img = blockIdx.x;
    __shared__ float mean[64], hid[16], g[64];
    if (threadIdx.x < 64) {
        float s = 0.f;
        for (int c = 0; c < chunks; ++c) s += gsum[((size_t)img * chunks + c) * 64 + threadIdx.x];
        mean[threadIdx.x] = s / (float)HW;
    }
    __syncthreads();
    if (threadIdx.x < 16) {
        float s = 0.f;
        for (int c = 0; c < 64; ++c) s += w1[threadIdx.x * 64 + c] * mean[c];
        hid[threadIdx.x] = fmaxf(s, 0.f);
    }
    __syncthreads();
    if (threadIdx.x < 64) {
        float s = 0.f;
        for (int k = 0; k < 16; ++k) s += w2[threadIdx.x * 16 + k] * hid[k];
        g[threadIdx.x] = 1.f / (1.f + expf(-s));
        gvec[img * 64 + threadIdx.x] = g[threadIdx.x];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int c = 0; c < 64; ++c) s += g[c];
        gmean[img] = s / 64.f;
    }
}

__global__ void asf_cmean_kernel(const uint4* __restrict__ a, long long npix_total, int HW,
                                 const float* __restrict__ gmean, float* __restrict__ m) {
    // 8 threads per pixel (one 16 B load each), shuffle-reduce
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long pix = t >> 3;
    const int cg = (int)(t & 7);
    float s = 0.f;
    if (pix < npix_total) {
        float f[8];
        unpack8(__ldg(a + pix * 8 + cg), f);
#pragma unroll
        for (int j = 0; j < 8; ++j) s += f[j];
    }
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    s += __shfl_xor_sync(0xffffffffu, s, 4);
    if (cg == 0 && pix < npix_total) m[pix] = s * (1.f / 64.f) + gmean[pix / HW];
}

struct AsfW {
    float sp3[9];     // spatial_wise.0.weight (1,1,3,3)
    float sp1;        // spatial_wise.2.weight (1,1,1,1)
    float att[4][64]; // attention_wise.0.weight (4,64,1,1)
};

__global__ void asf_apply_kernel(const uint4* __restrict__ a, const float* __restrict__ m,
                                 const float* __restrict__ gvec, int n_img, int H, int W, const AsfW wts,
                                 uint4* __restrict__ fuse /* [pix][256 ch] in place */) {
    // 8 threads per pixel: each owns 8 channels of `a` (attention logits) and then scales 32 channels of `fuse`
    __shared__ float s_att[4][64];  // thread-dependent indexing: shared memory, not the (serialising) constant bank
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_att[i >> 6][i & 63] = wts.att[i >> 6][i & 63];
    __syncthreads();
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long pix = t >> 3;
    const int cg = (int)(t & 7);
    const long long npix = (long long)n_img * H * W;
    const bool ok = pix < npix;
    float part[4] = {0.f, 0.f, 0.f, 0.f};
    if (ok) {
        const int w = (int)(pix % W);
        const int h = (int)((pix / W) % H);
        const int img = (int)(pix / ((long long)W * H));
        float conv = 0.f;
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
            for (int dx = -1; dx <= 1; ++dx) {
                const int y = h + dy, x = w + dx;
                if (y >= 0 && y < H && x >= 0 && x < W)
                    conv += wts.sp3[(dy + 1) * 3 + dx + 1] * __ldg(m + ((size_t)img * H + y) * W + x);
            }
        const float s = 1.f / (1.f + __expf(-(wts.sp1 * fmaxf(conv, 0.f))));
        float f[8];
        unpack8(__ldg(a + pix * 8 + cg), f);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float z = s + f[j] + __ldg(gvec + img * 64 + cg * 8 + j);
#pragma unroll
            for (int k = 0; k < 4; ++k) part[k] += s_att[k][cg * 8 + j] * z;
        }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        part[k] += __shfl_xor_sync(0xffffffffu, part[k], 1);
        part[k] += __shfl_xor_sync(0xffffffffu, part[k], 2);
        part[k] += __shfl_xor_sync(0xffffffffu, part[k], 4);
    }
    if (!ok) return;
    // thread cg scales channels [cg*32, cg*32+32) of the 256-channel fused map -> group cg/2
    const float sc = 1.f / (1.f + __expf(-part[cg >> 1]));
    uint4* fp = fuse + pix * 32 + cg * 4;
#pragma unroll
    for (int v = 0; v < 4; ++v) {
        float f[8];
        unpack8(fp[v], f);
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] *= sc;
        fp[v] = pack8(f);
    }
}

int launch_asf(const void* a, void* fuse, int n_img, int H, int W, const float* w1_dev, const float* w2_dev,
               const float* host_sp3, float host_sp1, const float* host_att, float* gsum, float* gvec, float* gmean,
               float* m, cudaStream_t st) {
    const int HW = H * W;
    dim3 g1(kAsfPoolChunks, n_img);                    // gsum: [n_img][kAsfPoolChunks][64] partial channel sums
    asf_pool_kernel<<<g1, 256, 0, st>>>(reinterpret_cast<const uint4*>(a), HW, gsum);
    asf_gate_kernel<<<n_img, 64, 0, st>>>(gsum, kAsfPoolChunks, HW, w1_dev, w2_dev, gvec, gmean);
    const long long npix = (long long)n_img * HW;
    const long long thr = npix * 8;
    asf_cmean_kernel<<<(unsigned)((thr + 255) / 256), 256, 0, st>>>(reinterpret_cast<const uint4*>(a), npix, HW, gmean,
                                                                    m);
    AsfW wts;
    for (int i = 0; i < 9; ++i) wts.sp3[i] = host_sp3[i];
    wts.sp1 = host_sp1;
    for (int k = 0; k < 4; ++k)
        for (int c = 0; c < 64; ++c) wts.att[k][c] = host_att[k * 64 + c];
    asf_apply_kernel<<<(unsigned)((thr + 255) / 256), 256, 0, st>>>(reinterpret_cast<const uint4*>(a), m, gvec, n_img, H,
                                                                    W, wts, reinterpret_cast<uint4*>(fuse));
    count_launch(4);
    return cudaGetLastError() != cudaSuccess;
}

// fp32 -> bf16 conversion helper for weight upload / debug
__global__ void op_to_f32_kernel(const op_t* __restrict__ in, float* __restrict__ out, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = op2f(in[i]);
}
int launch_op_to_f32(const void* in, float* out, long long n, cudaStream_t st) {
    op_to_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(reinterpret_cast<const op_t*>(in), out, n);
    return cudaGetLastError() != cudaSuccess;
}

}  // namespace ytk
