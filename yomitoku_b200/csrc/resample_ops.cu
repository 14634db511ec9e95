// Device resize of u8 BGR pages that are already in HBM: what the reference does per image on the host with Pillow,
// Image.resize((w, h), f) of the RGB page or crop, as two kernels over every source of a call:
//   * the RT-DETRv2 models' T.Resize(S) = BILINEAR to S x S, then ToTensor (layout parser, table structure recognizer,
//     cell detector);
//   * the searchable PDF's page images: LANCZOS to each page's own size, planar RGB for the JPEG encoder.
//
//   resample_first_kernel   first pass of the sources that need two (horizontal, or vertical for a tall narrow input,
//                           see resample_math.h): one thread per (source, intermediate pixel), BGR -> RGB, u8
//                           intermediate.  Not launched when no source needs it.
//   resample_second_kernel  one thread per output pixel: the second pass, the only pass of a source with one unchanged
//                           axis, or the BGR -> RGB copy of an unchanged source; writes one of three layouts
//                           (ResampleOut): the engine's NHWC-64 op_t input (the bytes pack_input_kernel makes of
//                           ToTensor's fp32 tensor), u8 RGB (op-level tests) or planar u8 RGB (JPEG encoder input)
//
// The arithmetic lives in resample_math.h and is compiled for the host as well (oracle/resample_host.cpp), where the CPU
// tests pin it bit for bit against Pillow.  The coefficients are computed here on the host, once per call, in double as
// Pillow does; this file MUST be compiled with --fmad=false and -ffp-contract=off (yomitoku_b200/build.py).  The
// number of taps is not bounded: a 9000-pixel side going to 640 has 31 (BILINEAR).
#include <cstring>
#include <map>
#include <utility>

#include "gemm_tc.h"
#include "ptx.cuh"
#include "resample_ops.h"

namespace ytk {

static constexpr int kResampleThreads = 256, kResampleMaxBlocks = 1024;
static_assert(sizeof(ResamplePlan) == 96, "ResamplePlan is uploaded as a packed array");

static long long align16(long long v) { return (v + 15) / 16 * 16; }

std::vector<ResampleSrc> square_sources(const RtSrc* srcs, int n, int S, long long pixel_bytes) {
    std::vector<ResampleSrc> out;
    if (!srcs || n < 1 || n > 65535) return out;
    out.resize(n);
    for (int i = 0; i < n; ++i) out[i] = ResampleSrc{srcs[i], S, S, (long long)i * S * S * pixel_bytes};
    return out;
}

int resample_prepare(const ResampleSrc* srcs, int n, int filter, long long pages_bytes, const char* who,
                     ResampleJob* job) {
    if (!srcs || n < 1 || n > 65535) {
        set_error("%s: %d sources (1..65535)", who, n);
        return 1;
    }
    if (!resample_filter_known(filter)) {
        set_error("%s: unknown filter %d (1 = LANCZOS, 2 = BILINEAR)", who, filter);
        return 1;
    }
    std::vector<ResamplePlan> plans(n);
    std::vector<int> coefs;
    std::map<std::pair<int, int>, long long> tables;  // (in, out) -> offset: equal axes share one table
    auto table = [&](int in, int out) {
        auto it = tables.find({in, out});
        if (it != tables.end()) return it->second;
        const long long off = (long long)coefs.size();
        coefs.resize(off + (long long)out * (resample_ksize(in, out, filter) + 2));
        resample_coeffs(in, out, filter, coefs.data() + off);
        tables[{in, out}] = off;
        return off;
    };
    long long inter = 0;
    job->max_inter = 0;
    job->max_out = 0;
    for (int i = 0; i < n; ++i) {
        const RtSrc& s = srcs[i].src;
        const bool ok = s.page_off >= 0 && s.H >= 1 && s.W >= 1 && s.page_off <= pages_bytes &&
                        (long long)s.H * s.W <= (pages_bytes - s.page_off) / 3 && s.x0 >= 0 && s.x0 < s.x1 &&
                        s.x1 <= s.W && s.y0 >= 0 && s.y0 < s.y1 && s.y1 <= s.H;
        if (!ok) {
            set_error("%s: source %d (page at %lld, %dx%d, rectangle x %d..%d y %d..%d) is empty or outside its page, "
                      "or its page overruns the %lld page bytes", who, i, s.page_off, s.H, s.W, s.x0, s.x1, s.y0, s.y1,
                      pages_bytes);
            return 1;
        }
        const int ow = srcs[i].out_w, oh = srcs[i].out_h;
        if (ow < 1 || oh < 1) {
            set_error("%s: source %d: output size %dx%d (width and height >= 1)", who, i, ow, oh);
            return 1;
        }
        const int cw = s.x1 - s.x0, ch = s.y1 - s.y0;
        ResamplePlan& p = plans[i];
        p.src = s;
        p.out_off = srcs[i].out_off;
        p.out_w = ow;
        p.out_h = oh;
        p.passes = resample_passes(cw, ch, ow, oh);
        p.icols = resample_inter_cols(cw, ow, p.passes);
        p.kx = resample_ksize(cw, ow, filter);
        p.ky = resample_ksize(ch, oh, filter);
        p.cx_off = (p.passes & kPassH) ? table(cw, ow) : 0;
        p.cy_off = (p.passes & kPassV) ? table(ch, oh) : 0;
        p.inter_off = inter;  // relative to the intermediate block until the layout is known
        const long long px = resample_inter_pixels(cw, ch, ow, oh, p.passes);
        inter += px * 3;
        if (px > job->max_inter) job->max_inter = px;
        if ((long long)ow * oh > job->max_out) job->max_out = (long long)ow * oh;
    }
    const long long plan_bytes = (long long)n * (long long)sizeof(ResamplePlan);
    job->coef_off = align16(plan_bytes);
    const long long inter_base = align16(job->coef_off + (long long)coefs.size() * 4);
    for (ResamplePlan& p : plans) p.inter_off += inter_base;
    job->n = n;
    job->bytes = inter_base + inter;
    job->host.assign((size_t)(job->coef_off + (long long)coefs.size() * 4), 0);
    memcpy(job->host.data(), plans.data(), (size_t)plan_bytes);
    memcpy(job->host.data() + job->coef_off, coefs.data(), coefs.size() * 4);
    return 0;
}

static __device__ __forceinline__ const uint8_t* crop_of(const uint8_t* pages, const RtSrc& s) {
    return pages + s.page_off + ((long long)s.y0 * s.W + s.x0) * 3;
}

__global__ void __launch_bounds__(kResampleThreads) resample_first_kernel(const uint8_t* __restrict__ pages,
                                                                           const ResamplePlan* __restrict__ plans,
                                                                           const int* __restrict__ coefs,
                                                                           uint8_t* __restrict__ scratch) {
    const ResamplePlan p = plans[blockIdx.y];
    const long long total = resample_inter_pixels(p.src.x1 - p.src.x0, p.src.y1 - p.src.y0, p.out_w, p.out_h, p.passes);
    const uint8_t* crop = crop_of(pages, p.src);
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(idx / p.icols);
        resample_first(crop, (long long)p.src.W * 3, p.passes, coefs + p.cx_off, p.kx, coefs + p.cy_off, p.ky, p.icols,
                       r, (int)(idx - (long long)r * p.icols), scratch + p.inter_off);
    }
}

template <int kLayout>
__global__ void __launch_bounds__(kResampleThreads) resample_second_kernel(const uint8_t* __restrict__ pages,
                                                                       const ResamplePlan* __restrict__ plans,
                                                                       const int* __restrict__ coefs,
                                                                       const uint8_t* __restrict__ scratch,
                                                                       uint8_t* __restrict__ out) {
    const ResamplePlan p = plans[blockIdx.y];
    const long long total = (long long)p.out_w * p.out_h;
    const uint8_t* crop = crop_of(pages, p.src);
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int oy = (int)(idx / p.out_w);
        uint8_t v[3];
        resample_second(crop, (long long)p.src.W * 3, scratch + p.inter_off, p.icols, p.passes, coefs + p.cx_off, p.kx,
                        coefs + p.cy_off, p.ky, oy, (int)(idx - (long long)oy * p.out_w), v);
        if (kLayout == kOutEngine) {
            // pixel = 64 channels = 8 x uint4; the first holds R, G, B, the rest is zero
            uint4* d = reinterpret_cast<uint4*>(out + p.out_off) + idx * 8;
            d[0] = make_uint4(pack_op(unit_from_u8(v[0]), unit_from_u8(v[1])), pack_op(unit_from_u8(v[2]), 0.f), 0u, 0u);
#pragma unroll
            for (int g = 1; g < 8; ++g) d[g] = make_uint4(0u, 0u, 0u, 0u);
        } else if (kLayout == kOutRGB) {
            uint8_t* o = out + p.out_off + idx * 3;
            o[0] = v[0];
            o[1] = v[1];
            o[2] = v[2];
        } else {
            uint8_t* o = out + p.out_off + idx;
            o[0] = v[0];
            o[total] = v[1];
            o[2 * total] = v[2];
        }
    }
}

static unsigned blocks_for(long long work) {
    const long long b = (work + kResampleThreads - 1) / kResampleThreads;
    return (unsigned)(b < kResampleMaxBlocks ? (b < 1 ? 1 : b) : kResampleMaxBlocks);
}

int launch_resample(const uint8_t* pages, const ResampleJob& job, uint8_t* scratch, void* out, ResampleOut layout,
                    cudaStream_t st) {
    cudaError_t err = cudaMemcpyAsync(scratch, job.host.data(), job.host.size(), cudaMemcpyHostToDevice, st);
    if (err != cudaSuccess) {
        set_error("resize: upload of the sources and coefficients failed: %s", cudaGetErrorString(err));
        return 1;
    }
    const ResamplePlan* plans = reinterpret_cast<const ResamplePlan*>(scratch);
    const int* coefs = reinterpret_cast<const int*>(scratch + job.coef_off);
    if (job.max_inter > 0) {
        resample_first_kernel<<<dim3(blocks_for(job.max_inter), (unsigned)job.n), kResampleThreads, 0, st>>>(
            pages, plans, coefs, scratch);
        count_launch();
        err = cudaGetLastError();
    }
    if (err == cudaSuccess) {
        const dim3 grid(blocks_for(job.max_out), (unsigned)job.n);
        uint8_t* o = static_cast<uint8_t*>(out);
        if (layout == kOutEngine)
            resample_second_kernel<kOutEngine><<<grid, kResampleThreads, 0, st>>>(pages, plans, coefs, scratch, o);
        else if (layout == kOutRGB)
            resample_second_kernel<kOutRGB><<<grid, kResampleThreads, 0, st>>>(pages, plans, coefs, scratch, o);
        else
            resample_second_kernel<kOutPlanar><<<grid, kResampleThreads, 0, st>>>(pages, plans, coefs, scratch, o);
        count_launch();
        err = cudaGetLastError();
    }
    if (err != cudaSuccess) {
        set_error("resize: kernel launch failed: %s", cudaGetErrorString(err));
        return 1;
    }
    return 0;
}

}  // namespace ytk
