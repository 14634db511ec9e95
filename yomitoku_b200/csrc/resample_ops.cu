// Device-side input resize of the three RT-DETRv2 models: what the reference does per image on the host with Pillow
// (T.Resize(S) = Image.resize((S, S), BILINEAR) of the RGB page or table crop, then ToTensor) as two kernels over every
// model input of a call, reading u8 BGR pages that are already in HBM:
//
//   resample_first_kernel   first pass (horizontal, or vertical for a tall narrow input, see resample_math.h): one
//                           thread per (input, intermediate pixel), BGR -> RGB, u8 intermediate
//   resample_second_kernel  second pass: one thread per output pixel; writes either the engine's NHWC-64 op_t input
//                           (the bytes pack_input_kernel makes of ToTensor's fp32 tensor) or u8 RGB (op-level tests)
//
// The arithmetic lives in resample_math.h and is compiled for the host as well (oracle/resample_host.cpp), where the CPU
// tests pin it bit for bit against Pillow.  The coefficients are computed here on the host, once per call, in double as
// Pillow does; this file MUST be compiled with --fmad=false and -ffp-contract=off (yomitoku_b200/build.py).  The
// number of taps is not bounded: a 9000-pixel side going to 640 has 31.
#include <cstring>
#include <map>
#include <utility>

#include "gemm_tc.h"
#include "ptx.cuh"
#include "resample_ops.h"

namespace ytk {

static constexpr int kResampleThreads = 256, kResampleMaxBlocks = 1024;
static_assert(sizeof(ResamplePlan) == 64, "ResamplePlan is uploaded as a packed array");

static long long align16(long long v) { return (v + 15) / 16 * 16; }

int resample_prepare(const RtSrc* srcs, int n, int S, long long pages_bytes, const char* who, ResampleJob* job) {
    if (!srcs || n < 1 || n > 65535 || S < 1) {
        set_error("%s: %d sources of size %d (1..65535 sources, size >= 1)", who, n, S);
        return 1;
    }
    std::vector<ResamplePlan> plans(n);
    std::vector<int> coefs;
    std::map<std::pair<int, int>, long long> tables;  // (in, out) -> offset: equal axes share one table
    auto table = [&](int in) {
        auto it = tables.find({in, S});
        if (it != tables.end()) return it->second;
        const long long off = (long long)coefs.size();
        coefs.resize(off + (long long)S * (bilinear_ksize(in, S) + 2));
        bilinear_coeffs(in, S, coefs.data() + off);
        tables[{in, S}] = off;
        return off;
    };
    long long inter = 0;
    job->max_inter = 0;
    for (int i = 0; i < n; ++i) {
        const RtSrc& s = srcs[i];
        const bool ok = s.page_off >= 0 && s.H >= 1 && s.W >= 1 && s.page_off <= pages_bytes &&
                        (long long)s.H * s.W <= (pages_bytes - s.page_off) / 3 && s.x0 >= 0 && s.x0 < s.x1 &&
                        s.x1 <= s.W && s.y0 >= 0 && s.y0 < s.y1 && s.y1 <= s.H;
        if (!ok) {
            set_error("%s: source %d (page at %lld, %dx%d, rectangle x %d..%d y %d..%d) is empty or outside its page, "
                      "or its page overruns the %lld page bytes", who, i, s.page_off, s.H, s.W, s.x0, s.x1, s.y0, s.y1,
                      pages_bytes);
            return 1;
        }
        const int cw = s.x1 - s.x0, ch = s.y1 - s.y0;
        ResamplePlan& p = plans[i];
        p.src = s;
        p.kx = bilinear_ksize(cw, S);
        p.ky = bilinear_ksize(ch, S);
        p.cx_off = table(cw);
        p.cy_off = table(ch);
        p.inter_off = inter;  // relative to the intermediate block until the layout is known
        const long long px = resample_inter_pixels(cw, ch, S);
        inter += px * 3;
        if (px > job->max_inter) job->max_inter = px;
    }
    const long long plan_bytes = (long long)n * (long long)sizeof(ResamplePlan);
    job->coef_off = align16(plan_bytes);
    const long long inter_base = align16(job->coef_off + (long long)coefs.size() * 4);
    for (ResamplePlan& p : plans) p.inter_off += inter_base;
    job->n = n;
    job->S = S;
    job->bytes = inter_base + inter;
    job->host.assign((size_t)(job->coef_off + (long long)coefs.size() * 4), 0);
    memcpy(job->host.data(), plans.data(), (size_t)plan_bytes);
    memcpy(job->host.data() + job->coef_off, coefs.data(), coefs.size() * 4);
    return 0;
}

__global__ void __launch_bounds__(kResampleThreads) resample_first_kernel(const uint8_t* __restrict__ pages,
                                                                           const ResamplePlan* __restrict__ plans,
                                                                           const int* __restrict__ coefs, int S,
                                                                           uint8_t* __restrict__ scratch) {
    const ResamplePlan p = plans[blockIdx.y];
    const int cw = p.src.x1 - p.src.x0, ch = p.src.y1 - p.src.y0;
    const long long total = resample_inter_pixels(cw, ch, S);
    const int cols = resample_vertical_first(cw, ch, S) ? cw : S;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(idx / cols);
        resample_first(pages, p.src, coefs + p.cx_off, p.kx, coefs + p.cy_off, p.ky, S, r, (int)(idx - (long long)r * cols),
                       scratch + p.inter_off);
    }
}

template <bool kPack>
__global__ void __launch_bounds__(kResampleThreads) resample_second_kernel(const ResamplePlan* __restrict__ plans,
                                                                       const int* __restrict__ coefs, int S,
                                                                       const uint8_t* __restrict__ scratch,
                                                                       void* __restrict__ out) {
    const ResamplePlan p = plans[blockIdx.y];
    const long long total = (long long)S * S;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int oy = (int)(idx / S);
        uint8_t v[3];
        resample_second(scratch + p.inter_off, p.src.x1 - p.src.x0, p.src.y1 - p.src.y0, coefs + p.cx_off, p.kx,
                        coefs + p.cy_off, p.ky, S, oy, (int)(idx - (long long)oy * S), v);
        const long long pix = (long long)blockIdx.y * total + idx;
        if (kPack) {
            // pixel = 64 channels = 8 x uint4; the first holds R, G, B, the rest is zero
            uint4* d = reinterpret_cast<uint4*>(out) + pix * 8;
            d[0] = make_uint4(pack_op(unit_from_u8(v[0]), unit_from_u8(v[1])), pack_op(unit_from_u8(v[2]), 0.f), 0u, 0u);
#pragma unroll
            for (int g = 1; g < 8; ++g) d[g] = make_uint4(0u, 0u, 0u, 0u);
        } else {
            uint8_t* o = reinterpret_cast<uint8_t*>(out) + pix * 3;
            o[0] = v[0];
            o[1] = v[1];
            o[2] = v[2];
        }
    }
}

static unsigned blocks_for(long long work) {
    const long long b = (work + kResampleThreads - 1) / kResampleThreads;
    return (unsigned)(b < kResampleMaxBlocks ? (b < 1 ? 1 : b) : kResampleMaxBlocks);
}

int launch_resample(const uint8_t* pages, const ResampleJob& job, uint8_t* scratch, void* out, int pack,
                    cudaStream_t st) {
    cudaError_t err = cudaMemcpyAsync(scratch, job.host.data(), job.host.size(), cudaMemcpyHostToDevice, st);
    if (err != cudaSuccess) {
        set_error("resize: upload of the sources and coefficients failed: %s", cudaGetErrorString(err));
        return 1;
    }
    const ResamplePlan* plans = reinterpret_cast<const ResamplePlan*>(scratch);
    const int* coefs = reinterpret_cast<const int*>(scratch + job.coef_off);
    resample_first_kernel<<<dim3(blocks_for(job.max_inter), (unsigned)job.n), kResampleThreads, 0, st>>>(
        pages, plans, coefs, job.S, scratch);
    count_launch();
    if ((err = cudaGetLastError()) == cudaSuccess) {
        const dim3 grid(blocks_for((long long)job.S * job.S), (unsigned)job.n);
        if (pack)
            resample_second_kernel<true><<<grid, kResampleThreads, 0, st>>>(plans, coefs, job.S, scratch, out);
        else
            resample_second_kernel<false><<<grid, kResampleThreads, 0, st>>>(plans, coefs, job.S, scratch, out);
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
