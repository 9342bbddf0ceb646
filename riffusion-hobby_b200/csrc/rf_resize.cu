// Bicubic resize of uint8 images, bit-exact with Pillow's Image.resize(size, Image.BICUBIC).
//
// Pillow (libImaging/Resample.c) resizes in two separable passes with 8-bit storage in between: the horizontal pass
// first, then the vertical one, each skipped when its extent does not change.  The filter taps are computed in fp64
// (precompute_coeffs: support 2 * max(in/out, 1), cubic a = -0.5, taps normalised by their sum) and rounded to int32
// with 22 fractional bits (normalize_coeffs_8bpc, round half away from zero); each output channel is
// clip8((1 << 21) + sum u8 * tap) = clamp(acc >> 22, 0, 255).  The tables are built here on the host exactly that way;
// the device passes are integer multiply-adds only, so the result does not depend on the order of the sum.
#include <cuda_fp16.h>

#include <cmath>
#include <cstdint>
#include <vector>

#include "rf_common.h"

namespace {

constexpr int kPrecisionBits = 22;          // 32 - 8 - 2
constexpr double kCubicA = -0.5;

double bicubic(double x) {
    if (x < 0.0) x = -x;
    if (x < 1.0) return ((kCubicA + 2.0) * x - (kCubicA + 3.0)) * x * x + 1;
    if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * kCubicA;
    return 0.0;
}

int taps_for(int in_size, int out_size) {
    const double filterscale = std::max(static_cast<double>(in_size) / out_size, 1.0);
    return static_cast<int>(std::ceil(2.0 * filterscale)) * 2 + 1;
}

// dst: int32[out_size][2 + taps] = (first input index, number of taps used, taps...), unused taps 0
void build_table(int in_size, int out_size, int32_t* dst) {
    const double scale = static_cast<double>(in_size) / out_size;
    const double filterscale = std::max(scale, 1.0);
    const double support = 2.0 * filterscale;
    const double ss = 1.0 / filterscale;
    const int taps = taps_for(in_size, out_size);
    std::vector<double> k(taps);
    for (int xx = 0; xx < out_size; ++xx) {
        const double center = (xx + 0.5) * scale;
        int xmin = static_cast<int>(center - support + 0.5);
        if (xmin < 0) xmin = 0;
        int xmax = static_cast<int>(center + support + 0.5);
        if (xmax > in_size) xmax = in_size;
        xmax -= xmin;
        double ww = 0.0;
        for (int x = 0; x < xmax; ++x) {
            k[x] = bicubic((x + xmin - center + 0.5) * ss);
            ww += k[x];
        }
        int32_t* row = dst + static_cast<size_t>(xx) * (2 + taps);
        row[0] = xmin;
        row[1] = xmax;
        for (int x = 0; x < taps; ++x) {
            double v = x < xmax ? k[x] : 0.0;
            if (x < xmax && ww != 0.0) v /= ww;
            row[2 + x] = v < 0 ? static_cast<int32_t>(-0.5 + v * (1 << kPrecisionBits))
                               : static_cast<int32_t>(0.5 + v * (1 << kPrecisionBits));
        }
    }
}

size_t align256(size_t n) { return (n + 255) & ~static_cast<size_t>(255); }

struct Layout {
    bool need_h, need_v;
    int taps_h, taps_v;
    size_t off_v, off_tmp, total, table_bytes;
};

Layout layout(int B, int in_h, int in_w, int channels, int out_h, int out_w) {
    Layout L{};
    L.need_h = out_w != in_w;
    L.need_v = out_h != in_h;
    L.taps_h = taps_for(in_w, out_w);
    L.taps_v = taps_for(in_h, out_h);
    L.off_v = static_cast<size_t>(out_w) * (2 + L.taps_h) * sizeof(int32_t);
    L.table_bytes = L.off_v + static_cast<size_t>(out_h) * (2 + L.taps_v) * sizeof(int32_t);
    L.off_tmp = align256(L.table_bytes);
    L.total = L.off_tmp + ((L.need_h && L.need_v) ? static_cast<size_t>(B) * in_h * out_w * channels : 0);
    return L;
}

// One output pixel (all channels) per thread.  VERT = false: in [B][H][in_w][C] -> out [B][H][out_w][C], taps along x;
// VERT = true: in [B][in_h][W][C] -> out [B][out_h][W][C], taps along y.  f16 (optional): [B][C][oh][ow] with
// 2 * (u8 / 255) - 1 in fp32, the arithmetic of riffusion_pipeline.preprocess_image.
template <bool VERT>
__global__ void __launch_bounds__(256) k_resize_bicubic_u8(const uint8_t* __restrict__ in, int B, int in_h, int in_w,
                                                            int C, int oh, int ow, const int32_t* __restrict__ tab,
                                                            int taps, uint8_t* __restrict__ out,
                                                            __half* __restrict__ f16) {
    const size_t n = static_cast<size_t>(B) * oh * ow;
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
         i += static_cast<size_t>(gridDim.x) * blockDim.x) {
        const int x = static_cast<int>(i % ow);
        const int y = static_cast<int>((i / ow) % oh);
        const int b = static_cast<int>(i / (static_cast<size_t>(ow) * oh));
        const int32_t* t = tab + static_cast<size_t>(VERT ? y : x) * (2 + taps);
        const int lo = __ldg(t), cnt = __ldg(t + 1);
        int acc[4] = {1 << (kPrecisionBits - 1), 1 << (kPrecisionBits - 1), 1 << (kPrecisionBits - 1),
                      1 << (kPrecisionBits - 1)};
        for (int j = 0; j < cnt; ++j) {
            const int w = __ldg(t + 2 + j);
            const uint8_t* p = VERT ? in + ((static_cast<size_t>(b) * in_h + lo + j) * in_w + x) * C
                                    : in + ((static_cast<size_t>(b) * in_h + y) * in_w + lo + j) * C;
#pragma unroll
            for (int c = 0; c < 4; ++c)
                if (c < C) acc[c] += static_cast<int>(p[c]) * w;
        }
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            if (c >= C) break;
            const int a = acc[c];
            const uint8_t v = a >= (1 << kPrecisionBits << 8) ? 255 : a <= 0 ? 0 : static_cast<uint8_t>(a >> kPrecisionBits);
            out[i * C + c] = v;
            if (f16) {
                const float u = __fdiv_rn(static_cast<float>(v), 255.0f);
                f16[((static_cast<size_t>(b) * C + c) * oh + y) * ow + x] = __float2half_rn(__fsub_rn(__fmul_rn(2.0f, u), 1.0f));
            }
        }
    }
}

bool bad_sizes(int in_size, int out_size) { return in_size <= 0 || out_size <= 0 || in_size > (1 << 20) || out_size > (1 << 20); }

}  // namespace

extern "C" int rf_resize_bicubic_taps(int in_size, int out_size) {
    if (bad_sizes(in_size, out_size)) {
        rf_fail(RF_ERR_INVALID, "rf_resize_bicubic_taps: bad size");
        return -1;
    }
    return taps_for(in_size, out_size);
}

extern "C" int rf_resize_bicubic_table(int in_size, int out_size, int32_t* dst, size_t bytes) {
    if (bad_sizes(in_size, out_size) || !dst) return rf_fail(RF_ERR_INVALID, "rf_resize_bicubic_table: bad argument");
    if (bytes != static_cast<size_t>(out_size) * (2 + taps_for(in_size, out_size)) * sizeof(int32_t))
        return rf_fail(RF_ERR_INVALID, "rf_resize_bicubic_table: bytes does not match out_size * (2 + taps) int32");
    build_table(in_size, out_size, dst);
    return RF_OK;
}

extern "C" size_t rf_resize_bicubic_workspace_bytes(int B, int in_h, int in_w, int channels, int out_h, int out_w) {
    if (B <= 0 || channels <= 0 || bad_sizes(in_h, out_h) || bad_sizes(in_w, out_w)) return 0;
    return layout(B, in_h, in_w, channels, out_h, out_w).total;
}

extern "C" int rf_resize_bicubic_u8(const uint8_t* d_in, int B, int in_h, int in_w, int channels, int out_h, int out_w,
                                    uint8_t* d_out, void* d_out_f16, void* d_workspace, size_t workspace_bytes,
                                    void* stream) {
    if (!d_in || !d_out || !d_workspace || B <= 0 || channels < 1 || channels > 4 || bad_sizes(in_h, out_h) ||
        bad_sizes(in_w, out_w))
        return rf_fail(RF_ERR_INVALID, "rf_resize_bicubic_u8: bad argument");
    const Layout L = layout(B, in_h, in_w, channels, out_h, out_w);
    if (workspace_bytes < L.total) return rf_fail(RF_ERR_INVALID, "rf_resize_bicubic_u8: workspace too small");
    std::vector<int32_t> host(L.table_bytes / sizeof(int32_t));
    build_table(in_w, out_w, host.data());
    build_table(in_h, out_h, host.data() + L.off_v / sizeof(int32_t));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    uint8_t* ws = static_cast<uint8_t*>(d_workspace);
    // pageable source: the call returns once `host` has been staged, so it may be freed on return
    RF_CUDA_TRY(cudaMemcpyAsync(ws, host.data(), L.table_bytes, cudaMemcpyHostToDevice, st));
    const int32_t* tab_h = reinterpret_cast<const int32_t*>(ws);
    const int32_t* tab_v = reinterpret_cast<const int32_t*>(ws + L.off_v);
    __half* f16 = static_cast<__half*>(d_out_f16);
    const unsigned cap = 8u * rf_num_sms();
    auto grid = [cap](size_t n) { return static_cast<unsigned>(std::min<size_t>((n + 255) / 256, cap)); };
    if (L.need_h) {
        // horizontal first (Pillow's order); straight into the output when there is no vertical pass
        uint8_t* dst = L.need_v ? ws + L.off_tmp : d_out;
        const size_t n = static_cast<size_t>(B) * in_h * out_w;
        k_resize_bicubic_u8<false><<<grid(n), 256, 0, st>>>(d_in, B, in_h, in_w, channels, in_h, out_w, tab_h, L.taps_h,
                                                           dst, L.need_v ? nullptr : f16);
        RF_CUDA_LAUNCH_CHECK("k_resize_bicubic_u8<h>");
        if (!L.need_v) return RF_OK;
        d_in = dst;
    }
    // the vertical pass; with equal heights its taps are the identity (bicubic(0) = 1, bicubic(+-1, +-2) = 0), which is
    // Pillow's plain copy
    const size_t n = static_cast<size_t>(B) * out_h * out_w;
    k_resize_bicubic_u8<true><<<grid(n), 256, 0, st>>>(d_in, B, in_h, out_w, channels, out_h, out_w, tab_v, L.taps_v,
                                                      d_out, f16);
    RF_CUDA_LAUNCH_CHECK("k_resize_bicubic_u8<v>");
    return RF_OK;
}
