// Image front end on the GPU: Pillow-exact 8-bit bicubic resampling + tiling + CLIP normalisation.
// Reference path: video_audio_demo.py:214-221 -> dynamic_preprocess (data_utils_video_audio_neg_patch.py:1214-1255,
// PIL Image.resize) -> process_images (mm_utils.py:30-43) -> CLIPImageProcessor (preprocessor_config.json constants).
//
// Integer work end to end, bit-exact by construction: the host computes Pillow's separable coefficient tables
// (double precision, rounded to 22-bit fixed point exactly as Resample.c does), the kernels do
// out = clip8((2^21 + sum p * k) >> 22) along one axis per pass (horizontal, then vertical, uint8 in between),
// and the last kernel cuts 448 x 448 tiles and maps every byte through a per-channel 256-entry bf16 table that holds
// the reference's rescale + normalise result.  HBM-bound byte streaming: the passes read each input byte ~ksize/scale
// times out of L1/L2, write each output byte once.
#include "common.h"
#include "ptx.cuh"

namespace vita {

constexpr int IMG_PRECISION_BITS = 32 - 8 - 2;

// One pass along `axis` of an interleaved [H, W, C] image.  Thread = one output pixel (all C channels).
// along: extent of the resampled axis in the input; other: extent of the untouched axis.
template <int C>
__global__ void __launch_bounds__(256)
image_resample_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int other, int out_size, long long in_stride_along,
                      long long in_stride_other, long long out_stride_along, long long out_stride_other,
                      const int* __restrict__ kk, const int* __restrict__ bounds, int ksize, int other_fast) {
    // thread index runs fastest over the axis that is contiguous in memory (x): coalesced stores in both passes
    const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const long long total = static_cast<long long>(other) * out_size;
    if (idx >= total) return;
    int o, p;
    if (other_fast) { p = static_cast<int>(idx % other); o = static_cast<int>(idx / other); }
    else            { o = static_cast<int>(idx % out_size); p = static_cast<int>(idx / out_size); }
    const int xmin = bounds[2 * o], xmax = bounds[2 * o + 1];
    const int* k = kk + static_cast<long long>(o) * ksize;
    int acc[C];
#pragma unroll
    for (int c = 0; c < C; ++c) acc[c] = 1 << (IMG_PRECISION_BITS - 1);
    const uint8_t* src = in + static_cast<long long>(xmin) * in_stride_along + static_cast<long long>(p) * in_stride_other;
    for (int x = 0; x < xmax; ++x) {
        const int w = __ldg(k + x);
#pragma unroll
        for (int c = 0; c < C; ++c) acc[c] += static_cast<int>(src[c]) * w;
        src += in_stride_along;
    }
    uint8_t* dst = out + static_cast<long long>(o) * out_stride_along + static_cast<long long>(p) * out_stride_other;
#pragma unroll
    for (int c = 0; c < C; ++c) {
        const int v = acc[c] >> IMG_PRECISION_BITS;     // arithmetic shift, as Pillow's clip8
        dst[c] = static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v));
    }
}

// img [gj*T, gi*T, 3] u8 -> out[tile0 + ty*gi + tx][c][y][x] = lut[c][img[ty*T + y][tx*T + x][c]] (bf16)
__global__ void __launch_bounds__(256)
image_tiles_lut_kernel(const uint8_t* __restrict__ img, const __nv_bfloat16* __restrict__ lut, __nv_bfloat16* __restrict__ out,
                       int gi, int gj, int T, int tile0) {
    __shared__ __nv_bfloat16 s_lut[3 * 256];
    for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) s_lut[i] = lut[i];
    __syncthreads();
    const long long n_pix = static_cast<long long>(gi) * gj * T * T;
    const int Wb = gi * T;
    for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < n_pix;
         idx += static_cast<long long>(gridDim.x) * blockDim.x) {
        // idx enumerates output pixels of one channel plane: x fastest inside a tile row -> coalesced bf16 stores
        const int x = static_cast<int>(idx % T);
        const int y = static_cast<int>((idx / T) % T);
        const int t = static_cast<int>(idx / (static_cast<long long>(T) * T));
        const int tx = t % gi, ty = t / gi;
        const uint8_t* px = img + (static_cast<long long>(ty * T + y) * Wb + tx * T + x) * 3;
        __nv_bfloat16* o = out + (static_cast<long long>(tile0 + t) * 3) * T * T + static_cast<long long>(y) * T + x;
#pragma unroll
        for (int c = 0; c < 3; ++c) o[static_cast<long long>(c) * T * T] = s_lut[c * 256 + px[c]];
    }
}

}  // namespace vita

using namespace vita;

extern "C" int vita_image_resample_u8(const uint8_t* in, uint8_t* out, int64_t H, int64_t W, int64_t C, int axis,
                                      int64_t out_size, const int32_t* kk, const int32_t* bounds, int64_t ksize,
                                      void* stream) {
    VITA_REQUIRE(in && out && kk && bounds, "image_resample: null pointer");
    VITA_REQUIRE(C == 3 || C == 1 || C == 4, "image_resample: 1, 3 or 4 interleaved channels");
    VITA_REQUIRE(axis == 0 || axis == 1, "image_resample: axis 0 (rows) or 1 (columns)");
    VITA_REQUIRE(H > 0 && W > 0 && out_size > 0 && ksize > 0, "image_resample: empty image");
    const int other = static_cast<int>(axis == 1 ? H : W);
    long long isa, iso, osa, oso;
    if (axis == 1) {   // horizontal: along = x, other = y; output [H, out_size, C]
        isa = C; iso = W * C; osa = C; oso = out_size * C;
    } else {           // vertical: along = y, other = x; output [out_size, W, C]
        isa = W * C; iso = C; osa = W * C; oso = C;
    }
    const long long total = static_cast<long long>(other) * out_size;
    const unsigned blocks = static_cast<unsigned>((total + 255) / 256);
    auto st = static_cast<cudaStream_t>(stream);
    const int other_fast = axis == 0 ? 1 : 0;
#define VITA_IMG_LAUNCH(CC)                                                                                           \
    image_resample_kernel<CC><<<blocks, 256, 0, st>>>(in, out, other, static_cast<int>(out_size), isa, iso, osa, oso, \
                                                      kk, bounds, static_cast<int>(ksize), other_fast)
    if (C == 3) VITA_IMG_LAUNCH(3);
    else if (C == 1) VITA_IMG_LAUNCH(1);
    else VITA_IMG_LAUNCH(4);
#undef VITA_IMG_LAUNCH
    return check_launch("image_resample_kernel");
}

extern "C" int vita_image_tiles_lut(const uint8_t* img, const void* lut, void* out, int64_t gi, int64_t gj, int64_t T,
                                    int64_t tile0, void* stream) {
    VITA_REQUIRE(img && lut && out, "image_tiles_lut: null pointer");
    VITA_REQUIRE(gi > 0 && gj > 0 && T > 0 && tile0 >= 0, "image_tiles_lut: bad geometry");
    const long long n_pix = gi * gj * T * T;
    long long blocks = (n_pix + 255) / 256;
    const long long cap = static_cast<long long>(num_sms() > 0 ? num_sms() : 132) * 16;
    if (blocks > cap) blocks = cap;
    image_tiles_lut_kernel<<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        img, BF16C(lut), static_cast<__nv_bfloat16*>(out), static_cast<int>(gi), static_cast<int>(gj),
        static_cast<int>(T), static_cast<int>(tile0));
    return check_launch("image_tiles_lut_kernel");
}
