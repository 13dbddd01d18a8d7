// Row/element addressing of the GEMM A operand (implicit im2col for the backbone convolutions).
// Shared by the fp32 SIMT GEMM and the wgmma GEMM so both see exactly the same operand.
#pragma once
#include "split16.cuh"

namespace cotr {

struct ARow {
    size_t off;          // element offset of the row start (row-major / token gather) or of the image (convolutions)
    int ih0, iw0;        // convolutions: input coordinate of tap (0,0)
    bool valid;
};

__device__ __forceinline__ ARow decode_a_row(const GemmParams& p, int m) {
    ARow r;
    r.valid = m < p.M;
    r.off = 0;
    r.ih0 = 0;
    r.iw0 = 0;
    if (!r.valid) return r;
    if (p.a_mode == A_ROWMAJOR) {
        r.off = (size_t)m * p.lda;
    } else if (p.a_mode == A_TOKENS) {
        // backbone.py:85 concatenates the two halves along W; transformer.py:50 flattens (i, j) -> i*32 + j
        const int pair = m >> 9, t = m & 511, i = t >> 5, j = t & 31;
        const int row = (p.a_pairs[2 * pair + (j >> 4)] * 16 + i) * 16 + (j & 15);
        r.off = (size_t)row * p.lda;
    } else {
        const int ohw = p.OH * p.OW;
        int n, oh, ow;
        if (((ohw & (ohw - 1)) | (p.OW & (p.OW - 1))) == 0) {      // every feature map of this network: powers of two
            const int s_img = 31 - __clz(ohw), s_row = 31 - __clz(p.OW);
            n = m >> s_img;
            const int rem = m & (ohw - 1);
            oh = rem >> s_row;
            ow = rem & (p.OW - 1);
        } else {
            n = m / ohw;
            const int rem = m - n * ohw;
            oh = rem / p.OW;
            ow = rem - oh * p.OW;
        }
        r.ih0 = oh * p.stride - p.pad;
        r.iw0 = ow * p.stride - p.pad;
        if (p.a_mode == A_CONV_NHWC) {
            r.off = (size_t)n * p.H * p.W * p.C;
        } else {  // A_STEM_NHWC4: pixel (2 oh, 2 ow) of the bordered canvas of image n = tap (0,0) of this output pixel
            r.off = (size_t)n * kStemCanvasElems + ((size_t)(2 * oh) * kStemCanvasPitch + 2 * ow) * 4;
        }
    }
    return r;
}

// Element offset of (row, k) for the split16 modes with K % 8 == 0 (and C % 8 == 0): k..k+7 are contiguous.
// Returns false for rows outside the matrix and for taps in the convolution padding.
__device__ __forceinline__ bool a_offset8(const GemmParams& p, const ARow& r, int k, size_t& off) {
    if (!r.valid || k >= p.K) return false;
    if (p.a_mode == A_CONV_NHWC) {
        const int tap = k / p.C;
        const int c = k - tap * p.C;
        const int kh = tap / p.KW;
        const int kw = tap - kh * p.KW;
        const int ih = r.ih0 + kh, iw = r.iw0 + kw;
        if (ih < 0 || ih >= p.H || iw < 0 || iw >= p.W) return false;
        off = r.off + ((size_t)ih * p.W + iw) * p.C + c;
        return true;
    }
    if (p.a_mode == A_STEM_NHWC4) {      // k = kh * 32 + (pixel slot * 4 + channel): 32 contiguous halves per filter row
        off = r.off + (size_t)(k >> 5) * (kStemCanvasPitch * 4) + (k & 31);
        return true;
    }
    off = r.off + k;
    return true;
}

}  // namespace cotr
