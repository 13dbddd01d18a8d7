// fp32 <-> split16 (fp16 hi + fp16 lo) conversions and the GEMM epilogue store shared by the SIMT and wgmma kernels.
#pragma once
#include "common.cuh"

namespace cotr {

// x ~= hi + lo with ~22 mantissa bits.  Both terms saturate at the fp16 range (cvt.rn.satfinite -> one
// F2FP.SATFINITE instruction), so the format represents |x| up to 131008 and clamps beyond (never inf / NaN); below
// 2^-3 the lo term is an fp16 subnormal, i.e. the absolute error floors at ~3e-8.
__device__ __forceinline__ uint32_t pack_f16x2_sat(float lo_elem, float hi_elem) {      // lo_elem -> bits [0,16)
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi_elem), "f"(lo_elem));
    return r;
}
__device__ __forceinline__ void split_f16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
    hi = pack_f16x2_sat(a, b);
    const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hi));
    lo = pack_f16x2_sat(a - hf.x, b - hf.y);
}
__device__ __forceinline__ void split_f16(float a, __half& hi, __half& lo) {
    const uint32_t h = pack_f16x2_sat(a, 0.f);
    hi = __ushort_as_half((unsigned short)(h & 0xFFFFu));
    const uint32_t l = pack_f16x2_sat(a - __half2float(hi), 0.f);
    lo = __ushort_as_half((unsigned short)(l & 0xFFFFu));
}
__device__ __forceinline__ float2 join_f16x2(uint32_t hi, uint32_t lo) {
    const float2 h = __half22float2(*reinterpret_cast<const __half2*>(&hi));
    const float2 l = __half22float2(*reinterpret_cast<const __half2*>(&lo));
    return make_float2(h.x + l.x, h.y + l.y);
}
__device__ __forceinline__ float join_f16(__half hi, __half lo) { return __half2float(hi) + __half2float(lo); }

// 8 consecutive elements (16 bytes per plane) -> 8 floats.
// Activations are read with ld.global.cg, never through the non-coherent path (__ldg / ld.global.nc): under
// programmatic dependent launch a kernel is resident while its predecessor still writes these buffers, so they are not
// read-only for the kernel's lifetime, which .nc requires - measured: an SM's L1 kept row statistics of the PREVIOUS
// forward across the launches in between and a .nc load after griddepcontrol.wait returned them.  Constants (weights, biases, gamma / beta, tables) keep __ldg.
__device__ __forceinline__ void load8_split(const CSplit16& t, size_t off, float (&v)[8]) {
    const uint4 h = __ldcg(reinterpret_cast<const uint4*>(t.hi + off));
    const uint4 l = __ldcg(reinterpret_cast<const uint4*>(t.lo + off));
    float2 f;
    f = join_f16x2(h.x, l.x); v[0] = f.x; v[1] = f.y;
    f = join_f16x2(h.y, l.y); v[2] = f.x; v[3] = f.y;
    f = join_f16x2(h.z, l.z); v[4] = f.x; v[5] = f.y;
    f = join_f16x2(h.w, l.w); v[6] = f.x; v[7] = f.y;
}
__device__ __forceinline__ void store8_split(const Split16& t, size_t off, const float* v) {
    uint4 h, l;
    split_f16x2(v[0], v[1], h.x, l.x);
    split_f16x2(v[2], v[3], h.y, l.y);
    split_f16x2(v[4], v[5], h.z, l.z);
    split_f16x2(v[6], v[7], h.w, l.w);
    *reinterpret_cast<uint4*>(t.hi + off) = h;
    *reinterpret_cast<uint4*>(t.lo + off) = l;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// out = LayerNorm(x) over 256 channels, eps 1e-5, biased variance.  One warp per row, 8 channels per lane.
__device__ __forceinline__ void load_vec8(const float* __restrict__ p, int lane, float (&v)[8]) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p + lane * 8)), b = __ldg(reinterpret_cast<const float4*>(p + lane * 8 + 4));
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

// v (8 channels per lane of one warp) <- LayerNorm over the 256 channels of the row
__device__ __forceinline__ void warp_layernorm256(float (&v)[8], const float* __restrict__ gamma, const float* __restrict__ beta, int lane) {
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) s += v[j];
    const float mean = warp_sum(s) * (1.f / kDModel);
    float sq = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) { v[j] -= mean; sq = fmaf(v[j], v[j], sq); }
    const float rstd = 1.f / sqrtf(warp_sum(sq) * (1.f / kDModel) + 1e-5f);
    float g[8], b[8];
    load_vec8(gamma, lane, g);
    load_vec8(beta, lane, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = v[j] * rstd * g[j] + b[j];
}

// Where column block [nb, nb+16) of output row `row` goes (GemmParams::remap / blk_map): returns true when the
// block is a transposed value projection, in which case `base` is the vt element offset of (column nb, this row)
// and consecutive columns are 512 elements apart; otherwise `base` is the row-major element offset.
__device__ __forceinline__ bool out_location(const GemmParams& p, int row, int nb, size_t& base) {
    int col = nb;
    if (p.remap) {
        const int m = p.blk_map[nb >> 8];
        if (m < 0 && p.kv_img != nullptr) { base = 0; return true; }      // attention operand image: store16 places it
        if (m < 0) {
            const int pair = row >> 9, key = row & (kTokens - 1);
            base = ((size_t)(pair * p.n_vt + (-m - 1)) * kDModel + (nb & 255)) * kTokens + key;
            return true;
        }
        col = m + (nb & 255);
    }
    base = (size_t)row * p.ldc + col;
    return false;
}

// Store 16 final values of columns [nb, nb+16) of `row` (split16 outputs need N % 16 == 0; the fp32 output is scalar).
__device__ __forceinline__ void store16(const GemmParams& p, int row, int nb, const float (&v)[16]) {
    if (p.out_f32) {
#pragma unroll
        for (int j = 0; j < 16; ++j)
            if (nb + j < p.N) p.out_f32[(size_t)row * p.ldc + nb + j] = v[j];
        return;
    }
    size_t base;
    if (p.remap && p.kv_img != nullptr && p.blk_map[nb >> 8] < 0) {
        // attention operand images (common.cuh): row = pair * 512 + key, columns nb .. nb+15 = head dims d0 .. d0+15 of
        // head (nb % 256) / 32.  Lanes hold consecutive keys.
        const int m = p.blk_map[nb >> 8];
        const bool is_key = m <= -1000;
        const int slot = is_key ? -1000 - m : -m - 1;
        const int pair = row >> 9, key = row & (kTokens - 1);
        const int c = nb & 255, head = c >> 5, d0 = c & 31;
        unsigned char* img = p.kv_img + ((size_t)(pair * p.n_vt + slot) * kHeads + head) * kAttnHeadImgBytes;
        if (is_key) {              // two groups of 8 head dims: one 16-byte piece per plane each (512-byte runs per warp)
            uint4 h0, l0, h1, l1;
            split_f16x2(v[0], v[1], h0.x, l0.x);   split_f16x2(v[2], v[3], h0.y, l0.y);
            split_f16x2(v[4], v[5], h0.z, l0.z);   split_f16x2(v[6], v[7], h0.w, l0.w);
            split_f16x2(v[8], v[9], h1.x, l1.x);   split_f16x2(v[10], v[11], h1.y, l1.y);
            split_f16x2(v[12], v[13], h1.z, l1.z); split_f16x2(v[14], v[15], h1.w, l1.w);
            unsigned char* d = img + (size_t)(d0 >> 3) * (kTokens * 16) + (size_t)key * 16;
            *reinterpret_cast<uint4*>(d) = h0;
            *reinterpret_cast<uint4*>(d + kTokens * 16) = h1;
            *reinterpret_cast<uint4*>(d + kAttnKPlaneBytes) = l0;
            *reinterpret_cast<uint4*>(d + kAttnKPlaneBytes + kTokens * 16) = l1;
        } else {                   // values: 8 consecutive keys of one head dim share a 16-byte piece
            __half* d = reinterpret_cast<__half*>(img + kAttnKImgBytes + (size_t)(key >> 3) * kAttnVGroupBytes + (size_t)d0 * 16) + (key & 7);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                __half h, l;
                split_f16(v[j], h, l);
                d[j * 8] = h;                        // next head dim: + 16 bytes
                d[j * 8 + 32 * 8] = l;               // lo rows follow the 32 hi rows of the key group
            }
        }
        return;
    }
    if (out_location(p, row, nb, base)) {
#pragma unroll
        for (int j = 0; j < 16; ++j) {       // lanes hold consecutive keys -> each store is a coalesced 64-byte run
            __half h, l;
            split_f16(v[j], h, l);
            p.vt.hi[base + (size_t)j * kTokens] = h;
            p.vt.lo[base + (size_t)j * kTokens] = l;
        }
    } else {
        store8_split(p.out, base, v);
        store8_split(p.out, base + 8, v + 8);
    }
}

}  // namespace cotr
