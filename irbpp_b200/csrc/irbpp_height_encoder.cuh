// irbpp_height_encoder.cuh -- DQNBPP's heightEncoder (model.py:258-264, the same nn.Sequential at both network
// levels) on its own, and its backward pass, for irbpp_height_encoder_forward / irbpp_height_encoder_backward:
//   conv1 1 -> 16, k4, stride 2, pad 1 (32 -> 16), conv2 16 -> 32, k4, stride 2, pad 1 (16 -> 8),
//   conv3 32 -> 4, k3, stride 1, pad 1 (8 -> 8), each followed by LeakyReLU; 256 features flattened (C, H, W).
//
// Forward: one CTA per sample runs ac_height_encoder (irbpp_actor.cuh), the convolutions the act kernels of both
// levels run, on the sample's heightmap.
// Backward: one CTA per sample recomputes c1, c2 and the map with that same function (nothing is kept between the two
// calls), then, with leaky'(x) = 1 where the layer's output is > 0 and the slope elsewhere (torch's
// leaky_relu_backward tests the input > 0, the same set for a slope >= 0):
//   dpre3 = d_map * leaky'(map);
//   dW3, db3 from dpre3 and c2;  dpre2 = (conv3^T dpre3) * leaky'(c2);
//   dW2, db2 from dpre2 and c1;  dpre1 = (conv2^T dpre2, stride 2) * leaky'(c1);
//   dW1, db1 from dpre1 and the heightmap.
// No gradient is taken for the heightmap (an observation).  Every sum runs in a fixed order: each of a sample's
// HE_GRADS weight and bias gradients is a sum over output positions in row-major order, stored as the sample's
// partial in the scratch; irbpp_height_encoder_reduce_kernel then sums the partials over the samples in groups of
// HE_GROUP consecutive samples, pass after pass, in sample order.  No atomics: the results depend on B only, not on
// the grid, and two calls give bit-identical results.
#pragma once
#include <stdint.h>

#include "irbpp_actor.cuh"

namespace irbpp {

// the conv fields ac_height_encoder reads (include/irbpp.h irbpp_height_encoder_weights)
struct HeightEncoderWeights {
    const float *conv1_w, *conv1_b, *conv2_w, *conv2_b, *conv3_w, *conv3_b;
    float slope;
};

// the gradients of those tensors (include/irbpp.h irbpp_height_encoder_grads)
struct HeightEncoderGrads {
    float *conv1_w, *conv1_b, *conv2_w, *conv2_b, *conv3_w, *conv3_b;
};

// one sample's gradients, in this order: conv1 w [16][1][4][4], b [16]; conv2 w [32][16][4][4], b [32];
// conv3 w [4][32][3][3], b [4]
constexpr int HE_W1 = 0, HE_B1 = HE_W1 + 16 * 16, HE_W2 = HE_B1 + 16, HE_B2 = HE_W2 + 32 * 16 * 16, HE_W3 = HE_B2 + 32,
              HE_B3 = HE_W3 + 4 * 32 * 9, HE_GRADS = HE_B3 + 4;
static_assert(HE_GRADS == 9652, "the six gradient tensors of the height encoder");
constexpr int HE_GROUP = 16;          // samples summed per pass of the reduction
constexpr int HE_LD2 = 65;            // row stride of dpre2 [32][8 x 8] in shared memory (conflict-free columns)

struct HeightEncoderParams {
    HeightEncoderWeights w;
    const float* hm; int64_t hm_stride;       // sample b's 32 x 32 heightmap at hm + b * hm_stride
    int32_t B;
    float* map;                               // forward: [B][256]
    const float* d_map;                       // backward: [B][256]
    float* part;                              // backward: [B][HE_GRADS] per-sample gradients (scratch)
};

__host__ __device__ inline int64_t height_encoder_scratch_bytes(int64_t B) { return actor_align(B * HE_GRADS * 4); }

// the CTA's copy of sample b's heightmap (the barrier is in ac_height_encoder)
__device__ __forceinline__ void he_load(const HeightEncoderParams& P, float* hm) {
    const float* src = P.hm + (int64_t)blockIdx.x * P.hm_stride;
    for (int i = threadIdx.x; i < AC_HM * AC_HM; i += AC_THREADS) hm[i] = src[i];
}

__global__ void __launch_bounds__(AC_THREADS) irbpp_height_encoder_kernel(const HeightEncoderParams P) {
    __shared__ __align__(16) float hm[AC_HM * AC_HM];          // [1][32][32]
    __shared__ __align__(16) float c1[16 * 16 * 16];            // [16][16][16]
    __shared__ __align__(16) float c2[32 * 8 * 8];              // [32][8][8]
    he_load(P, hm);
    ac_height_encoder(P.w, hm, c1, c2, P.map + (int64_t)blockIdx.x * 256);
}

__global__ void __launch_bounds__(AC_THREADS) irbpp_height_encoder_backward_kernel(const HeightEncoderParams P) {
    __shared__ __align__(16) float hm[AC_HM * AC_HM];          // [1][32][32]
    __shared__ __align__(16) float c1[16 * 16 * 16];            // [16][16][16] c1, then dpre1
    __shared__ __align__(16) float c2[32 * 8 * 8];              // [32][8][8]
    __shared__ __align__(16) float d3[256];                     // the map, then dpre3
    __shared__ __align__(16) float d2[32 * HE_LD2];             // dpre2 [32][65]
    const int tid = threadIdx.x, b = blockIdx.x;
    const float slope = P.w.slope;
    const HeightEncoderWeights& w = P.w;
    float* part = P.part + (int64_t)b * HE_GRADS;
    he_load(P, hm);
    ac_height_encoder(w, hm, c1, c2, d3);
    {
        const float g = P.d_map[(int64_t)b * 256 + tid];
        d3[tid] = d3[tid] > 0.0f ? g : g * slope;
    }
    __syncthreads();
    // conv3: dW3[co][ci][ky][kx] = sum_(y, x) dpre3[co][y][x] c2[ci][y + ky - 1][x + kx - 1], db3[co] = sum dpre3[co]
    for (int o = tid; o < 4 * 32 * 9 + 4; o += AC_THREADS) {
        float acc = 0.0f;
        if (o < 4 * 32 * 9) {
            const int co = o / 288, ci = (o / 9) % 32, ky = (o % 9) / 3, kx = o % 3;
            const float* d = d3 + co * 64;
            const float* in = c2 + ci * 64;
            for (int y = 0; y < 8; ++y) {
                const int iy = y + ky - 1;
                if (iy < 0 || iy >= 8) continue;
                for (int x = 0; x < 8; ++x) {
                    const int ix = x + kx - 1;
                    if (ix < 0 || ix >= 8) continue;
                    acc = __fmaf_rn(d[y * 8 + x], in[iy * 8 + ix], acc);
                }
            }
            part[HE_W3 + o] = acc;
        } else {
            const float* d = d3 + (o - 4 * 32 * 9) * 64;
            for (int p = 0; p < 64; ++p) acc += d[p];
            part[HE_B3 + o - 4 * 32 * 9] = acc;
        }
    }
    // dpre2[ci][y][x] = sum_(co, ky, kx) dpre3[co][y - ky + 1][x - kx + 1] W3[co][ci][ky][kx], times leaky'(c2)
    for (int o = tid; o < 32 * 64; o += AC_THREADS) {
        const int ci = o >> 6, y = (o >> 3) & 7, x = o & 7;
        float acc = 0.0f;
        for (int co = 0; co < 4; ++co) {
            const float* wk = w.conv3_w + (co * 32 + ci) * 9;
            const float* d = d3 + co * 64;
            for (int ky = 0; ky < 3; ++ky) {
                const int oy = y - ky + 1;
                if (oy < 0 || oy >= 8) continue;
                for (int kx = 0; kx < 3; ++kx) {
                    const int ox = x - kx + 1;
                    if (ox < 0 || ox >= 8) continue;
                    acc = __fmaf_rn(d[oy * 8 + ox], wk[ky * 3 + kx], acc);
                }
            }
        }
        d2[ci * HE_LD2 + (o & 63)] = c2[o] > 0.0f ? acc : acc * slope;
    }
    __syncthreads();
    // conv2: dW2[co][ci][ky][kx] = sum_(y, x) dpre2[co][y][x] c1[ci][2y - 1 + ky][2x - 1 + kx].  A thread owns the 16
    // taps of one (co, ci) pair: lanes over co (dpre2's padded rows), a warp's ci shared (c1 reads broadcast).
    for (int pr = tid; pr < 32 * 16; pr += AC_THREADS) {
        const int co = pr & 31, ci = pr >> 5;
        const float* d = d2 + co * HE_LD2;
        const float* in = c1 + ci * 256;
        float acc[16];
#pragma unroll
        for (int t = 0; t < 16; ++t) acc[t] = 0.0f;
        for (int y = 0; y < 8; ++y)
            for (int x = 0; x < 8; ++x) {
                const float g = d[y * 8 + x];
#pragma unroll
                for (int ky = 0; ky < 4; ++ky) {
                    const int iy = 2 * y - 1 + ky;
#pragma unroll
                    for (int kx = 0; kx < 4; ++kx) {
                        const int ix = 2 * x - 1 + kx;
                        if (iy >= 0 && iy < 16 && ix >= 0 && ix < 16)
                            acc[ky * 4 + kx] = __fmaf_rn(g, in[iy * 16 + ix], acc[ky * 4 + kx]);
                    }
                }
            }
        float* out = part + HE_W2 + (co * 16 + ci) * 16;
#pragma unroll
        for (int t = 0; t < 16; ++t) out[t] = acc[t];
    }
    if (tid < 32) {
        float acc = 0.0f;
        for (int p = 0; p < 64; ++p) acc += d2[tid * HE_LD2 + p];
        part[HE_B2 + tid] = acc;
    }
    __syncthreads();
    // dpre1[ci][iy][ix] = sum_co sum_(ky, kx: iy = 2y - 1 + ky, ix = 2x - 1 + kx) dpre2[co][y][x] W2[co][ci][ky][kx],
    // times leaky'(c1); in place (each thread reads and writes only its own elements of c1)
    for (int o = tid; o < 16 * 256; o += AC_THREADS) {
        const int ci = o >> 8, iy = (o >> 4) & 15, ix = o & 15;
        const int ky0 = (iy + 1) & 1, kx0 = (ix + 1) & 1;    // the two taps of each axis: k0 and k0 + 2
        float acc = 0.0f;
        for (int co = 0; co < 32; ++co) {
            const float* wk = w.conv2_w + (co * 16 + ci) * 16;
            const float* d = d2 + co * HE_LD2;
#pragma unroll
            for (int a = 0; a < 2; ++a) {
                const int ky = ky0 + 2 * a, y = (iy + 1 - ky) / 2;
                if (y < 0 || y >= 8) continue;
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int kx = kx0 + 2 * c, x = (ix + 1 - kx) / 2;
                    if (x < 0 || x >= 8) continue;
                    acc = __fmaf_rn(d[y * 8 + x], wk[ky * 4 + kx], acc);
                }
            }
        }
        c1[o] = c1[o] > 0.0f ? acc : acc * slope;
    }
    __syncthreads();
    // conv1: dW1[co][0][ky][kx] = sum_(y, x) dpre1[co][y][x] hm[2y - 1 + ky][2x - 1 + kx]; db1[co] = sum dpre1[co]
    for (int o = tid; o < 16 * 16 + 16; o += AC_THREADS) {
        float acc = 0.0f;
        if (o < 16 * 16) {
            const int co = o >> 4, ky = (o >> 2) & 3, kx = o & 3;
            const float* d = c1 + co * 256;
            for (int y = 0; y < 16; ++y) {
                const int iy = 2 * y - 1 + ky;
                if (iy < 0 || iy >= AC_HM) continue;
                for (int x = 0; x < 16; ++x) {
                    const int ix = 2 * x - 1 + kx;
                    if (ix < 0 || ix >= AC_HM) continue;
                    acc = __fmaf_rn(d[y * 16 + x], hm[iy * AC_HM + ix], acc);
                }
            }
            part[HE_W1 + o] = acc;
        } else {
            const float* d = c1 + (o - 16 * 16) * 256;
            for (int p = 0; p < 256; ++p) acc += d[p];
            part[HE_B1 + o - 16 * 16] = acc;
        }
    }
}

// One pass of the reduction over the samples: rows of HE_GRADS floats at part + r * row_stride, r < rows; row g *
// HE_GROUP of the result (stored in place, at row g * HE_GROUP) is the sum of rows g * HE_GROUP .. g * HE_GROUP +
// HE_GROUP - 1 in order.  With rows <= HE_GROUP the pass is the last one and writes the six outputs.
__global__ void __launch_bounds__(AC_THREADS) irbpp_height_encoder_reduce_kernel(float* part, int64_t row_stride,
                                                                                 int32_t rows, const HeightEncoderGrads G) {
    const int64_t groups = (rows + HE_GROUP - 1) / HE_GROUP, total = groups * HE_GRADS;
    for (int64_t i = (int64_t)blockIdx.x * AC_THREADS + threadIdx.x; i < total; i += (int64_t)gridDim.x * AC_THREADS) {
        const int64_t g = i / HE_GRADS;
        const int e = (int)(i % HE_GRADS);
        const int64_t r0 = g * HE_GROUP, r1 = r0 + HE_GROUP < rows ? r0 + HE_GROUP : rows;
        float* p = part + r0 * row_stride + e;
        float s = *p;
        for (int64_t r = r0 + 1; r < r1; ++r) s += part[r * row_stride + e];
        if (groups > 1) { *p = s; continue; }
        if (e < HE_B1) G.conv1_w[e - HE_W1] = s;
        else if (e < HE_W2) G.conv1_b[e - HE_B1] = s;
        else if (e < HE_B2) G.conv2_w[e - HE_W2] = s;
        else if (e < HE_W3) G.conv2_b[e - HE_B2] = s;
        else if (e < HE_B3) G.conv3_w[e - HE_W3] = s;
        else G.conv3_b[e - HE_B3] = s;
    }
}

}  // namespace irbpp
