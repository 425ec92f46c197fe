// irbpp_pack.cuh -- lossless compact form of the location observation for the rollout gather (SURVEY.md 8e).
//
// The float32 observation of a bin is [sel x (rot, x, y, H, V) | next_item_vec(9) | heightmap(1024)] = 14 132 bytes at
// sel = 500 (binPhy.py:196-227), most of it small integers stored as floats and zero padding.  Between GPUs it travels as
//   u16 rot << 10 | x << 5 | y  per row  |  f32 H per row  |  one V bit per row  |  f32 item id  |  f32 heightmap
// = 7 184 bytes at sel = 500 (51 %), and is expanded on the receiver.  The encoding is exact for what the environment
// emits on either action grid: rot < 64, x, y < 32 integers, V in {0, 1}, next_item_vec = (id, 0, ..., 0) (binPhy.py:191).
#pragma once
#include <stdint.h>

namespace irbpp {

__host__ __device__ inline int packed_words(int sel) {       // 32-bit words per bin, a multiple of 4 (16 bytes)
    const int w = (sel + 1) / 2 + sel + (sel + 31) / 32 + 1 + 1024;
    return (w + 3) & ~3;
}

// one CTA per bin
__global__ void irbpp_pack_obs_kernel(const float* __restrict__ obs, int64_t obs_stride, int sel, uint32_t* __restrict__ out, int n) {
    const int b = blockIdx.x;
    if (b >= n) return;
    const float* o = obs + (int64_t)b * obs_stride;
    uint32_t* p = out + (int64_t)b * packed_words(sel);
    const int ncw = (sel + 1) / 2, nvw = (sel + 31) / 32;
    for (int i = threadIdx.x; i < ncw; i += blockDim.x) {
        uint32_t w = 0;
        for (int h = 0; h < 2; ++h) {
            const int row = 2 * i + h;
            if (row < sel) {
                const float* r = o + row * 5;
                w |= ((((uint32_t)r[0]) << 10) | (((uint32_t)r[1]) << 5) | ((uint32_t)r[2])) << (16 * h);
            }
        }
        p[i] = w;
    }
    float* hp = reinterpret_cast<float*>(p + ncw);
    for (int row = threadIdx.x; row < sel; row += blockDim.x) hp[row] = o[row * 5 + 3];
    uint32_t* vp = p + ncw + sel;
    for (int i = threadIdx.x; i < nvw; i += blockDim.x) {
        uint32_t w = 0;
        for (int k = 0; k < 32; ++k) { const int row = 32 * i + k; if (row < sel && o[row * 5 + 4] != 0.0f) w |= 1u << k; }
        vp[i] = w;
    }
    float* ip = reinterpret_cast<float*>(vp + nvw);
    if (threadIdx.x == 0) ip[0] = o[sel * 5];
    const float* hm = o + sel * 5 + 9;
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) ip[1 + i] = hm[i];
}

__global__ void irbpp_unpack_obs_kernel(const uint32_t* __restrict__ in, int sel, float* __restrict__ obs, int64_t obs_stride, int n) {
    const int b = blockIdx.x;
    if (b >= n) return;
    const uint32_t* p = in + (int64_t)b * packed_words(sel);
    float* o = obs + (int64_t)b * obs_stride;
    const int ncw = (sel + 1) / 2, nvw = (sel + 31) / 32;
    const float* hp = reinterpret_cast<const float*>(p + ncw);
    const uint32_t* vp = p + ncw + sel;
    for (int row = threadIdx.x; row < sel; row += blockDim.x) {
        const uint32_t c = (p[row >> 1] >> (16 * (row & 1))) & 0xFFFFu;
        float* r = o + row * 5;
        r[0] = (float)(c >> 10); r[1] = (float)((c >> 5) & 31u); r[2] = (float)(c & 31u);
        r[3] = hp[row];
        r[4] = ((vp[row >> 5] >> (row & 31)) & 1u) ? 1.0f : 0.0f;
    }
    const float* ip = reinterpret_cast<const float*>(vp + nvw);
    if (threadIdx.x < 9) o[sel * 5 + threadIdx.x] = threadIdx.x == 0 ? ip[0] : 0.0f;
    float* hm = o + sel * 5 + 9;
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) hm[i] = ip[1 + i];
}

}  // namespace irbpp
