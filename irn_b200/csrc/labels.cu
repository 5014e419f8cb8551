// S1: random-walk scores -> label map.
// Reference: step/make_sem_seg_labels.py:43-49 and step/make_ins_seg_labels.py:137-143:
//   rw_up = bilinear x4 (align_corners=False)[..., :H, :W];  rw_up /= max(rw_up);
//   argmax over [bg_thres, rw_up_0, rw_up_1, ...] (ties -> lowest index);  keys[argmax].
#include "common.h"

namespace irn {

constexpr int kMaxKeys = IRN_CAM_MAX_CLASSES + 1;

struct LabelKeys {     // class id per argmax index (entry 0 = background), passed by value: no device copy, no host sync
    int n;
    int v[kMaxKeys];
};

// torch upsample_bilinear2d, align_corners=False, scale_factor=4: src = max(0,(dst+0.5)/4-0.5)
__device__ __forceinline__ void src_index4(int dst, int in_size, int& i0, int& i1, float& l1) {
    float s = ((float)dst + 0.5f) * 0.25f - 0.5f;
    s = s < 0.f ? 0.f : s;
    i0 = (int)s;
    if (i0 > in_size - 1) i0 = in_size - 1;
    i1 = i0 + (i0 < in_size - 1 ? 1 : 0);
    l1 = s - (float)i0;
}

__device__ __forceinline__ float bilerp4(const float* __restrict__ p, int w, int y0, int y1, float ly, int x0, int x1, float lx) {
    const float ly0 = 1.f - ly, lx0 = 1.f - lx;
    // same association as ATen's CPU kernel: w_y0*(w_x0*a + w_x1*b) + w_y1*(w_x0*c + w_x1*d)
    const float top = __fadd_rn(__fmul_rn(lx0, p[y0 * w + x0]), __fmul_rn(lx, p[y0 * w + x1]));
    const float bot = __fadd_rn(__fmul_rn(lx0, p[y1 * w + x0]), __fmul_rn(lx, p[y1 * w + x1]));
    return __fadd_rn(__fmul_rn(ly0, top), __fmul_rn(ly, bot));
}

// pass 1: global max of the upsampled, cropped scores (all >= 0, so int compare works)
__global__ void labels_max_kernel(const float* __restrict__ rw, int C, int h, int w, int H, int W, int* __restrict__ gmax_bits) {
    const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y;
    float m = 0.f;
    if (X < W) {
        int y0, y1, x0, x1;
        float ly, lx;
        src_index4(Y, h, y0, y1, ly);
        src_index4(X, w, x0, x1, lx);
        for (int c = 0; c < C; ++c) m = fmaxf(m, bilerp4(rw + (size_t)c * h * w, w, y0, y1, ly, x0, x1, lx));
    }
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    __shared__ float s_m[32];
    if ((threadIdx.x & 31) == 0) s_m[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x < 32) {
        m = threadIdx.x < (blockDim.x >> 5) ? s_m[threadIdx.x] : 0.f;
        for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (threadIdx.x == 0) atomicMax(gmax_bits, __float_as_int(m));
    }
}

// pass 2: normalise, argmax against the background plane, map through keys
__global__ void labels_argmax_kernel(const float* __restrict__ rw, int C, int h, int w, int H, int W, float bg,
                                     LabelKeys keys, const int* __restrict__ gmax_bits,
                                     uint8_t* __restrict__ labels, int32_t* __restrict__ index_out,
                                     float* __restrict__ up_norm) {
    const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y;
    if (X >= W) return;
    const float gmax = __int_as_float(*gmax_bits);
    int y0, y1, x0, x1;
    float ly, lx;
    src_index4(Y, h, y0, y1, ly);
    src_index4(X, w, x0, x1, lx);
    float best = bg;
    int arg = 0;
    for (int c = 0; c < C; ++c) {
        const float v = __fdiv_rn(bilerp4(rw + (size_t)c * h * w, w, y0, y1, ly, x0, x1, lx), gmax);
        if (up_norm) up_norm[((size_t)c * H + Y) * W + X] = v;
        if (v > best || (v != v && best == best)) {   // strict: ties keep the lower index; NaN wins like torch.argmax
            best = v;
            arg = c + 1;
        }
    }
    if (labels) labels[(size_t)Y * W + X] = (uint8_t)(keys.n ? keys.v[arg] : arg);
    if (index_out) index_out[(size_t)Y * W + X] = arg;
}

}  // namespace irn

using namespace irn;

extern "C" int irn_rw_labels(const float* rw, int C, int h, int w, int H, int W, float bg_thres, const int32_t* keys_host,
                             uint8_t* labels, int32_t* index_out, float* up_norm, void* scratch, irn_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    launch_counter() = 0;
    if (!rw || !scratch || (!labels && !index_out && !up_norm)) return fail(kBadArg, "irn_rw_labels: null pointer");
    if (C <= 0 || h <= 0 || w <= 0 || H <= 0 || W <= 0 || H > 4 * h || W > 4 * w)
        return fail(kBadArg, "irn_rw_labels: bad sizes C=%d h=%d w=%d H=%d W=%d (need H<=4h, W<=4w)", C, h, w, H, W);
    LabelKeys keys;
    keys.n = 0;
    if (keys_host) {
        if (C + 1 > kMaxKeys)
            return fail(kUnsupported, "irn_rw_labels: a key table of %d entries exceeds %d (pass NULL and map the index map on the host)", C + 1,
                        kMaxKeys);
        keys.n = C + 1;
        for (int i = 0; i <= C; ++i) keys.v[i] = keys_host[i];
    }
    IRN_CUDA(cudaMemsetAsync(scratch, 0, sizeof(int), stream));
    dim3 block(128), grid((W + 127) / 128, H);
    labels_max_kernel<<<grid, block, 0, stream>>>(rw, C, h, w, H, W, (int*)scratch);
    IRN_LAUNCH_CHECK("labels_max_kernel");
    labels_argmax_kernel<<<grid, block, 0, stream>>>(rw, C, h, w, H, W, bg_thres, keys, (const int*)scratch, labels,
                                                     index_out, up_norm);
    IRN_LAUNCH_CHECK("labels_argmax_kernel");
    return kOk;
}
