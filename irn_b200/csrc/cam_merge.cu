// C4: multi-scale CAM merge.  Reference: step/make_cam.py:38-52.
//   strided_cam = sum_s bilinear(cam_s -> (ceil(H/4), ceil(W/4)));     highres = sum_s bilinear(cam_s -> (16*ceil(H/16), ...))[:H,:W]
//   keep the classes present in the image label; each kept map /= (its max over pixels + 1e-5).
// F.interpolate(size=..., mode='bilinear', align_corners=False): src = max(0, (dst+0.5)*in/out - 0.5).
#include "common.h"

namespace irn {

constexpr int kMaxScales = 8;

struct MergeArgs {
    const float* cam[kMaxScales];   // each [C, hs, ws]
    int hs[kMaxScales], ws[kMaxScales];
    int n_scales, n_cls;
    int keys[IRN_CAM_MAX_CLASSES];  // classes present (<= C), by value
};

__device__ __forceinline__ void src_index(int dst, float scale, int in_size, int& i0, int& i1, float& l1) {
    float s = scale * ((float)dst + 0.5f) - 0.5f;
    s = s < 0.f ? 0.f : s;
    i0 = (int)s;
    if (i0 > in_size - 1) i0 = in_size - 1;
    i1 = i0 + (i0 < in_size - 1 ? 1 : 0);
    l1 = s - (float)i0;
    l1 = l1 < 0.f ? 0.f : (l1 > 1.f ? 1.f : l1);
}

// out[k, y, x] (y < Hc, x < Wc) = sum over scales of the bilinear resample to a (Ho, Wo) grid; also tracks max per k
__global__ void cam_merge_kernel(MergeArgs a, int K, int Ho, int Wo, int Hc, int Wc,
                                 float* __restrict__ out, int* __restrict__ max_bits) {
    const int k = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    float v = 0.f;
    if (i < Hc * Wc) {
        const int y = i / Wc, x = i % Wc;
        const int cls = a.keys[k];
        for (int s = 0; s < a.n_scales; ++s) {
            const int hs = a.hs[s], ws = a.ws[s];
            int y0, y1, x0, x1;
            float ly, lx;
            src_index(y, (float)hs / (float)Ho, hs, y0, y1, ly);
            src_index(x, (float)ws / (float)Wo, ws, x0, x1, lx);
            const float* p = a.cam[s] + (size_t)cls * hs * ws;
            const float top = __fadd_rn(__fmul_rn(1.f - lx, p[y0 * ws + x0]), __fmul_rn(lx, p[y0 * ws + x1]));
            const float bot = __fadd_rn(__fmul_rn(1.f - lx, p[y1 * ws + x0]), __fmul_rn(lx, p[y1 * ws + x1]));
            v = __fadd_rn(v, __fadd_rn(__fmul_rn(1.f - ly, top), __fmul_rn(ly, bot)));
        }
        out[(size_t)k * Hc * Wc + i] = v;
    }
    float m = v;   // CAMs are sums of ReLU outputs: >= 0, so the int ordering of the bit patterns is the float ordering
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(max_bits + k, __float_as_int(m));
}

__global__ void cam_norm_kernel(float* __restrict__ x, const int* __restrict__ max_bits, int n_per) {
    const int k = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_per) return;
    const float d = __int_as_float(max_bits[k]) + 1e-5f;   // step/make_cam.py:49,52
    x[(size_t)k * n_per + i] = __fdiv_rn(x[(size_t)k * n_per + i], d);
}

}  // namespace irn

using namespace irn;

extern "C" int irn_cam_merge_classes(const float* const* cams, const int* hs, const int* ws, int n_scales, int n_classes, int H, int W,
                                     const int32_t* keys_host, int K, float* strided_out, float* highres_out, void* scratch,
                                     irn_stream_t stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    launch_counter() = 0;
    if (!cams || !hs || !ws || !scratch || n_scales <= 0 || n_scales > kMaxScales || H <= 0 || W <= 0 || K < 0)
        return fail(kBadArg, "irn_cam_merge: bad argument (n_scales must be 1..%d)", kMaxScales);
    if (K == 0) return kOk;
    if (!keys_host || (!strided_out && !highres_out)) return fail(kBadArg, "irn_cam_merge: null pointer");
    if (n_classes < 1 || n_classes > IRN_CAM_MAX_CLASSES)
        return fail(kBadArg, "irn_cam_merge: %d classes, need 1..%d", n_classes, IRN_CAM_MAX_CLASSES);
    if (K > n_classes) return fail(kBadArg, "irn_cam_merge: K=%d exceeds the %d classes", K, n_classes);
    MergeArgs a;
    a.n_scales = n_scales;
    a.n_cls = n_classes;
    for (int k = 0; k < K; ++k) {
        if (keys_host[k] < 0 || keys_host[k] >= n_classes)
            return fail(kBadArg, "irn_cam_merge: class id %d out of range [0, %d)", keys_host[k], n_classes);
        a.keys[k] = keys_host[k];
    }
    for (int s = 0; s < n_scales; ++s) {
        a.cam[s] = cams[s];
        a.hs[s] = hs[s];
        a.ws[s] = ws[s];
    }
    int* mx = (int*)scratch;
    IRN_CUDA(cudaMemsetAsync(mx, 0, (size_t)2 * K * sizeof(int), st));
    const int h4 = (H - 1) / 4 + 1, w4 = (W - 1) / 4 + 1;                 // misc/imutils.py:173-174
    const int Hu = ((H - 1) / 16 + 1) * 16, Wu = ((W - 1) / 16 + 1) * 16;   // misc/imutils.py:177-179
    if (strided_out) {
        dim3 grid((h4 * w4 + 255) / 256, K);
        cam_merge_kernel<<<grid, 256, 0, st>>>(a, K, h4, w4, h4, w4, strided_out, mx);
        IRN_LAUNCH_CHECK("cam_merge_kernel(strided)");
        cam_norm_kernel<<<grid, 256, 0, st>>>(strided_out, mx, h4 * w4);
        IRN_LAUNCH_CHECK("cam_norm_kernel(strided)");
    }
    if (highres_out) {
        dim3 grid((H * W + 255) / 256, K);
        cam_merge_kernel<<<grid, 256, 0, st>>>(a, K, Hu, Wu, H, W, highres_out, mx + K);
        IRN_LAUNCH_CHECK("cam_merge_kernel(highres)");
        cam_norm_kernel<<<grid, 256, 0, st>>>(highres_out, mx + K, H * W);
        IRN_LAUNCH_CHECK("cam_norm_kernel(highres)");
    }
    return kOk;
}

extern "C" int irn_cam_merge(const float* const* cams, const int* hs, const int* ws, int n_scales, int H, int W, const int32_t* keys_host,
                             int K, float* strided_out, float* highres_out, void* scratch, irn_stream_t stream_) {
    return irn_cam_merge_classes(cams, hs, ws, n_scales, 20, H, W, keys_host, K, strided_out, highres_out, scratch, stream_);
}
