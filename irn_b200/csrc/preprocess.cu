// C1: multi-scale input preparation on the device.
// Reference: voc12/dataloader.py:191-201 (per scale: rescale, normalise, HWC->CHW, stack with the W-flip),
// misc/imutils.py:8-22 (PIL BICUBIC resize of the uint8 image), voc12/dataloader.py:65-78 (TorchvisionNormalize).
// The bicubic arithmetic is Pillow's 8-bit path (Resample.c, not part of the reference tree): separable, horizontal
// pass first, double-precision coefficients normalised and rounded half away from zero to 22 fractional bits, 8-bit
// intermediate image, accumulators start at 2^21, arithmetic shift, clamp.  Integer work: bit-exact by construction.
// Normalisation has 256 possible inputs per channel: a table computed in double and rounded once to fp32, like numpy.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "common.h"

namespace irn {

constexpr int kPrecisionBits = 32 - 8 - 2;

static inline double bicubic_filter(double x) {
    const double a = -0.5;
    if (x < 0.0) x = -x;
    if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
    if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
    return 0.0;
}

static int coeff_ksize(int in_size, int out_size) {
    const double scale = (double)((float)in_size - 0.0f) / out_size;
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    return (int)std::ceil(2.0 * filterscale) * 2 + 1;
}

// bounds[2*xx] = first source index, bounds[2*xx+1] = tap count; kk[xx*ksize + t] = 22-bit fixed-point weight
static void resize_coeffs(int in_size, int out_size, int32_t* bounds, int32_t* kk, int ksize) {
    const double scale = (double)((float)in_size - 0.0f) / out_size;   // Pillow keeps the box corners as C floats
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    const double support = 2.0 * filterscale;
    const double ss = 1.0 / filterscale;
    std::vector<double> w((size_t)ksize);
    for (int xx = 0; xx < out_size; ++xx) {
        const double center = 0.0 + (xx + 0.5) * scale;
        int xmin = (int)(center - support + 0.5);
        if (xmin < 0) xmin = 0;
        int xmax = (int)(center + support + 0.5);
        if (xmax > in_size) xmax = in_size;
        xmax -= xmin;
        double ww = 0.0;
        for (int x = 0; x < xmax; ++x) {
            w[x] = bicubic_filter((x + xmin - center + 0.5) * ss);
            ww += w[x];
        }
        for (int x = 0; x < ksize; ++x) {
            int32_t v = 0;
            if (x < xmax) {
                const double k = ww != 0.0 ? w[x] / ww : w[x];
                v = k < 0 ? (int32_t)(-0.5 + k * (double)(1 << kPrecisionBits)) : (int32_t)(0.5 + k * (double)(1 << kPrecisionBits));
            }
            kk[(size_t)xx * ksize + x] = v;
        }
        bounds[2 * xx] = xmin;
        bounds[2 * xx + 1] = xmax;
    }
}

__device__ __forceinline__ int clip8(int acc) {
    const int v = acc >> kPrecisionBits;   // arithmetic shift, like Pillow's table lookup on in >> PRECISION_BITS
    return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// One output pixel of a resampling pass: the n taps k[] over the RGB pixels p, p + step, ..., each channel clipped to 8 bits
__device__ __forceinline__ void filter3(const uint8_t* __restrict__ p, size_t step, const int32_t* __restrict__ k, int n, int (&v)[3]) {
    int s0 = 1 << (kPrecisionBits - 1), s1 = s0, s2 = s0;
    for (int t = 0; t < n; ++t) {
        const int kv = k[t];
        s0 += (int)p[0] * kv;
        s1 += (int)p[1] * kv;
        s2 += (int)p[2] * kv;
        p += step;
    }
    v[0] = clip8(s0); v[1] = clip8(s1); v[2] = clip8(s2);
}

// horizontal pass: src [B,H,W,3] -> dst [B,H,ow,3]
__global__ void resize_h_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, const int32_t* __restrict__ bounds,
                                const int32_t* __restrict__ kk, int ksize, int rows, int W, int ow) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)rows * ow) return;
    const int ox = (int)(i % ow);
    const size_t row = i / ow;
    int v[3];
    filter3(src + (row * W + bounds[2 * ox]) * 3, 3, kk + (size_t)ox * ksize, bounds[2 * ox + 1], v);
    uint8_t* o = dst + i * 3;
    o[0] = (uint8_t)v[0];
    o[1] = (uint8_t)v[1];
    o[2] = (uint8_t)v[2];
}

// vertical pass (or identity), then normalise through the table and write both the image and its W-flip as NCHW fp32:
// out[2b] = chw, out[2b+1] = chw[..., ::-1]  (voc12/dataloader.py:199).  src [B,Hs,ow,3].
__global__ void resize_v_norm_kernel(const uint8_t* __restrict__ src, const int32_t* __restrict__ bounds, const int32_t* __restrict__ kk,
                                     int ksize, int has_v, const float* __restrict__ lut, float* __restrict__ out,
                                     uint8_t* __restrict__ out_u8, int B, int Hs, int oh, int ow) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)B * oh * ow) return;
    const int ox = (int)(i % ow);
    const int oy = (int)((i / ow) % oh);
    const int b = (int)(i / ((size_t)ow * oh));
    int v[3];
    if (has_v) {
        filter3(src + (((size_t)b * Hs + bounds[2 * oy]) * ow + ox) * 3, (size_t)ow * 3, kk + (size_t)oy * ksize, bounds[2 * oy + 1], v);
    } else {
        const uint8_t* p = src + (((size_t)b * Hs + oy) * ow + ox) * 3;
        v[0] = p[0]; v[1] = p[1]; v[2] = p[2];
    }
    const int v0 = v[0], v1 = v[1], v2 = v[2];
    if (out_u8) {
        uint8_t* o = out_u8 + i * 3;
        o[0] = (uint8_t)v0; o[1] = (uint8_t)v1; o[2] = (uint8_t)v2;
    }
    if (out) {
        const size_t plane = (size_t)oh * ow;
        float* o = out + (size_t)(2 * b) * 3 * plane + (size_t)oy * ow;
        const float f0 = lut[v0], f1 = lut[256 + v1], f2 = lut[512 + v2];
        o[ox] = f0; o[plane + ox] = f1; o[2 * plane + ox] = f2;
        o += 3 * plane;
        const int fx = ow - 1 - ox;
        o[fx] = f0; o[plane + fx] = f1; o[2 * plane + fx] = f2;
    }
}

// ---- ragged pyramid: images of different sizes, each resized to its own (oh, ow) at the top-left corner of one canvas.
// One descriptor per image, uploaded with the coefficient tables: bounds_h at coef[ch], kk_h at coef[ch + 2 ow] (ksh taps per output
// column; ksh 0 = no horizontal pass, ow == w), likewise bounds_v / kk_v at cv (ksv taps, ksv 0 = no vertical pass, oh == h).
struct RaggedResize {
    long long src;   // byte offset of the uint8 [h,w,3] image in the packed buffer
    long long mid;   // byte offset of its horizontal pass's uint8 [h,ow,3] output in the intermediate buffer
    int h, w, oh, ow, ksh, ksv, ch, cv;
};

// resize_h_kernel for image blockIdx.y.  grid (ceil(max h*ow / 256), P)
__global__ void ragged_resize_h_kernel(const uint8_t* __restrict__ img, const RaggedResize* __restrict__ d, const int32_t* __restrict__ coef,
                                       uint8_t* __restrict__ mid) {
    const RaggedResize r = d[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (r.ksh == 0 || i >= r.h * r.ow) return;
    const int ox = i % r.ow, row = i / r.ow;
    int v[3];
    filter3(img + r.src + ((size_t)row * r.w + coef[r.ch + 2 * ox]) * 3, 3, coef + r.ch + 2 * r.ow + (size_t)ox * r.ksh, coef[r.ch + 2 * ox + 1], v);
    uint8_t* o = mid + r.mid + (size_t)i * 3;
    o[0] = (uint8_t)v[0];
    o[1] = (uint8_t)v[1];
    o[2] = (uint8_t)v[2];
}

// resize_v_norm_kernel for image j = blockIdx.y onto the canvas out [2P,3,Hc,Wc]: sample 2j is the resized image, 2j+1 its W-flip
// within its own width ow, both +0.0 outside oh x ow.  Each thread owns canvas pixel (y, x) of sample 2j, and of sample 2j+1 where that
// pixel is padding.  grid (ceil(Hc*Wc / 256), P)
__global__ void ragged_resize_v_norm_kernel(const uint8_t* __restrict__ img, const RaggedResize* __restrict__ d, const int32_t* __restrict__ coef,
                                            const uint8_t* __restrict__ mid, const float* __restrict__ lut, float* __restrict__ out, int Hc, int Wc) {
    const int j = blockIdx.y;
    const RaggedResize r = d[j];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Hc * Wc) return;
    const int x = i % Wc, y = i / Wc;
    const size_t plane = (size_t)Hc * Wc;
    float* o0 = out + (size_t)(2 * j) * 3 * plane;
    float* o1 = o0 + 3 * plane;
    if (y >= r.oh || x >= r.ow) {
        o0[i] = 0.f; o0[plane + i] = 0.f; o0[2 * plane + i] = 0.f;
        o1[i] = 0.f; o1[plane + i] = 0.f; o1[2 * plane + i] = 0.f;
        return;
    }
    const uint8_t* src = r.ksh ? mid + r.mid : img + r.src;   // [h, ow, 3]
    int v[3];
    if (r.ksv) {
        filter3(src + ((size_t)coef[r.cv + 2 * y] * r.ow + x) * 3, (size_t)r.ow * 3, coef + r.cv + 2 * r.oh + (size_t)y * r.ksv,
                coef[r.cv + 2 * y + 1], v);
    } else {
        const uint8_t* p = src + ((size_t)y * r.ow + x) * 3;
        v[0] = p[0]; v[1] = p[1]; v[2] = p[2];
    }
    const float f0 = lut[v[0]], f1 = lut[256 + v[1]], f2 = lut[512 + v[2]];
    o0[i] = f0; o0[plane + i] = f1; o0[2 * plane + i] = f2;
    const size_t fi = (size_t)y * Wc + (r.ow - 1 - x);
    o1[fi] = f0; o1[plane + fi] = f1; o1[2 * plane + fi] = f2;
}

// Lays out the descriptors and coefficient tables of a ragged pyramid (table: int32 words, descriptors first) and the intermediate
// buffer's size (image i at byte offsets[i]); with table == nullptr only counts
static void ragged_resize_layout(const int32_t* hw, const int32_t* ohw, const int64_t* offsets, int P, std::vector<int32_t>* table,
                                 size_t* table_bytes, size_t* mid_bytes) {
    const size_t desc_words = align_up((size_t)P * sizeof(RaggedResize), 256) / 4;
    size_t words = desc_words, mid = 0;
    std::vector<RaggedResize> desc(P);
    for (int i = 0; i < P; ++i) {
        RaggedResize& r = desc[i];
        r.h = hw[2 * i]; r.w = hw[2 * i + 1]; r.oh = ohw[2 * i]; r.ow = ohw[2 * i + 1];
        r.ksh = r.ow != r.w ? coeff_ksize(r.w, r.ow) : 0;
        r.ksv = r.oh != r.h ? coeff_ksize(r.h, r.oh) : 0;
        r.ch = (int)(words - desc_words);
        words += r.ksh ? (size_t)r.ow * (2 + r.ksh) : 0;
        r.cv = (int)(words - desc_words);
        words += r.ksv ? (size_t)r.oh * (2 + r.ksv) : 0;
        r.src = offsets ? (long long)offsets[i] : 0;
        r.mid = (long long)mid;
        if (r.ksh) mid += align_up((size_t)r.h * r.ow * 3, 256);
    }
    *table_bytes = align_up(words * 4, 256);
    *mid_bytes = mid;
    if (!table) return;
    table->assign(words, 0);
    int32_t* coef = table->data() + desc_words;
    for (int i = 0; i < P; ++i) {
        const RaggedResize& r = desc[i];
        if (r.ksh) resize_coeffs(r.w, r.ow, coef + r.ch, coef + r.ch + 2 * r.ow, r.ksh);
        if (r.ksv) resize_coeffs(r.h, r.oh, coef + r.cv, coef + r.cv + 2 * r.oh, r.ksv);
    }
    std::memcpy(table->data(), desc.data(), (size_t)P * sizeof(RaggedResize));
}

}  // namespace irn

using namespace irn;

struct irn_resize_plan {
    int H, W, oh, ow, ksize_h, ksize_v;
    int32_t *bounds_h, *kk_h, *bounds_v, *kk_v;   // device
    float* lut;                                   // device [3][256]
};

extern "C" int irn_resize_ksize(int in_size, int out_size) {
    if (in_size <= 0 || out_size <= 0) return 0;
    return coeff_ksize(in_size, out_size);
}

extern "C" int irn_resize_coeffs(int in_size, int out_size, int32_t* bounds, int32_t* kk) {
    if (in_size <= 0 || out_size <= 0 || !bounds || !kk) return fail(kBadArg, "irn_resize_coeffs: bad argument");
    resize_coeffs(in_size, out_size, bounds, kk, coeff_ksize(in_size, out_size));
    return kOk;
}

extern "C" int irn_normalize_lut(const double* mean3, const double* std3, float* lut768) {
    if (!mean3 || !std3 || !lut768) return fail(kBadArg, "irn_normalize_lut: null pointer");
    for (int c = 0; c < 3; ++c)
        for (int u = 0; u < 256; ++u) lut768[c * 256 + u] = (float)(((double)u / 255. - mean3[c]) / std3[c]);
    return kOk;
}

static int upload_i32(const std::vector<int32_t>& h, int32_t** d) {
    *d = nullptr;
    if (h.empty()) return kOk;
    IRN_CUDA(cudaMalloc((void**)d, h.size() * sizeof(int32_t)));
    IRN_CUDA(cudaMemcpy(*d, h.data(), h.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
    return kOk;
}

extern "C" int irn_resize_plan_destroy(irn_resize_plan* p) {
    if (!p) return kOk;
    cudaFree(p->bounds_h); cudaFree(p->kk_h); cudaFree(p->bounds_v); cudaFree(p->kk_v); cudaFree(p->lut);
    delete p;
    return kOk;
}

extern "C" int irn_resize_plan_create(int H, int W, int out_h, int out_w, const double* mean3, const double* std3, irn_resize_plan** out) {
    if (!out) return fail(kBadArg, "irn_resize_plan_create: null output");
    *out = nullptr;
    if (H <= 0 || W <= 0 || out_h <= 0 || out_w <= 0 || !mean3 || !std3) return fail(kBadArg, "irn_resize_plan_create: bad argument");
    irn_resize_plan* p = new irn_resize_plan();
    p->H = H; p->W = W; p->oh = out_h; p->ow = out_w;
    p->ksize_h = out_w != W ? coeff_ksize(W, out_w) : 0;
    p->ksize_v = out_h != H ? coeff_ksize(H, out_h) : 0;
    p->bounds_h = p->kk_h = p->bounds_v = p->kk_v = nullptr;
    p->lut = nullptr;
    int rc = kOk;
    if (p->ksize_h) {
        std::vector<int32_t> b((size_t)2 * out_w), k((size_t)out_w * p->ksize_h);
        resize_coeffs(W, out_w, b.data(), k.data(), p->ksize_h);
        if (!rc) rc = upload_i32(b, &p->bounds_h);
        if (!rc) rc = upload_i32(k, &p->kk_h);
    }
    if (!rc && p->ksize_v) {
        std::vector<int32_t> b((size_t)2 * out_h), k((size_t)out_h * p->ksize_v);
        resize_coeffs(H, out_h, b.data(), k.data(), p->ksize_v);
        if (!rc) rc = upload_i32(b, &p->bounds_v);
        if (!rc) rc = upload_i32(k, &p->kk_v);
    }
    if (!rc) {
        float lut[768];
        irn_normalize_lut(mean3, std3, lut);
        rc = check_cuda(cudaMalloc((void**)&p->lut, sizeof(lut)), "cudaMalloc(lut)");
        if (!rc) rc = check_cuda(cudaMemcpy(p->lut, lut, sizeof(lut), cudaMemcpyHostToDevice), "cudaMemcpy(lut)");
    }
    if (rc) {
        irn_resize_plan_destroy(p);
        return rc;
    }
    *out = p;
    return kOk;
}

extern "C" size_t irn_resize_workspace_bytes(const irn_resize_plan* p, int B) {
    if (!p || B <= 0) return 0;
    return p->ksize_h ? align_up((size_t)B * p->H * p->ow * 3, 256) : 256;
}

extern "C" int irn_resize_forward(const irn_resize_plan* p, const uint8_t* img, int B, float* out, uint8_t* out_u8, void* workspace,
                                  size_t workspace_bytes, irn_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    launch_counter() = 0;
    if (!p || !img || B <= 0 || (!out && !out_u8)) return fail(kBadArg, "irn_resize_forward: bad argument");
    const uint8_t* src = img;
    if (p->ksize_h) {
        const size_t need = irn_resize_workspace_bytes(p, B);
        if (!workspace || workspace_bytes < need) return fail(kWorkspace, "irn_resize_forward: workspace %zu < required %zu bytes", workspace_bytes, need);
        const size_t n = (size_t)B * p->H * p->ow;
        resize_h_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(img, (uint8_t*)workspace, p->bounds_h, p->kk_h, p->ksize_h, B * p->H,
                                                                        p->W, p->ow);
        IRN_LAUNCH_CHECK("resize_h_kernel");
        src = (const uint8_t*)workspace;
    }
    const size_t n = (size_t)B * p->oh * p->ow;
    resize_v_norm_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(src, p->bounds_v, p->kk_v, p->ksize_v, p->ksize_v ? 1 : 0, p->lut, out,
                                                                         out_u8, B, p->H, p->oh, p->ow);
    IRN_LAUNCH_CHECK("resize_v_norm_kernel");
    return kOk;
}

static bool ragged_sizes_ok(const int32_t* hw, const int32_t* ohw, int P, int Hc, int Wc) {
    for (int i = 0; i < P; ++i)
        if (hw[2 * i] <= 0 || hw[2 * i + 1] <= 0 || ohw[2 * i] <= 0 || ohw[2 * i + 1] <= 0 || ohw[2 * i] > Hc || ohw[2 * i + 1] > Wc)
            return false;
    return true;
}

extern "C" size_t irn_resize_ragged_workspace_bytes(const int32_t* sizes_hw, const int32_t* out_hw, int P) {
    if (!sizes_hw || !out_hw || P <= 0 || !ragged_sizes_ok(sizes_hw, out_hw, P, INT32_MAX, INT32_MAX)) return 0;
    size_t table, mid;
    ragged_resize_layout(sizes_hw, out_hw, nullptr, P, nullptr, &table, &mid);
    return table + mid;
}

extern "C" int irn_resize_ragged_forward(const uint8_t* img_u8, size_t img_bytes, const int64_t* img_offsets, const int32_t* sizes_hw,
                                         const int32_t* out_hw, int P, int Hc, int Wc, const float* lut768, float* out, void* workspace,
                                         size_t workspace_bytes, irn_stream_t stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    launch_counter() = 0;
    const char* fn = "irn_resize_ragged_forward";
    if (!img_u8 || !img_offsets || !sizes_hw || !out_hw || !lut768 || !out || !workspace) return fail(kBadArg, "%s: bad argument", fn);
    if (P <= 0 || P > 65535 || Hc <= 0 || Wc <= 0)
        return fail(kBadArg, "%s: need 0 < P <= 65535 and a positive canvas; got P=%d Hc=%d Wc=%d", fn, P, Hc, Wc);
    if (is_device_ptr(img_offsets) || is_device_ptr(sizes_hw) || is_device_ptr(out_hw))
        return fail(kBadArg, "%s: offsets and sizes must be host memory", fn);
    if (!ragged_sizes_ok(sizes_hw, out_hw, P, Hc, Wc)) return fail(kBadArg, "%s: need positive sizes and 0 < out_h <= Hc %d, 0 < out_w <= Wc %d", fn, Hc, Wc);
    for (int i = 0; i < P; ++i) {
        const int64_t off = img_offsets[i];
        const uint64_t n = (uint64_t)sizes_hw[2 * i] * sizes_hw[2 * i + 1] * 3;
        if (off < 0 || (uint64_t)off > img_bytes || img_bytes - (uint64_t)off < n)
            return fail(kBadArg, "%s: image %d (%llu bytes at offset %lld) lies outside the %zu-byte image buffer", fn, i, (unsigned long long)n,
                        (long long)off, img_bytes);
    }
    if (!is_device_ptr(img_u8) || !is_device_ptr(lut768) || !is_device_ptr(out) || !is_device_ptr(workspace))
        return fail(kBadArg, "%s: images, table, output and workspace must be device memory", fn);
    if (((uintptr_t)workspace & 255) != 0) return fail(kBadArg, "%s: workspace must be 256-byte aligned", fn);
    std::vector<int32_t> table;
    size_t table_bytes, mid_bytes;
    ragged_resize_layout(sizes_hw, out_hw, img_offsets, P, &table, &table_bytes, &mid_bytes);
    if (workspace_bytes < table_bytes + mid_bytes) return fail(kWorkspace, "%s: workspace too small", fn);
    const RaggedResize* desc = (const RaggedResize*)workspace;
    const int32_t* coef = (const int32_t*)workspace + align_up((size_t)P * sizeof(RaggedResize), 256) / 4;
    uint8_t* mid = (uint8_t*)workspace + table_bytes;
    // one upload per call: it is ordered after the kernels that last read this workspace on the stream
    IRN_CUDA(cudaMemcpyAsync(workspace, table.data(), table.size() * 4, cudaMemcpyHostToDevice, st));
    int most_h = 0;
    for (int i = 0; i < P; ++i)
        if (out_hw[2 * i + 1] != sizes_hw[2 * i + 1]) most_h = std::max(most_h, sizes_hw[2 * i] * out_hw[2 * i + 1]);
    if (most_h > 0) {
        ragged_resize_h_kernel<<<dim3((unsigned)((most_h + 255) / 256), P), 256, 0, st>>>(img_u8, desc, coef, mid);
        IRN_LAUNCH_CHECK("ragged_resize_h_kernel");
    }
    ragged_resize_v_norm_kernel<<<dim3((unsigned)(((size_t)Hc * Wc + 255) / 256), P), 256, 0, st>>>(img_u8, desc, coef, mid, lut768, out, Hc, Wc);
    IRN_LAUNCH_CHECK("ragged_resize_v_norm_kernel");
    return kOk;
}
