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

// strict: ties keep the lower index; the first NaN wins like torch.argmax / np.argmax
__device__ __forceinline__ bool argmax_takes(float v, float best) { return v > best || (v != v && best == best); }

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
        if (argmax_takes(v, best)) {
            best = v;
            arg = c + 1;
        }
    }
    if (labels) labels[(size_t)Y * W + X] = (uint8_t)(keys.n ? keys.v[arg] : arg);
    if (index_out) index_out[(size_t)Y * W + X] = arg;
}

// ---------------------------------------------------------------------------------------------- background-threshold sweep
// At threshold t a pixel is labelled keys[c+1] if its foreground maximum m (first index c on ties, the first NaN if any) exceeds t,
// else background (m == t is background: the argmax keeps index 0).  c and m do not depend on t, so each pixel is counted once in
// hist[g][p][b], b = number of thresholds below m (T for NaN), p = keys[c+1] (0 when b == 0), and threshold j's confusion is the
// suffix sum over b > j; its background column is the rest of row g.
constexpr int kSweepMaxThresholds = 256;

struct SweepTable {    // ascending float32 thresholds and the image's key table, passed by value like LabelKeys
    int T;
    float thr[kSweepMaxThresholds];
    LabelKeys keys;
};

// error words after the histogram: [0] flags (1 = a predicted label >= n_class, 2 = a ground truth >= n_class and != 255),
// [1] the largest such label, [2] the largest such ground truth
constexpr int kSweepErrWords = 4;

__host__ __device__ inline size_t sweep_hist_bytes(int T, int n_class) {
    return (size_t)n_class * n_class * (T + 1) * sizeof(unsigned long long);
}

// kWalk: scores are the walk [C,h,w], upsampled x4, cropped to (H,W) and divided by the global max as in labels_argmax_kernel;
// otherwise full-resolution planes [C,H,W] used as stored
template <bool kWalk>
__global__ void sweep_accumulate_kernel(const float* __restrict__ s, int C, int h, int w, int H, int W, const __grid_constant__ SweepTable tab,
                                        const int* __restrict__ gmax_bits, const uint8_t* __restrict__ gt, int n_class,
                                        unsigned long long* __restrict__ hist, int* __restrict__ err) {
    const int X = blockIdx.x * blockDim.x + threadIdx.x, Y = blockIdx.y;
    int bin = -1;
    const int g = X < W ? gt[(size_t)Y * W + X] : 255;
    if (g != 255 && g >= n_class) {
        atomicOr(err, 2);
        atomicMax(err + 2, g);
    } else if (g != 255) {
        int b = 0, label = 0;
        if (C > 0) {
            float best;
            int arg = 0;
            if (kWalk) {
                const float gmax = __int_as_float(*gmax_bits);
                int y0, y1, x0, x1;
                float ly, lx;
                src_index4(Y, h, y0, y1, ly);
                src_index4(X, w, x0, x1, lx);
                best = __fdiv_rn(bilerp4(s, w, y0, y1, ly, x0, x1, lx), gmax);
                for (int c = 1; c < C; ++c) {
                    const float v = __fdiv_rn(bilerp4(s + (size_t)c * h * w, w, y0, y1, ly, x0, x1, lx), gmax);
                    if (argmax_takes(v, best)) {
                        best = v;
                        arg = c;
                    }
                }
            } else {
                const size_t plane = (size_t)H * W, at = (size_t)Y * W + X;
                best = s[at];
                for (int c = 1; c < C; ++c) {
                    const float v = s[c * plane + at];
                    if (argmax_takes(v, best)) {
                        best = v;
                        arg = c;
                    }
                }
            }
            if (best != best) {
                b = tab.T;                      // NaN wins against every threshold
            } else {
                int lo = 0, hi = tab.T;         // first threshold >= best
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (tab.thr[mid] < best) lo = mid + 1;
                    else hi = mid;
                }
                b = lo;
            }
            if (b > 0) {
                label = tab.keys.v[arg + 1];
                if ((unsigned)label >= (unsigned)n_class) {
                    atomicOr(err, 1);
                    atomicMax(err + 1, label);
                    b = -1;
                }
            }
        }
        if (b >= 0) bin = (g * n_class + label) * (tab.T + 1) + b;
    }
    // neighbouring pixels mostly share a bin: one atomic per distinct bin of the warp
    const unsigned peers = __match_any_sync(0xffffffffu, bin);
    if (bin >= 0 && (int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(hist + bin, (unsigned long long)__popc(peers));
}

// one block per ground-truth class g: conf[j][g][p] = sum_{b>j} hist[g][p][b] for p >= 1, conf[j][g][0] = row total - the rest
__global__ void sweep_finalize_kernel(const unsigned long long* __restrict__ hist, int T, int n, long long* __restrict__ conf) {
    const int g = blockIdx.x;
    __shared__ unsigned long long total;
    if (threadIdx.x == 0) total = 0;
    __syncthreads();
    unsigned long long part = 0;
    for (int p = threadIdx.x; p < n; p += blockDim.x) {
        const unsigned long long* row = hist + ((size_t)g * n + p) * (T + 1);
        unsigned long long acc = 0;
        for (int b = T; b >= 1; --b) {
            acc += row[b];
            if (p) conf[((size_t)(b - 1) * n + g) * n + p] = (long long)acc;
        }
        part += acc + row[0];
    }
    atomicAdd(&total, part);
    __syncthreads();
    for (int j = threadIdx.x; j < T; j += blockDim.x) {
        long long* r = conf + ((size_t)j * n + g) * n;
        long long fg = 0;
        for (int p = 1; p < n; ++p) fg += r[p];
        r[0] = (long long)total - fg;
    }
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

extern "C" size_t irn_threshold_sweep_bytes(int T, int n_class) {
    if (T < 1 || T > kSweepMaxThresholds || n_class < 1 || n_class > kMaxKeys) return 0;
    return sweep_hist_bytes(T, n_class) + kSweepErrWords * sizeof(int);
}

static int sweep_check_table(const char* who, int T, int n_class) {
    if (T < 1 || T > kSweepMaxThresholds) return fail(kBadArg, "%s: %d thresholds (need 1..%d)", who, T, kSweepMaxThresholds);
    if (n_class < 1 || n_class > kMaxKeys) return fail(kBadArg, "%s: n_class=%d (need 1..%d)", who, n_class, kMaxKeys);
    return kOk;
}

extern "C" int irn_threshold_sweep_accumulate(int source, const float* scores, int C, int h, int w, int H, int W, const int32_t* keys_host,
                                              const uint8_t* gt, const float* thresholds_host, int T, int n_class, void* hist, void* scratch,
                                              irn_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    launch_counter() = 0;
    const char* who = "irn_threshold_sweep_accumulate";
    if (int rc = sweep_check_table(who, T, n_class)) return rc;
    if (source != IRN_SWEEP_PLANES && source != IRN_SWEEP_WALK) return fail(kBadArg, "%s: unknown score source %d", who, source);
    const bool walk = source == IRN_SWEEP_WALK;
    if (!gt || !hist || !keys_host || !thresholds_host || (C > 0 && (!scores || (walk && !scratch))))
        return fail(kBadArg, "%s: null pointer", who);
    if (C < 0 || C + 1 > kMaxKeys) return fail(kBadArg, "%s: C=%d classes (need 0..%d)", who, C, kMaxKeys - 1);
    if (H <= 0 || W <= 0 || H > 65535 || h <= 0 || w <= 0 || (walk ? (H > 4 * h || W > 4 * w) : (h != H || w != W)))
        return fail(kBadArg, "%s: sizes h=%d w=%d do not match H=%d W=%d (%s)", who, h, w, H, W,
                    walk ? "a walk needs H<=4h, W<=4w" : "planes are [C,H,W]");
    SweepTable tab;
    tab.T = T;
    for (int i = 0; i < T; ++i) {
        tab.thr[i] = thresholds_host[i];
        if (!(thresholds_host[i] == thresholds_host[i]) || (i && !(thresholds_host[i - 1] < thresholds_host[i])))
            return fail(kBadArg, "%s: thresholds must be strictly ascending and not NaN (entry %d = %g)", who, i, (double)thresholds_host[i]);
    }
    if (keys_host[0] != 0) return fail(kBadArg, "%s: key table entry 0 (background) is %d, must be 0", who, keys_host[0]);
    tab.keys.n = C + 1;
    for (int i = 0; i <= C; ++i) tab.keys.v[i] = keys_host[i];
    unsigned long long* hh = (unsigned long long*)hist;
    int* err = (int*)((char*)hist + sweep_hist_bytes(T, n_class));
    dim3 block(128), grid((W + 127) / 128, H);
    if (walk && C > 0) {
        IRN_CUDA(cudaMemsetAsync(scratch, 0, sizeof(int), stream));
        labels_max_kernel<<<grid, block, 0, stream>>>(scores, C, h, w, H, W, (int*)scratch);
        IRN_LAUNCH_CHECK("labels_max_kernel");
        sweep_accumulate_kernel<true><<<grid, block, 0, stream>>>(scores, C, h, w, H, W, tab, (const int*)scratch, gt, n_class, hh, err);
    } else {
        sweep_accumulate_kernel<false><<<grid, block, 0, stream>>>(scores, C, h, w, H, W, tab, nullptr, gt, n_class, hh, err);
    }
    IRN_LAUNCH_CHECK("sweep_accumulate_kernel");
    return kOk;
}

extern "C" int irn_threshold_sweep_finalize(const void* hist, int T, int n_class, int64_t* conf, irn_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    launch_counter() = 0;
    const char* who = "irn_threshold_sweep_finalize";
    if (int rc = sweep_check_table(who, T, n_class)) return rc;
    if (!hist || !conf) return fail(kBadArg, "%s: null pointer", who);
    int err[kSweepErrWords];
    IRN_CUDA(cudaMemcpyAsync(err, (const char*)hist + sweep_hist_bytes(T, n_class), sizeof(err), cudaMemcpyDeviceToHost, stream));
    IRN_CUDA(cudaStreamSynchronize(stream));
    if (err[0] & 1) return fail(kBadArg, "%s: a predicted label %d is outside [0, %d)", who, err[1], n_class);
    if (err[0] & 2) return fail(kBadArg, "%s: a ground-truth label %d is outside [0, %d) (255 = ignore)", who, err[2], n_class);
    sweep_finalize_kernel<<<n_class, 128, 0, stream>>>((const unsigned long long*)hist, T, n_class, (long long*)conf);
    IRN_LAUNCH_CHECK("sweep_finalize_kernel");
    return kOk;
}
