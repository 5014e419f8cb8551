// C2/C3/I1/I2: ResNet-50 trunk, CAM head and IRNet edge/displacement heads as a native plan.
//
// Reference: net/resnet50.py:17-91 (Bottleneck / ResNet, strides (2,2,2,1)), net/resnet50_cam.py:55-70
// (CAM.forward), net/resnet50_irn.py:23-133,216-234 (heads, MeanShift, EdgeDisplacement.forward).
//
// The plan owns the repacked weights on the device: FixedBatchNorm folded into (weight, bias), weights
// transposed to [kh*kw*Cin][Cout] for the SIMT kernel and split for the tensor-core kernel (SplitWeights).  Activations
// are NHWC fp32 in a caller-provided workspace.  The host walks the fixed topology and enqueues kernels on the caller's
// stream; nothing synchronises.
#include <cuda_fp16.h>

#include <cmath>
#include <cstring>
#include <vector>

#include "common.h"
#include "conv_simt.cuh"
#include "conv_wgmma.cuh"

namespace irn {

// Device allocations of a plan, freed with it
struct DeviceAllocs {
    std::vector<void*> ptrs;
    DeviceAllocs() = default;
    DeviceAllocs(const DeviceAllocs&) = delete;
    DeviceAllocs& operator=(const DeviceAllocs&) = delete;
    ~DeviceAllocs() {
        for (void* p : ptrs) cudaFree(p);
    }
};

// Weights [cout][K] (K-major) split into hi / lo planes for the tensor-core kernel in one of its two arithmetics (pack_split):
// 3xTF32 fp32 planes, or f16x3 fp16 planes of the weights pre-scaled per output channel by a power of two
struct SplitWeights {
    bool ok = false;                    // packed: the conv is eligible for this arithmetic
    const void* hi = nullptr;           // device [cout][K]
    const void* lo = nullptr;
    CUtensorMap map_hi[2], map_lo[2];   // boxes {one k-block, 64 | 128 rows}; [1] only when cout % 128 == 0
    float* oscale = nullptr;            // f16x3: [cout], the inverse pre-scale applied in the epilogue
};

struct Conv {
    int cin = 0, cout = 0, k = 1, stride = 1, pad = 0;
    float* wt = nullptr;     // device [k*k*cin][cout]   (SIMT kernel)
    float* bias = nullptr;   // device [cout] or null
    SplitWeights tf32, f16;  // the stem's are repacked over its zero-haloed NHWC4 input (build_stem)
};

struct Head {            // conv1x1 (no bias) -> GroupNorm(groups) -> [upsample] -> ReLU
    Conv conv;
    int groups = 1, up = 1;
    float* gamma = nullptr;
    float* beta = nullptr;
};

struct Block {
    Conv c1, c2, c3, ds;
    bool has_ds = false;
    // f16x3 mode: conv3 and the projection shortcut as ONE K-concatenated 1x1 conv, out = relu([W3 | Wds] . [t2 ; x_strided] + b3 + bds):
    // the shortcut tensor (as wide as the block's output) is neither written nor read back
    Conv c3ds;
    bool has_c3ds = false;
};

}  // namespace irn

struct irn_net {
    int kind = 0;   // 0 = CAM, 1 = IRN (EdgeDisplacement)
    int conv_mode = 2;   // 0 = SIMT exact-fp32 convolutions only, 1 = wgmma 3xTF32 where eligible, 2 = wgmma f16x3 (default; 3xTF32 / SIMT for the layers it cannot take)
    irn::Conv stem;
    std::vector<irn::Block> blocks[4];
    // CAM
    float* classifier = nullptr;   // [20][2048] (SIMT head kernel)
    irn::Conv cls_conv;            // the same weights as a 2048 -> 64 1x1 conv (rows 20..63 zero) for the tensor-core path
    // IRN
    irn::Head edge[5], dp[7];
    float* edge6_w = nullptr;      // [1][160]
    float* edge6_b = nullptr;      // [1]
    float* dp7_w = nullptr;        // [2][256]
    float* mean_shift = nullptr;   // [2]
    struct Tap {
        float* dst = nullptr;
        size_t bytes = 0;
    };
    Tap taps[IRN_TAP_COUNT];       // irn_net_set_tap
    irn::DeviceAllocs mem;
};

namespace irn {

static const int kPlanes[4] = {64, 128, 256, 512};
static const int kBlocks[4] = {3, 4, 6, 3};
static const int kStrides[4] = {1, 2, 2, 1};   // layer1..4 under the reference's strides=(2,2,2,1)

struct Reader {
    const float* p;
    size_t left;
    bool ok = true;
    const float* take(size_t n) {
        if (n > left) {
            ok = false;
            return nullptr;
        }
        const float* r = p;
        p += n;
        left -= n;
        return r;
    }
};

template <class T>
static int upload(DeviceAllocs& mem, const std::vector<T>& h, T** out) {
    void* d = nullptr;
    IRN_CUDA(cudaMalloc(&d, h.size() * sizeof(T)));
    mem.ptrs.push_back(d);
    IRN_CUDA(cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
    *out = (T*)d;
    return kOk;
}

// The tensor-core kernel takes a conv whose Cin is a multiple of the arithmetic's k-block `bk` (3xTF32 kTcBK, f16x3 kBfBK), whose
// Cout is a multiple of the 64-wide N tile, with k 1 or 3 and stride 1 or 2
static bool split_eligible(int cin, int cout, int k, int stride, int bk) {
    return cin % bk == 0 && cout % 64 == 0 && (k == 1 || k == 3) && (stride == 1 || stride == 2);
}

// Splits folded fp32 weights wt [K][cout] into the hi / lo planes [cout][K] of one tensor-core arithmetic, uploads them and encodes
// their tensor maps.
//   3xTF32  hi = w rounded to nearest (ties away) to 10 explicit mantissa bits, like cvt.rna.tf32.f32; lo = w - hi.
//   f16x3   every output channel is first scaled by a power of two so that max |w| lies in [1,2): the lo parts stay clear of fp16's
//           subnormal range whatever FixedBatchNorm's gamma / sqrt(var) did to the channel, and the epilogue undoes the scale
//           exactly (oscale).  hi = fp16(v), lo = fp16(v - hi), both rounded to nearest.
static int pack_split(DeviceAllocs& mem, bool f16, const float* wt, size_t K, int cout, SplitWeights& s) {
    const size_t n = (size_t)cout * K;
    int rc;
    if (f16) {
        std::vector<uint16_t> hi(n), lo(n);
        std::vector<float> inv(cout, 1.0f);
        for (int o = 0; o < cout; ++o) {
            float mx = 0.f;
            for (size_t kk = 0; kk < K; ++kk) mx = std::max(mx, std::fabs(wt[kk * cout + o]));
            int e = 1;
            if (mx > 0.f && std::isfinite(mx)) std::frexp(mx, &e);          // mx = m * 2^e, m in [0.5, 1)
            const int sh = 1 - e;                                           // w * 2^sh has its maximum in [1, 2)
            inv[o] = std::ldexp(1.0f, -sh);
            for (size_t kk = 0; kk < K; ++kk) {
                const float v = std::ldexp(wt[kk * cout + o], sh);
                const __half h = __float2half_rn(v);
                const __half l = __float2half_rn(v - __half2float(h));
                hi[(size_t)o * K + kk] = __half_as_ushort(h);
                lo[(size_t)o * K + kk] = __half_as_ushort(l);
            }
        }
        uint16_t *dhi, *dlo;
        if ((rc = upload(mem, inv, &s.oscale)) || (rc = upload(mem, hi, &dhi)) || (rc = upload(mem, lo, &dlo))) return rc;
        s.hi = dhi;
        s.lo = dlo;
    } else {
        std::vector<float> hi(n), lo(n);
        for (int o = 0; o < cout; ++o)
            for (size_t kk = 0; kk < K; ++kk) {
                const float v = wt[kk * cout + o];
                uint32_t u;
                std::memcpy(&u, &v, 4);
                uint32_t h = (u + 0x1000u) & 0xFFFFE000u;
                float hf;
                std::memcpy(&hf, &h, 4);
                if (!std::isfinite(hf)) hf = v;
                hi[(size_t)o * K + kk] = hf;
                lo[(size_t)o * K + kk] = v - hf;
            }
        float *dhi, *dlo;
        if ((rc = upload(mem, hi, &dhi)) || (rc = upload(mem, lo, &dlo))) return rc;
        s.hi = dhi;
        s.lo = dlo;
    }
    const CUtensorMapDataType dt = f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    const uint64_t dims[2] = {(uint64_t)K, (uint64_t)cout};
    const uint64_t strides[1] = {(uint64_t)K * (f16 ? sizeof(uint16_t) : sizeof(float))};
    for (int i = 0; i < 2; ++i) {
        const uint32_t rows = 64u << i;
        if (cout % rows != 0) continue;
        const uint32_t box[2] = {(uint32_t)(f16 ? kBfBK : kTcBK), rows};
        if ((rc = make_tensor_map(&s.map_hi[i], dt, 2, s.hi, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
        if ((rc = make_tensor_map(&s.map_lo[i], dt, 2, s.lo, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
    }
    s.ok = true;
    return kOk;
}

struct HostWeights {   // folded fp32 weights [K][cout] and bias [cout] (empty without BN)
    std::vector<float> wt, bias;
};

// Reads conv weight [cout][cin][k][k] (+ optional BN gamma, beta, mean, var) and uploads the folded tensors: transposed for the
// SIMT kernel and, where eligible, split for both tensor-core arithmetics.  Fold: y = (conv - mean) / sqrt(var + 1e-5) * gamma + beta
// (net/resnet50.py:11-14).  `host`, if given, receives the folded weights for the callers that repack them.
static int read_conv(DeviceAllocs& mem, Reader& rd, Conv& c, int cin, int cout, int k, int stride, int pad, bool bn,
                     HostWeights* host = nullptr) {
    c.cin = cin; c.cout = cout; c.k = k; c.stride = stride; c.pad = pad;
    const size_t nw = (size_t)cout * cin * k * k;
    const float* w = rd.take(nw);
    const float *ga = nullptr, *be = nullptr, *mu = nullptr, *va = nullptr;
    if (bn) {
        ga = rd.take(cout); be = rd.take(cout); mu = rd.take(cout); va = rd.take(cout);
    }
    if (!rd.ok) return fail(kBadArg, "parameter blob too short (conv %dx%d k%d)", cin, cout, k);
    std::vector<float> wt(nw), bias;
    std::vector<double> scale(cout, 1.0);
    if (bn) {
        bias.resize(cout);
        for (int o = 0; o < cout; ++o) {
            scale[o] = (double)ga[o] / std::sqrt((double)va[o] + 1e-5);
            bias[o] = (float)((double)be[o] - (double)mu[o] * scale[o]);
        }
    }
    for (int o = 0; o < cout; ++o)
        for (int ci = 0; ci < cin; ++ci)
            for (int r = 0; r < k; ++r)
                for (int s = 0; s < k; ++s)
                    wt[((size_t)(r * k + s) * cin + ci) * cout + o] = (float)((double)w[(((size_t)o * cin + ci) * k + r) * k + s] * scale[o]);
    int rc = upload(mem, wt, &c.wt);
    if (rc) return rc;
    if (bn && (rc = upload(mem, bias, &c.bias))) return rc;
    const size_t K = (size_t)k * k * cin;
    if (split_eligible(cin, cout, k, stride, kBfBK) && (rc = pack_split(mem, true, wt.data(), K, cout, c.f16))) return rc;
    if (split_eligible(cin, cout, k, stride, kTcBK) && (rc = pack_split(mem, false, wt.data(), K, cout, c.tf32))) return rc;
    if (host) {
        host->wt = std::move(wt);
        host->bias = std::move(bias);
    }
    return kOk;
}

static int read_vec(DeviceAllocs& mem, Reader& rd, size_t n, float** out) {
    const float* p = rd.take(n);
    if (!rd.ok) return fail(kBadArg, "parameter blob too short (vector of %zu)", n);
    return upload(mem, std::vector<float>(p, p + n), out);
}

// Splits the stem's folded 7x7x3 weights (wt [49*3][64] from read_conv) for the tensor-core kernel over the zero-haloed NHWC4 input:
// filter row r, tap t, channel ci at k = r*32 + t*4 + ci, tap 7 and channel 3 zero.  3xTF32: K = 7 rows x 32 = 224, one filter row
// per k-block; f16x3: K = 8 rows x 32 = 256 (row 7 zero), four 64-wide k-blocks.
static int build_stem(DeviceAllocs& mem, Conv& c, const std::vector<float>& wt) {
    std::vector<float> rows((size_t)256 * 64, 0.f);
    for (int o = 0; o < 64; ++o)
        for (int r = 0; r < 7; ++r)
            for (int t = 0; t < 7; ++t)
                for (int ci = 0; ci < 3; ++ci)
                    rows[(size_t)(r * 32 + t * 4 + ci) * 64 + o] = wt[((size_t)(r * 7 + t) * 3 + ci) * 64 + o];
    int rc = pack_split(mem, false, rows.data(), 224, 64, c.tf32);
    if (rc) return rc;
    return pack_split(mem, true, rows.data(), 256, 64, c.f16);
}

// The fused conv3 + projection shortcut reads both inputs in whole f16x3 k-blocks
static bool c3ds_eligible(int planes, int cin, int stride) {
    return split_eligible(planes, 4 * planes, 1, 1, kBfBK) && split_eligible(cin, 4 * planes, 1, stride, kBfBK);
}

// f16x3 mode: conv3 and the projection shortcut of a first block (blk.c3 and blk.ds read with BN, h3 and hds their folded host
// weights) as one K-concatenated 1x1 conv; blk.has_c3ds says whether it was eligible
static int build_c3ds(DeviceAllocs& mem, Block& blk, const HostWeights& h3, const HostWeights& hds) {
    const int planes = blk.c3.cin, cin = blk.ds.cin, cout = blk.c3.cout;
    blk.has_c3ds = false;
    if (!c3ds_eligible(planes, cin, blk.ds.stride)) return kOk;
    Conv& f = blk.c3ds;
    f.cin = planes + cin; f.cout = cout; f.k = 1; f.stride = 1; f.pad = 0;
    std::vector<float> wt(h3.wt), bias(cout);
    wt.insert(wt.end(), hds.wt.begin(), hds.wt.end());
    for (int o = 0; o < cout; ++o) bias[o] = h3.bias[o] + hds.bias[o];
    int rc;
    if ((rc = upload(mem, bias, &f.bias))) return rc;
    if ((rc = pack_split(mem, true, wt.data(), f.cin, cout, f.f16))) return rc;
    blk.has_c3ds = true;
    return kOk;
}

static int read_trunk(irn_net* net, Reader& rd) {
    HostWeights stem;
    int rc = read_conv(net->mem, rd, net->stem, 3, 64, 7, 2, 3, true, &stem);
    if (rc) return rc;
    if ((rc = build_stem(net->mem, net->stem, stem.wt))) return rc;
    int cin = 64;
    for (int l = 0; l < 4; ++l) {
        net->blocks[l].resize(kBlocks[l]);
        for (int b = 0; b < kBlocks[l]; ++b) {
            Block& blk = net->blocks[l][b];
            const int planes = kPlanes[l], stride = b == 0 ? kStrides[l] : 1;
            HostWeights h3, hds;
            if ((rc = read_conv(net->mem, rd, blk.c1, cin, planes, 1, 1, 0, true))) return rc;
            if ((rc = read_conv(net->mem, rd, blk.c2, planes, planes, 3, stride, 1, true))) return rc;   // stride on conv2 (net/resnet50.py:24)
            if ((rc = read_conv(net->mem, rd, blk.c3, planes, planes * 4, 1, 1, 0, true, &h3))) return rc;
            blk.has_ds = b == 0;
            if (blk.has_ds && (rc = read_conv(net->mem, rd, blk.ds, cin, planes * 4, 1, stride, 0, true, &hds))) return rc;
            if (blk.has_ds && (rc = build_c3ds(net->mem, blk, h3, hds))) return rc;
            cin = planes * 4;
        }
    }
    return kOk;
}

static int read_head(DeviceAllocs& mem, Reader& rd, Head& h, int cin, int cout, int groups, int up) {
    int rc = read_conv(mem, rd, h.conv, cin, cout, 1, 1, 0, false);
    if (rc) return rc;
    h.groups = groups;
    h.up = up;
    if ((rc = read_vec(mem, rd, cout, &h.gamma))) return rc;
    return read_vec(mem, rd, cout, &h.beta);
}

// ------------------------------------------------------------------ launch helpers
static inline int conv_out(int n, int k, int s, int p) { return (n + 2 * p - k) / s + 1; }

// Copies tap `id`'s tensor, n floats at src, into the caller's buffer when one is set (irn_net_set_tap); nothing otherwise
static int tap(const irn_net* net, int id, const float* src, size_t n, cudaStream_t st) {
    const irn_net::Tap& t = net->taps[id];
    if (!t.dst) return kOk;
    if (t.bytes < n * sizeof(float)) return fail(kBadArg, "tap %d: buffer of %zu bytes, the tensor has %zu", id, t.bytes, n * sizeof(float));
    IRN_CUDA(cudaMemcpyAsync(t.dst, src, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return kOk;
}

template <bool F16, int BN>
static int launch_wg(const TcMaps& maps, const TcArgs& a, cudaStream_t st) {
    using Cfg = WgCfg<F16, BN>;
    static DeviceOnce once;   // n_sm[] holds the number of co-resident CTAs of the device
    const int ds = once.slot();
    if (once.need(ds)) {
        IRN_CUDA(cudaFuncSetAttribute((conv_wg_kernel<F16, BN>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::kSmem));
        int dev = 0, n_sm = 0, per_sm = 0;
        IRN_CUDA(cudaGetDevice(&dev));
        IRN_CUDA(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
        IRN_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, conv_wg_kernel<F16, BN>, kWgThreads, Cfg::kSmem));
        if (per_sm < 1) return fail(kCudaError, "conv_wg_kernel: no CTA fits on an SM (%zu bytes of shared memory)", Cfg::kSmem);
        once.n_sm[ds] = n_sm * per_sm;
        once.done[ds] = true;
    }
    // persistent CTAs: each walks the work items (spatial tile x N tile) with stride gridDim.x
    const long long items = (long long)a.tiles_x * a.tiles_y * a.B * (a.Cout / BN);
    const long long grid = items < once.n_sm[ds] ? items : once.n_sm[ds];
    conv_wg_kernel<F16, BN><<<(unsigned)grid, kWgThreads, Cfg::kSmem, st>>>(maps, a);
    IRN_LAUNCH_CHECK(F16 ? "conv_wg_kernel<f16x3>" : "conv_wg_kernel<3xtf32>");
    return kOk;
}

static TcArgs conv_args(const Conv& c, int B, int Ho, int Wo, const float* residual, float* out, bool relu) {
    TcArgs a;
    a.bias = c.bias; a.residual = residual; a.out = out;
    a.B = B; a.Ho = Ho; a.Wo = Wo; a.Cout = c.cout; a.Cin = c.cin; a.ksize = c.k; a.stride = c.stride; a.pad = c.pad;
    a.relu = relu ? 1 : 0;
    a.tiles_x = (Wo + kTcTW - 1) / kTcTW;
    a.tiles_y = (Ho + kTcTH - 1) / kTcTH;
    return a;
}

// NHWC fp32 [B,H,W,cin] read as boxes {32 ch, 16 px, 8 rows, 1 image} of output pixels: element strides give stride-s sampling
static int act_map(CUtensorMap* m, const float* in, int B, int H, int W, int cin, int stride) {
    const uint64_t dims[4] = {(uint64_t)cin, (uint64_t)W, (uint64_t)H, (uint64_t)B};
    const uint64_t strides[3] = {(uint64_t)cin * 4, (uint64_t)W * cin * 4, (uint64_t)H * W * cin * 4};
    const uint32_t box[4] = {32u, (uint32_t)(kTcTW * stride), (uint32_t)(kTcTH * stride), 1};
    const uint32_t estr[4] = {1, (uint32_t)stride, (uint32_t)stride, 1};
    return make_tensor_map(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, in, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B, estr);
}

// Stem input x4 = zero-haloed NHWC4 [B, Hin+6, Win+8, 4]: dim0 = the 32 contiguous floats (8 px x 4 ch) of one filter-row window,
// dim1 = output column (windows overlap: stride 2 px = 32 B), dim2 = padded input row, dim3 = image
static int stem_map(CUtensorMap* m, const float* x4, int B, int Hin, int Win) {
    const int Hp = Hin + 6, Wp = Win + 8;
    const int Wo = conv_out(Win, 7, 2, 3);
    const uint64_t dims[4] = {32, (uint64_t)Wo, (uint64_t)Hp, (uint64_t)B};
    const uint64_t strides[3] = {32, (uint64_t)Wp * 16, (uint64_t)Hp * Wp * 16};
    const uint32_t box[4] = {32, (uint32_t)kTcTW, (uint32_t)(kTcTH * 2), 1};
    const uint32_t estr[4] = {1, 1, 2, 1};
    return make_tensor_map(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, x4, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B, estr);
}

// The tensor-core convolution in one arithmetic: weights `w` (f16x3 or 3xTF32 split, as `f16` says), activations through `act` and,
// for a K-concatenated conv (a.kb_split), `act2`; N tile 128 when it divides Cout, else 64
static int launch_tc(bool f16, const SplitWeights& w, const CUtensorMap& act, const CUtensorMap* act2, TcArgs a, cudaStream_t st) {
    const bool wide = a.Cout % 128 == 0;
    TcMaps maps;
    maps.a = act;
    maps.a2 = act2 ? *act2 : act;
    maps.b_hi = w.map_hi[wide ? 1 : 0];
    maps.b_lo = w.map_lo[wide ? 1 : 0];
    a.oscale = f16 ? w.oscale : nullptr;
    if (f16) return wide ? launch_wg<true, 128>(maps, a, st) : launch_wg<true, 64>(maps, a, st);
    return wide ? launch_wg<false, 128>(maps, a, st) : launch_wg<false, 64>(maps, a, st);
}

// One conv in `mode` (as irn_net_set_conv_mode): the f16x3 or 3xTF32 tensor-core kernel where the conv is eligible, SIMT otherwise
static int run_conv(int mode, const Conv& c, const float* in, int B, int H, int W, const float* residual, float* out, bool relu,
                    cudaStream_t st, int* Ho_, int* Wo_) {
    ConvGeom g;
    g.B = B; g.H = H; g.W = W; g.Cin = c.cin;
    g.Ho = conv_out(H, c.k, c.stride, c.pad);
    g.Wo = conv_out(W, c.k, c.stride, c.pad);
    g.Cout = c.cout; g.k = c.k; g.stride = c.stride; g.pad = c.pad;
    if (Ho_) *Ho_ = g.Ho;
    if (Wo_) *Wo_ = g.Wo;
    const SplitWeights* sw = mode == 2 && c.f16.ok ? &c.f16 : mode >= 1 && c.tf32.ok ? &c.tf32 : nullptr;
    if (sw) {
        CUtensorMap act;
        int rc = act_map(&act, in, B, H, W, c.cin, c.stride);
        if (rc) return rc;
        return launch_tc(sw == &c.f16, *sw, act, nullptr, conv_args(c, B, g.Ho, g.Wo, residual, out, relu), st);
    }
    const int M = B * g.Ho * g.Wo;
    dim3 grid((M + kBM - 1) / kBM, (c.cout + kBN - 1) / kBN);
    if (c.cin % 16 == 0)
        conv_simt_kernel<true><<<grid, 256, 0, st>>>(in, c.wt, c.bias, residual, out, g, relu ? 1 : 0);
    else
        conv_simt_kernel<false><<<grid, 256, 0, st>>>(in, c.wt, c.bias, residual, out, g, relu ? 1 : 0);
    IRN_LAUNCH_CHECK("conv_simt_kernel");
    return kOk;
}

struct Arena {
    char* base;
    size_t size, off = 0;
    bool ok = true;
    float* take(size_t n_floats) {
        const size_t bytes = align_up(n_floats * sizeof(float), 256);
        if (off + bytes > size) {
            ok = false;
            return nullptr;
        }
        float* p = (float*)(base + off);
        off += bytes;
        return p;
    }
};

struct TrunkShapes {
    int H1, W1, H2, W2;          // after stem conv, after maxpool (= layer1 grid)
    int Hl[4], Wl[4];            // output grid of layer1..4
    size_t max_act;              // largest activation (floats) among stem out / block tensors
};

static TrunkShapes trunk_shapes(int B, int H, int W) {
    TrunkShapes s;
    s.H1 = conv_out(H, 7, 2, 3); s.W1 = conv_out(W, 7, 2, 3);
    s.H2 = conv_out(s.H1, 3, 2, 1); s.W2 = conv_out(s.W1, 3, 2, 1);
    int h = s.H2, w = s.W2;
    s.max_act = (size_t)B * s.H1 * s.W1 * 64;
    for (int l = 0; l < 4; ++l) {
        // conv1 of the first block still runs on the incoming grid with `planes` channels
        s.max_act = std::max(s.max_act, (size_t)B * h * w * kPlanes[l]);
        h = conv_out(h, 3, kStrides[l], 1);
        w = conv_out(w, 3, kStrides[l], 1);
        s.Hl[l] = h; s.Wl[l] = w;
        s.max_act = std::max(s.max_act, (size_t)B * h * w * kPlanes[l] * 4);
    }
    return s;
}

// conv3 + projection shortcut in one reduction (Block::c3ds): out = relu([W3 | Wds] . [t2 ; x sampled at the block's stride] + b3 + bds),
// x NHWC on the block's input grid h x w, t2 and out on its output grid ho x wo
static int run_c3ds(const Block& blk, const float* t2, const float* x, int B, int h, int w, int ho, int wo, float* out, cudaStream_t st) {
    const Conv& f = blk.c3ds;
    const int cin1 = f.cin - blk.ds.cin;   // channels of t2
    CUtensorMap act, act2;
    int rc = act_map(&act, t2, B, ho, wo, cin1, f.stride);
    if (rc) return rc;
    if ((rc = act_map(&act2, x, B, h, w, blk.ds.cin, blk.ds.stride))) return rc;
    TcArgs a = conv_args(f, B, ho, wo, nullptr, out, true);
    a.kb_split = cin1 / kBfBK;
    a.stride2 = blk.ds.stride;
    return launch_tc(true, f.f16, act, &act2, a, st);
}

// floats of the zero-haloed NHWC4 stem input of the tensor-core stems, the larger of run_stem's two input layouts
static size_t stem_halo_floats(int B, int Hin, int Win) { return (size_t)B * (Hin + 6) * (Win + 8) * 4; }

// floats of run_stem's input buffer x_in: the zero-haloed NHWC4 layout for the tensor-core stems, plain NHWC otherwise
static size_t stem_input_floats(int mode, int B, int Hin, int Win) {
    return mode >= 1 ? stem_halo_floats(B, Hin, Win) : (size_t)B * Hin * Win * 3;
}

// The stem's conv 7x7/s2 + bias + ReLU in `mode` on x_in, already laid out as stem_input_floats says for an Hin x Win input ->
// out NHWC [B, conv_out(Hin, 7, 2, 3), conv_out(Win, 7, 2, 3), 64]
static int run_stem_conv(int mode, const Conv& c, int B, int Hin, int Win, float* x_in, float* out, cudaStream_t st) {
    if (mode >= 1) {
        CUtensorMap act;
        int rc = stem_map(&act, x_in, B, Hin, Win);
        if (rc) return rc;
        TcArgs a = conv_args(c, B, conv_out(Hin, 7, 2, 3), conv_out(Win, 7, 2, 3), nullptr, out, true);
        a.stem = 1;
        if (mode == 2) {   // f16x3: K = 8 filter rows x 32 = four 64-wide k-blocks
            a.Cin = 256; a.ksize = 1; a.pad = 0;
            return launch_tc(true, c.f16, act, nullptr, a, st);
        }
        a.Cin = 32;        // 3xTF32: one filter row of 8 taps x 4 channels per k-block
        return launch_tc(false, c.tf32, act, nullptr, a, st);
    }
    return run_conv(0, c, x_in, B, Hin, Win, nullptr, out, true, st, nullptr, nullptr);
}

// The stem (`c`, built by build_stem) in `mode`: x_nchw [B,3,H,W] zero-padded (logically) to Hin x Win is laid out in x_in
// (stem_input_floats), then conv 7x7/s2 + bias + ReLU -> out NHWC [B, conv_out(Hin, 7, 2, 3), conv_out(Win, 7, 2, 3), 64]
static int run_stem(int mode, const Conv& c, const float* x_nchw, int B, int H, int W, int Hin, int Win, float* x_in, float* out,
                    cudaStream_t st) {
    if (mode >= 1) {
        const size_t total = (size_t)B * (Hin + 6) * (Win + 8);
        nchw_to_nhwc4_halo_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x_nchw, (float4*)x_in, B, H, W, Hin + 6, Win + 8);
        IRN_LAUNCH_CHECK("nchw_to_nhwc4_halo_kernel");
    } else {
        const size_t total = (size_t)B * Hin * Win * 3;
        nchw_to_nhwc_pad_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x_nchw, x_in, B, 3, H, W, Hin, Win);
        IRN_LAUNCH_CHECK("nchw_to_nhwc_pad_kernel");
    }
    return run_stem_conv(mode, c, B, Hin, Win, x_in, out, st);
}

// A ragged batch of P decoded uint8 RGB images (device, packed; HOST offsets and sizes) for the EdgeDisplacement forward
struct RaggedBatch {
    const uint8_t* img;
    const int64_t* off;     // host [P]: byte offset of image i
    const int32_t* hw;      // host [P][2]: H_i, W_i
    const float* lut;       // device [3][256] normalisation table (irn_normalize_lut)
    int P;
};

// Copies images i0 .. i0+n-1 of `rg` into a kernel parameter block
static RaggedChunk ragged_chunk(const RaggedBatch& rg, int i0, int n) {
    RaggedChunk c;
    for (int j = 0; j < n; ++j) {
        c.off[j] = rg.off[i0 + j];
        c.h[j] = rg.hw[2 * (i0 + j)];
        c.w[j] = rg.hw[2 * (i0 + j) + 1];
    }
    return c;
}

// The stem on a ragged batch: its images (and their W-flips) laid out straight into x_in on the Hin x Win canvas, then run_stem_conv.
// x_in holds what run_stem builds for the scale-1.0 pyramid of each image, byte for byte.
static int run_stem_ragged(int mode, const Conv& c, const RaggedBatch& rg, int Hin, int Win, float* x_in, float* out, cudaStream_t st) {
    const int Hp = mode >= 1 ? Hin + 6 : Hin, Wp = mode >= 1 ? Win + 8 : Win;
    for (int i0 = 0; i0 < rg.P; i0 += kRaggedChunk) {
        const int n = std::min(kRaggedChunk, rg.P - i0);
        const dim3 grid((unsigned)((Hp * Wp + 255) / 256), 2 * n);
        if (mode >= 1) {
            ragged_stem_input_kernel<true><<<grid, 256, 0, st>>>(rg.img, ragged_chunk(rg, i0, n), rg.lut, x_in, i0, Hp, Wp);
            IRN_LAUNCH_CHECK("ragged_stem_input_kernel<halo>");
        } else {
            ragged_stem_input_kernel<false><<<grid, 256, 0, st>>>(rg.img, ragged_chunk(rg, i0, n), rg.lut, x_in, i0, Hp, Wp);
            IRN_LAUNCH_CHECK("ragged_stem_input_kernel<nhwc>");
        }
    }
    return run_stem_conv(mode, c, 2 * rg.P, Hin, Win, x_in, out, st);
}

// Extent of a pair on the grid `levels` stride-2 operators below the input: every one maps an extent n at the origin to ceil(n/2)
static inline int level_extent(int n, int levels) { return ((n - 1) >> levels) + 1; }

// Zeroes what lies outside each pair's extent in x NHWC [2P,H,W,C], the grid `levels` stride-2 operators below the input
// (hw: HOST [P][2] input extents)
static int mask_outside(float* x, int H, int W, int C, const int32_t* hw, int P, int levels, cudaStream_t st) {
    for (int i0 = 0; i0 < P; i0 += kRaggedChunk) {
        const int n = std::min(kRaggedChunk, P - i0);
        PairExtents e;
        size_t most = 0;
        for (int j = 0; j < n; ++j) {
            e.h[j] = level_extent(hw[2 * (i0 + j)], levels);
            e.w[j] = level_extent(hw[2 * (i0 + j) + 1], levels);
            most = std::max(most, ((size_t)H * W - (size_t)e.h[j] * e.w[j]) * (C / 4));
        }
        if (most == 0) continue;   // every pair of the chunk fills the grid
        zero_outside_kernel<<<dim3((unsigned)((most + 255) / 256), 2 * n), 256, 0, st>>>(x, H, W, C, e, i0);
        IRN_LAUNCH_CHECK("zero_outside_kernel");
    }
    return kOk;
}

// Runs input layout transform + stem + maxpool + layer1..4 on x_nchw [B,3,H,W] zero-padded (logically) to Hin x Win, or, when `rg` is
// given, on its images and their flips (B = 2 rg->P) each zero-padded to Hin x Win.
// feats[0] = after maxpool (x1 of IRNet), feats[1..4] = layer outputs.  When `keep` is set every feats[i] lives in
// its own arena buffer (IRNet taps them); otherwise buffers rotate.
// `ext` (HOST [B/2][2], or null): pair p of x_nchw holds an image of ext[p] pixels at the top-left corner of the canvas and zeros
// elsewhere.  Then the stem's output and every block's conv1 output, the only tensors a spatial operator reads beyond an image's
// extent, are zeroed outside it (mask_outside), so each pair's features inside its extent are those of the pair alone.
static int run_trunk(const irn_net* net, const float* x_nchw, int B, int H, int W, int Hin, int Win, Arena& ar, bool keep,
                     const float* feats[5], TrunkShapes& sh, cudaStream_t st, const RaggedBatch* rg = nullptr,
                     const int32_t* ext = nullptr) {
    sh = trunk_shapes(B, Hin, Win);
    float* x_in = ar.take(stem_input_floats(net->conv_mode, B, Hin, Win));
    float* stem_out = ar.take((size_t)B * sh.H1 * sh.W1 * 64);
    float* pool_out = ar.take((size_t)B * sh.H2 * sh.W2 * 64);
    float* t1 = ar.take(sh.max_act);
    float* t2 = ar.take(sh.max_act);
    float* dsb = ar.take(sh.max_act);
    float* ping[2] = {ar.take(sh.max_act), ar.take(sh.max_act)};
    if (!ar.ok) return fail(kWorkspace, "network workspace too small");
    int rc = rg ? run_stem_ragged(net->conv_mode, net->stem, *rg, Hin, Win, x_in, stem_out, st)
                : run_stem(net->conv_mode, net->stem, x_nchw, B, H, W, Hin, Win, x_in, stem_out, st);
    if (rc) return rc;
    if (ext && (rc = mask_outside(stem_out, sh.H1, sh.W1, 64, ext, B / 2, 1, st))) return rc;
    if ((rc = tap(net, IRN_TAP_STEM, stem_out, (size_t)B * sh.H1 * sh.W1 * 64, st))) return rc;
    {
        const size_t total = (size_t)B * sh.H2 * sh.W2 * 16;
        maxpool3s2_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(stem_out, pool_out, B, sh.H1, sh.W1, 64, sh.H2, sh.W2);
        IRN_LAUNCH_CHECK("maxpool3s2_kernel");
    }
    if ((rc = tap(net, IRN_TAP_POOL, pool_out, (size_t)B * sh.H2 * sh.W2 * 64, st))) return rc;
    feats[0] = pool_out;
    const float* x = pool_out;
    int h = sh.H2, w = sh.W2, flip = 0, levels = 2;   // levels: stride-2 operators between the input and x
    int tj = IRN_TAP_BLOCK0;                           // the taps of the next block: t1, t2, output
    for (int l = 0; l < 4; ++l) {
        const int nb = (int)net->blocks[l].size();
        for (int b = 0; b < nb; ++b) {
            const Block& blk = net->blocks[l][b];
            int ho, wo;
            if ((rc = run_conv(net->conv_mode, blk.c1, x, B, h, w, nullptr, t1, true, st, nullptr, nullptr))) return rc;
            if (ext && (rc = mask_outside(t1, h, w, blk.c1.cout, ext, B / 2, levels, st))) return rc;   // conv2 reads one pixel beyond
            if ((rc = tap(net, tj, t1, (size_t)B * h * w * blk.c1.cout, st))) return rc;
            if ((rc = run_conv(net->conv_mode, blk.c2, t1, B, h, w, nullptr, t2, true, st, &ho, &wo))) return rc;
            if ((rc = tap(net, tj + 1, t2, (size_t)B * ho * wo * blk.c2.cout, st))) return rc;
            if (blk.c2.stride == 2) ++levels;
            const bool fused = net->conv_mode == 2 && blk.has_c3ds;
            const float* res = x;
            if (blk.has_ds && !fused) {
                if ((rc = run_conv(net->conv_mode, blk.ds, x, B, h, w, nullptr, dsb, false, st, nullptr, nullptr))) return rc;
                res = dsb;
            }
            float* out;
            if (keep && b == nb - 1) {   // IRNet taps every stage output: give it a buffer of its own
                out = ar.take((size_t)B * ho * wo * blk.c3.cout);
                if (!ar.ok) return fail(kWorkspace, "network workspace too small");
            } else {
                out = ping[flip];
                flip ^= 1;
            }
            if (fused) {
                if ((rc = run_c3ds(blk, t2, x, B, h, w, ho, wo, out, st))) return rc;
            } else if ((rc = run_conv(net->conv_mode, blk.c3, t2, B, ho, wo, res, out, true, st, nullptr, nullptr))) return rc;   // out += residual; relu (net/resnet50.py:51-52)
            if ((rc = tap(net, tj + 2, out, (size_t)B * ho * wo * blk.c3.cout, st))) return rc;
            tj += 3;
            x = out;
            h = ho;
            w = wo;
        }
        feats[l + 1] = x;
    }
    return kOk;
}

static size_t trunk_workspace_floats(int B, int H, int W, bool keep) {
    TrunkShapes s = trunk_shapes(B, H, W);
    size_t n = stem_halo_floats(B, H, W) + (size_t)B * s.H1 * s.W1 * 64 + (size_t)B * s.H2 * s.W2 * 64 + 5 * s.max_act;
    if (keep)
        for (int l = 0; l < 4; ++l) n += (size_t)B * s.Hl[l] * s.Wl[l] * kPlanes[l] * 4;
    return n + 64 * 32;   // alignment slack (256 B per buffer)
}

}  // namespace irn

using namespace irn;

// ---- single convolution as a plan of its own (unit tests / integration of other networks).  A handle is of one kind, set by the
// call that created it, and each forward call refuses the other kinds.
struct irn_conv {
    enum Kind { kConv, kStem, kShortcut } kind;
    irn::DeviceAllocs mem;
    irn::Conv conv;     // kConv; kStem: the stem with its repacked splits (build_stem)
    irn::Block block;   // kShortcut: c3, ds and the fused c3ds (build_c3ds)
    explicit irn_conv(Kind k) : kind(k) {}
};

extern "C" int irn_conv_create(const float* weight_oihw, const float* bn4 /* gamma,beta,mean,var or NULL */, int cin, int cout, int k,
                               int stride, int pad, irn_conv** out) {
    if (!weight_oihw || !out || cin <= 0 || cout <= 0 || k <= 0 || stride <= 0 || pad < 0) return fail(kBadArg, "irn_conv_create: bad argument");
    const size_t nw = (size_t)cout * cin * k * k;
    std::vector<float> blob(weight_oihw, weight_oihw + nw);
    if (bn4) blob.insert(blob.end(), bn4, bn4 + 4 * (size_t)cout);
    irn_conv* c = new irn_conv(irn_conv::kConv);
    Reader rd{blob.data(), blob.size()};
    int rc = read_conv(c->mem, rd, c->conv, cin, cout, k, stride, pad, bn4 != nullptr);
    if (rc) {
        delete c;
        return rc;
    }
    *out = c;
    return kOk;
}

extern "C" void irn_conv_destroy(irn_conv* c) { delete c; }

// The network's stem as a plan of its own, built and run by the same code as the trunk's (build_stem, run_stem)
extern "C" int irn_stem_create(const float* weight_oihw, const float* bn4, irn_conv** out) {
    if (!weight_oihw || !out) return fail(kBadArg, "irn_stem_create: bad argument");
    std::vector<float> blob(weight_oihw, weight_oihw + (size_t)64 * 3 * 7 * 7);
    if (bn4) blob.insert(blob.end(), bn4, bn4 + 4 * 64);
    irn_conv* c = new irn_conv(irn_conv::kStem);
    Reader rd{blob.data(), blob.size()};
    HostWeights host;
    int rc = read_conv(c->mem, rd, c->conv, 3, 64, 7, 2, 3, bn4 != nullptr, &host);
    if (!rc) rc = build_stem(c->mem, c->conv, host.wt);
    if (rc) {
        delete c;
        return rc;
    }
    *out = c;
    return kOk;
}

extern "C" size_t irn_stem_workspace_bytes(int B, int Hin, int Win) {
    if (B <= 0 || Hin <= 0 || Win <= 0) return 0;
    return stem_halo_floats(B, Hin, Win) * sizeof(float);   // the larger of the two stem_input_floats layouts
}

extern "C" int irn_stem_forward(irn_conv* c, const float* x_nchw, int B, int H, int W, int Hin, int Win, float* out_nhwc, int mode,
                                void* workspace, size_t workspace_bytes, irn_stream_t stream) {
    launch_counter() = 0;
    if (!c || c->kind != irn_conv::kStem) return fail(kBadArg, "irn_stem_forward: not a handle from irn_stem_create");
    if (!x_nchw || !out_nhwc || !workspace) return fail(kBadArg, "irn_stem_forward: bad argument");
    if (B <= 0 || H <= 0 || W <= 0 || H > Hin || W > Win)
        return fail(kBadArg, "irn_stem_forward: need B > 0 and 0 < H <= Hin, 0 < W <= Win; got B=%d H=%d W=%d Hin=%d Win=%d", B, H, W, Hin, Win);
    if (mode < 0 || mode > 2) return fail(kBadArg, "irn_stem_forward: mode must be 0, 1 or 2");
    if (((uintptr_t)workspace & 255) != 0) return fail(kBadArg, "irn_stem_forward: workspace must be 256-byte aligned");
    if (workspace_bytes < irn_stem_workspace_bytes(B, Hin, Win)) return fail(kWorkspace, "irn_stem_forward: workspace too small");
    return run_stem(mode, c->conv, x_nchw, B, H, W, Hin, Win, (float*)workspace, out_nhwc, (cudaStream_t)stream);
}

// conv3 + projection shortcut of a first bottleneck block as the f16x3 network runs them: one K-concatenated 1x1 conv (build_c3ds)
extern "C" int irn_shortcut_conv_create(const float* w3, const float* bn3, const float* wds, const float* bnds, int planes, int cin,
                                        int stride, irn_conv** out) {
    if (!w3 || !bn3 || !wds || !bnds || !out || planes <= 0 || cin <= 0 || !(stride == 1 || stride == 2))
        return fail(kBadArg, "irn_shortcut_conv_create: bad argument");
    if (!c3ds_eligible(planes, cin, stride))
        return fail(kUnsupported, "irn_shortcut_conv_create: the fused conv needs planes %% %d == 0 and cin %% %d == 0 (got %d, %d)", kBfBK,
                    kBfBK, planes, cin);
    const int cout = planes * 4;
    std::vector<float> b3(w3, w3 + (size_t)cout * planes), bd(wds, wds + (size_t)cout * cin);
    b3.insert(b3.end(), bn3, bn3 + 4 * (size_t)cout);
    bd.insert(bd.end(), bnds, bnds + 4 * (size_t)cout);
    irn_conv* c = new irn_conv(irn_conv::kShortcut);
    Block& blk = c->block;
    Reader r3{b3.data(), b3.size()}, rd{bd.data(), bd.size()};
    HostWeights h3, hds;
    int rc = read_conv(c->mem, r3, blk.c3, planes, cout, 1, 1, 0, true, &h3);
    if (!rc) rc = read_conv(c->mem, rd, blk.ds, cin, cout, 1, stride, 0, true, &hds);
    blk.has_ds = true;
    if (!rc) rc = build_c3ds(c->mem, blk, h3, hds);
    if (rc) {
        delete c;
        return rc;
    }
    *out = c;
    return kOk;
}

// relu(conv3(t2) + shortcut(x)): x NHWC [B,H,W,cin], t2 and out NHWC on the strided grid [B,Ho,Wo,planes | 4 planes]
extern "C" int irn_shortcut_conv_forward(irn_conv* c, const float* t2, const float* x, int B, int H, int W, float* out, irn_stream_t stream) {
    launch_counter() = 0;
    if (!c || c->kind != irn_conv::kShortcut) return fail(kBadArg, "irn_shortcut_conv_forward: not a handle from irn_shortcut_conv_create");
    if (!t2 || !x || !out || B <= 0 || H <= 0 || W <= 0) return fail(kBadArg, "irn_shortcut_conv_forward: bad argument");
    const Block& blk = c->block;
    return run_c3ds(blk, t2, x, B, H, W, conv_out(H, 1, blk.ds.stride, 0), conv_out(W, 1, blk.ds.stride, 0), out, (cudaStream_t)stream);
}

// in NHWC fp32 [B,H,W,cin] -> out NHWC [B,Ho,Wo,cout]; residual NHWC like out or NULL; mode as irn_net_set_conv_mode
extern "C" int irn_conv_forward(irn_conv* c, const float* in, int B, int H, int W, const float* residual, float* out, int relu, int mode,
                                irn_stream_t stream) {
    launch_counter() = 0;
    if (!c || c->kind != irn_conv::kConv) return fail(kBadArg, "irn_conv_forward: not a handle from irn_conv_create");
    if (!in || !out || B <= 0 || H <= 0 || W <= 0) return fail(kBadArg, "irn_conv_forward: bad argument");
    if (mode < 0 || mode > 2) return fail(kBadArg, "irn_conv_forward: mode must be 0, 1 or 2");
    const Conv& cv = c->conv;
    const int bk = mode == 2 ? kBfBK : kTcBK;
    if (mode >= 1 && !split_eligible(cv.cin, cv.cout, cv.k, cv.stride, bk))
        return fail(kUnsupported, "irn_conv_forward: this convolution is not eligible for the %s kernel (Cin %% %d, Cout %% 64, k in {1,3}, stride in {1,2})",
                    mode == 2 ? "f16x3" : "3xTF32", bk);
    return run_conv(mode, cv, in, B, H, W, residual, out, relu != 0, (cudaStream_t)stream, nullptr, nullptr);
}

extern "C" int irn_net_set_conv_mode(irn_net* net, int mode) {
    if (!net || mode < 0 || mode > 2) return fail(kBadArg, "irn_net_set_conv_mode: mode must be 0 (SIMT fp32), 1 (wgmma 3xTF32) or 2 (wgmma f16x3)");
    net->conv_mode = mode;
    return kOk;
}

extern "C" int irn_net_get_conv_mode(const irn_net* net) { return net ? net->conv_mode : -1; }

extern "C" int irn_net_set_tap(irn_net* net, int id, float* dst, size_t bytes) {
    if (!net || id < 0 || id >= IRN_TAP_COUNT || (net->kind == 0 && id > IRN_TAP_CAM_CLS))
        return fail(kBadArg, "irn_net_set_tap: no tap %d on this network", id);
    net->taps[id].dst = dst;
    net->taps[id].bytes = dst ? bytes : 0;
    return kOk;
}

extern "C" int irn_net_tap_shape(int kind, int id, int B, int H, int W, int crop_size, int shape[4]) {
    if (!shape || !(kind == 0 || kind == 1) || B <= 0) return fail(kBadArg, "irn_net_tap_shape: bad argument");
    if (kind == 1) H = W = crop_size;
    if (H <= 0 || W <= 0) return fail(kBadArg, "irn_net_tap_shape: bad input size %d x %d", H, W);
    const TrunkShapes s = trunk_shapes(B, H, W);
    int h = 0, w = 0, c = 0;
    if (id == IRN_TAP_STEM || id == IRN_TAP_POOL) {
        h = id == IRN_TAP_STEM ? s.H1 : s.H2;
        w = id == IRN_TAP_STEM ? s.W1 : s.W2;
        c = 64;
    } else if (id >= IRN_TAP_BLOCK0 && id < IRN_TAP_BLOCK0 + 48) {
        int j = (id - IRN_TAP_BLOCK0) / 3, l = 0;
        while (j >= kBlocks[l]) j -= kBlocks[l++];
        const int which = (id - IRN_TAP_BLOCK0) % 3;
        const bool in_grid = which == 0 && j == 0;   // conv1 of a stage's first block runs on the previous stage's grid
        h = in_grid ? (l ? s.Hl[l - 1] : s.H2) : s.Hl[l];
        w = in_grid ? (l ? s.Wl[l - 1] : s.W2) : s.Wl[l];
        c = which == 2 ? 4 * kPlanes[l] : kPlanes[l];
    } else if (kind == 0 && id == IRN_TAP_CAM_CLS) {
        h = s.Hl[3]; w = s.Wl[3]; c = 64;
    } else if (kind == 1 && id >= IRN_TAP_HEAD0 && id < IRN_TAP_COUNT) {
        // grid of each head's conv (edge1..5, dp1..7) and its channels; then ecat, dcat3, dcat2, dp7a, elog, dlog
        static const int lvl[18] = {0, 1, 2, 3, 3, 0, 1, 2, 3, 3, 2, 1, 1, 2, 1, 1, 1, 1};   // 0 = x1 grid, 1..3 = Hl[0..2]
        static const int ch[18] = {32, 32, 32, 32, 32, 64, 128, 256, 256, 256, 256, 256, 160, 768, 448, 256, 1, 2};
        const int i = id - IRN_TAP_HEAD0;
        h = lvl[i] ? s.Hl[lvl[i] - 1] : s.H2;
        w = lvl[i] ? s.Wl[lvl[i] - 1] : s.W2;
        c = ch[i];
    } else {
        return fail(kBadArg, "irn_net_tap_shape: no tap %d on a network of kind %d", id, kind);
    }
    shape[0] = B; shape[1] = h; shape[2] = w; shape[3] = c;
    return kOk;
}

extern "C" void irn_net_destroy(irn_net* net) { delete net; }

extern "C" int irn_cam_net_create(const float* params, size_t n_floats, irn_net** out) {
    if (!params || !out) return fail(kBadArg, "irn_cam_net_create: null pointer");
    irn_net* net = new irn_net();
    net->kind = 0;
    Reader rd{params, n_floats};
    int rc = read_trunk(net, rd);
    if (!rc) {
        const float* cw = rd.p;
        rc = read_vec(net->mem, rd, (size_t)20 * 2048, &net->classifier);
        if (!rc) {
            std::vector<float> padded((size_t)64 * 2048, 0.f);
            std::memcpy(padded.data(), cw, (size_t)20 * 2048 * sizeof(float));
            Reader r2{padded.data(), padded.size()};
            rc = read_conv(net->mem, r2, net->cls_conv, 2048, 64, 1, 1, 0, false);
        }
    }
    if (!rc && rd.left != 0) rc = fail(kBadArg, "irn_cam_net_create: %zu unread floats in the parameter blob", rd.left);
    if (rc) {
        irn_net_destroy(net);
        return rc;
    }
    *out = net;
    return kOk;
}

extern "C" int irn_irn_net_create(const float* params, size_t n_floats, irn_net** out) {
    if (!params || !out) return fail(kBadArg, "irn_irn_net_create: null pointer");
    irn_net* net = new irn_net();
    net->kind = 1;
    Reader rd{params, n_floats};
    int rc = read_trunk(net, rd);
    // heads in the order of net/resnet50_irn.py:23-93
    static const int e_cin[5] = {64, 256, 512, 1024, 2048}, e_up[5] = {1, 1, 2, 4, 4};
    for (int i = 0; i < 5 && !rc; ++i) rc = read_head(net->mem, rd, net->edge[i], e_cin[i], 32, 4, e_up[i]);
    if (!rc) rc = read_vec(net->mem, rd, 160, &net->edge6_w);
    if (!rc) rc = read_vec(net->mem, rd, 1, &net->edge6_b);
    static const int d_cin[7] = {64, 256, 512, 1024, 2048, 768, 448}, d_cout[7] = {64, 128, 256, 256, 256, 256, 256},
                     d_g[7] = {8, 16, 16, 16, 16, 16, 16}, d_up[7] = {1, 1, 1, 2, 2, 2, 1};
    for (int i = 0; i < 7 && !rc; ++i) rc = read_head(net->mem, rd, net->dp[i], d_cin[i], d_cout[i], d_g[i], d_up[i]);
    if (!rc) rc = read_vec(net->mem, rd, 2 * 256, &net->dp7_w);
    if (!rc) rc = read_vec(net->mem, rd, 2, &net->mean_shift);
    if (!rc && rd.left != 0) rc = fail(kBadArg, "irn_irn_net_create: %zu unread floats in the parameter blob", rd.left);
    if (rc) {
        irn_net_destroy(net);
        return rc;
    }
    *out = net;
    return kOk;
}

extern "C" size_t irn_cam_workspace_bytes(int B, int H, int W) {
    if (B <= 0 || (B & 1) || H <= 0 || W <= 0) return 0;
    const TrunkShapes sh = trunk_shapes(B, H, W);
    return (trunk_workspace_floats(B, H, W, false) + (size_t)B * sh.Hl[3] * sh.Wl[3] * 64 + 128) * sizeof(float);
}

// The CAM heads of a ragged batch (ext HOST [P][2] input extents): kernel(e, i0, n) launches the head of pairs i0 .. i0+n-1 with
// their extents on the CAM grid in e
template <class Launch>
static int ragged_heads(const int32_t* ext, int P, Launch kernel) {
    for (int i0 = 0; i0 < P; i0 += kRaggedChunk) {
        const int n = std::min(kRaggedChunk, P - i0);
        PairExtents e;
        for (int j = 0; j < n; ++j) {
            e.h[j] = level_extent(ext[2 * (i0 + j)], 4);
            e.w[j] = level_extent(ext[2 * (i0 + j) + 1], 4);
        }
        const int rc = kernel(e, i0, n);
        if (rc) return rc;
    }
    return kOk;
}

// CAM.forward for P = B/2 (image, flipped image) pairs of x NCHW fp32 [B,3,H,W] -> cam [P,20,ceil(H/16),ceil(W/16)].  With `ext`
// (HOST [P][2]), pair p is an image of ext[p] pixels at the top-left corner of the canvas, zero elsewhere (run_trunk): each pair's
// head flips within its own CAM width and writes 0 outside its CAM extent.
static int run_cam(const irn_net* net, const float* x_nchw, int B, int H, int W, const int32_t* ext, float* cam_out, Arena& ar,
                   cudaStream_t st) {
    const float* feats[5];
    TrunkShapes sh;
    int rc = run_trunk(net, x_nchw, B, H, W, H, W, ar, false, feats, sh, st, nullptr, ext);
    if (rc) return rc;
    const int P = B / 2, h = sh.Hl[3], w = sh.Wl[3];
    if (net->conv_mode >= 1 && net->cls_conv.tf32.ok) {
        // classifier as a 2048 -> 64 tensor-core conv with fused ReLU (the one-warp-per-pixel head re-reads the 160 KB weight
        // matrix per pixel), then flip-add + NHWC -> NCHW on the 20 real channels
        float* tmp = ar.take((size_t)B * h * w * 64);
        if (!ar.ok) return fail(kWorkspace, "irn_cam_forward: workspace too small");
        if ((rc = run_conv(net->conv_mode, net->cls_conv, feats[4], B, h, w, nullptr, tmp, true, st, nullptr, nullptr))) return rc;
        if ((rc = tap(net, IRN_TAP_CAM_CLS, tmp, (size_t)B * h * w * 64, st))) return rc;
        if (ext)
            return ragged_heads(ext, P, [&](const PairExtents& e, int i0, int n) -> int {
                cam_flip_add_ragged_kernel<<<dim3((unsigned)((20 * h * w + 255) / 256), n), 256, 0, st>>>(tmp, cam_out, h, w, 64, e, i0);
                IRN_LAUNCH_CHECK("cam_flip_add_ragged_kernel");
                return kOk;
            });
        const size_t total = (size_t)P * 20 * h * w;
        cam_flip_add_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(tmp, cam_out, P, h, w, 64);
        IRN_LAUNCH_CHECK("cam_flip_add_kernel");
        return kOk;
    }
    if (ext)
        return ragged_heads(ext, P, [&](const PairExtents& e, int i0, int n) -> int {
            cam_head_ragged_kernel<<<dim3((unsigned)((h * w * 32 + 255) / 256), n), 256, 0, st>>>(feats[4], net->classifier, cam_out, h, w,
                                                                                              2048, e, i0);
            IRN_LAUNCH_CHECK("cam_head_ragged_kernel");
            return kOk;
        });
    const size_t warps = (size_t)P * h * w;
    cam_head_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(feats[4], net->classifier, cam_out, P, h, w, 2048);
    IRN_LAUNCH_CHECK("cam_head_kernel");
    return kOk;
}

// CAM.forward for P = B/2 (image, flipped image) pairs: x NCHW fp32 [B,3,H,W] -> cam [P,20,ceil(H/16),ceil(W/16)]
extern "C" int irn_cam_forward(const irn_net* net, const float* x_nchw, int B, int H, int W, float* cam_out, void* workspace,
                               size_t workspace_bytes, irn_stream_t stream_) {
    launch_counter() = 0;
    if (!net || net->kind != 0 || !x_nchw || !cam_out || !workspace) return fail(kBadArg, "irn_cam_forward: bad argument");
    if (B <= 0 || (B & 1) || H <= 0 || W <= 0) return fail(kBadArg, "irn_cam_forward: B must be a positive even number (image + flipped image), got B=%d H=%d W=%d", B, H, W);
    if (((uintptr_t)workspace & 255) != 0) return fail(kBadArg, "irn_cam_forward: workspace must be 256-byte aligned");
    Arena ar{(char*)workspace, workspace_bytes};
    return run_cam(net, x_nchw, B, H, W, nullptr, cam_out, ar, (cudaStream_t)stream_);
}

static size_t irn_head_floats(int B, const TrunkShapes& s) {
    const size_t g2 = (size_t)B * s.Hl[0] * s.Wl[0];       // stride-4 grid (x1, x2)
    const size_t g3 = (size_t)B * s.Hl[1] * s.Wl[1];       // stride-8 grid (x3)
    size_t n = 0;
    n += g2 * 256;                 // raw conv output scratch (largest head conv: 256 ch on the stride-4 grid)
    n += g2 * 160;                 // edge concat
    n += g3 * 768;                 // dp3|dp4|dp5 concat
    n += g2 * 448;                 // dp1|dp2|dp_up3 concat
    n += g2 * 256;                 // dp7 activations
    n += g2 * 3;                   // edge logits + dp
    n += (size_t)B * 16 * 4 + 64;  // GN sums (fp64): B x (<= 16 groups, enforced in run_head) x (sum, sum of squares)
    return n + 64 * 16;
}

extern "C" size_t irn_edge_displacement_workspace_bytes(int P, int H, int W, int crop_size) {
    if (P <= 0 || H <= 0 || W <= 0 || H > crop_size || W > crop_size) return 0;
    const int B = 2 * P;
    TrunkShapes s = trunk_shapes(B, crop_size, crop_size);
    return (trunk_workspace_floats(B, crop_size, crop_size, true) + irn_head_floats(B, s) + 64) * sizeof(float);
}

// One head (conv1x1 -> GroupNorm -> upsample -> ReLU) into channels [coff, coff + cout) of dst; `id` is the tap of its raw conv output
static int run_head(const irn_net* net, int id, const Head& hd, const float* x, int B, int H, int W, float* raw, float* stats, float* dst, int Hd,
                    int Wd, int Cd, int coff, cudaStream_t st) {
    int rc = run_conv(net->conv_mode, hd.conv, x, B, H, W, nullptr, raw, false, st, nullptr, nullptr);
    if (rc) return rc;
    if ((rc = tap(net, id, raw, (size_t)B * H * W * hd.conv.cout, st))) return rc;
    if (hd.conv.cout > 256 || 256 % hd.conv.cout != 0 || hd.groups > 16) return fail(kUnsupported, "GroupNorm head with %d channels / %d groups", hd.conv.cout, hd.groups);
    IRN_CUDA(cudaMemsetAsync(stats, 0, (size_t)B * hd.groups * 2 * sizeof(double), st));
    {
        const int slices = std::max(1, std::min(256, (H * W) / 256));
        gn_partial_kernel<<<dim3(slices, B), 256, 0, st>>>(raw, (double*)stats, H * W, hd.conv.cout, hd.groups);
        IRN_LAUNCH_CHECK("gn_partial_kernel");
    }
    const size_t total = (size_t)B * Hd * Wd * (hd.conv.cout / 4);
    gn_up_relu_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(raw, (const double*)stats, hd.gamma, hd.beta, dst, B, H, W, hd.conv.cout, hd.groups,
                                                                      hd.up, Hd, Wd, Cd, coff);
    IRN_LAUNCH_CHECK("gn_up_relu_kernel");
    return kOk;
}

// Net.forward of IRNet (net/resnet50_irn.py:110-133) on B = 2P samples on the S x S canvas, from x_nchw [B,3,H,W] or the ragged batch
// `rg` (run_trunk): edge logits -> *elog NHWC [B,h2,w2,1], displacements -> *dlog NHWC [B,h2,w2,2] (both in the arena), h2 x w2 the
// stride-4 grid
static int run_irn(const irn_net* net, const float* x_nchw, const RaggedBatch* rg, int B, int H, int W, int S, Arena& ar, float** elog_,
                   float** dlog_, int* h2_, int* w2_, cudaStream_t st) {
    const float* f[5];
    TrunkShapes sh;
    int rc = run_trunk(net, x_nchw, B, H, W, S, S, ar, true, f, sh, st, rg);
    if (rc) return rc;
    const int h2 = sh.Hl[0], w2 = sh.Wl[0];   // stride 4 (x1, x2)
    const int h3 = sh.Hl[1], w3 = sh.Wl[1];   // stride 8 (x3)
    const int h4 = sh.Hl[2], w4 = sh.Wl[2];   // stride 16 (x4, x5)
    const size_t g2 = (size_t)B * h2 * w2, g3 = (size_t)B * h3 * w3;
    float* raw = ar.take(g2 * 256);
    float* ecat = ar.take(g2 * 160);
    float* dcat3 = ar.take(g3 * 768);
    float* dcat2 = ar.take(g2 * 448);
    float* dp7a = ar.take(g2 * 256);
    float* elog = ar.take(g2);
    float* dlog = ar.take(g2 * 2);
    float* stats = ar.take((size_t)B * 16 * 4 + 64);
    if (!ar.ok) return fail(kWorkspace, "irn_edge_displacement_forward: workspace too small");

    // edge branch (net/resnet50_irn.py:117-122): every map lands on the stride-4 grid, cropped to edge2's size
    const int eh[5] = {h2, h2, h3, h4, h4}, ew[5] = {w2, w2, w3, w4, w4};
    for (int i = 0; i < 5; ++i)
        if ((rc = run_head(net, IRN_TAP_HEAD0 + i, net->edge[i], f[i], B, eh[i], ew[i], raw, stats, ecat, h2, w2, 160, 32 * i, st))) return rc;
    if ((rc = tap(net, IRN_TAP_ECAT, ecat, g2 * 160, st))) return rc;
    conv1x1_smalln_kernel<1><<<(unsigned)((g2 * 32 + 255) / 256), 256, 0, st>>>(ecat, net->edge6_w, net->edge6_b, nullptr, elog, g2, 160);
    IRN_LAUNCH_CHECK("conv1x1_smalln_kernel<1>");
    if ((rc = tap(net, IRN_TAP_ELOG, elog, g2, st))) return rc;

    // displacement branch (net/resnet50_irn.py:124-131)
    const int d = IRN_TAP_HEAD0 + 5;
    if ((rc = run_head(net, d, net->dp[0], f[0], B, h2, w2, raw, stats, dcat2, h2, w2, 448, 0, st))) return rc;           // dp1 64
    if ((rc = run_head(net, d + 1, net->dp[1], f[1], B, h2, w2, raw, stats, dcat2, h2, w2, 448, 64, st))) return rc;      // dp2 128
    if ((rc = run_head(net, d + 2, net->dp[2], f[2], B, h3, w3, raw, stats, dcat3, h3, w3, 768, 0, st))) return rc;       // dp3
    if ((rc = run_head(net, d + 3, net->dp[3], f[3], B, h4, w4, raw, stats, dcat3, h3, w3, 768, 256, st))) return rc;     // dp4 up x2, crop to dp3
    if ((rc = run_head(net, d + 4, net->dp[4], f[4], B, h4, w4, raw, stats, dcat3, h3, w3, 768, 512, st))) return rc;     // dp5 up x2
    if ((rc = tap(net, IRN_TAP_DCAT3, dcat3, g3 * 768, st))) return rc;
    if ((rc = run_head(net, d + 5, net->dp[5], dcat3, B, h3, w3, raw, stats, dcat2, h2, w2, 448, 192, st))) return rc;    // dp6 up x2, crop to dp2
    if ((rc = tap(net, IRN_TAP_DCAT2, dcat2, g2 * 448, st))) return rc;
    if ((rc = run_head(net, d + 6, net->dp[6], dcat2, B, h2, w2, raw, stats, dp7a, h2, w2, 256, 0, st))) return rc;       // dp7 conv/GN/ReLU
    if ((rc = tap(net, IRN_TAP_DP7A, dp7a, g2 * 256, st))) return rc;
    conv1x1_smalln_kernel<2><<<(unsigned)((g2 * 32 + 255) / 256), 256, 0, st>>>(dp7a, net->dp7_w, nullptr, net->mean_shift, dlog, g2, 256);
    IRN_LAUNCH_CHECK("conv1x1_smalln_kernel<2>");
    if ((rc = tap(net, IRN_TAP_DLOG, dlog, g2 * 2, st))) return rc;
    *elog_ = elog;
    *dlog_ = dlog;
    *h2_ = h2;
    *w2_ = w2;
    return kOk;
}

// EdgeDisplacement.forward: x NCHW fp32 [2,3,H,W] (image, flipped image) -> edge [1,fh,fw], dp [2,fh,fw],
// fh = ceil(H/4), fw = ceil(W/4).  The input is zero-padded to crop_size x crop_size (net/resnet50_irn.py:226).
extern "C" int irn_edge_displacement_forward(const irn_net* net, const float* x_nchw, int P, int H, int W, int crop_size, float* edge_out,
                                             float* dp_out, void* workspace, size_t workspace_bytes, irn_stream_t stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    launch_counter() = 0;
    if (!net || net->kind != 1 || !x_nchw || !edge_out || !dp_out || !workspace) return fail(kBadArg, "irn_edge_displacement_forward: bad argument");
    if (P <= 0 || H <= 0 || W <= 0 || H > crop_size || W > crop_size || (crop_size % 16) != 0)
        return fail(kBadArg, "irn_edge_displacement_forward: need P > 0 and 0 < H,W <= crop_size (multiple of 16); got P=%d H=%d W=%d crop=%d", P, H, W, crop_size);
    if (((uintptr_t)workspace & 255) != 0) return fail(kBadArg, "irn_edge_displacement_forward: workspace must be 256-byte aligned");
    Arena ar{(char*)workspace, workspace_bytes};
    float *elog, *dlog;
    int h2, w2;
    int rc = run_irn(net, x_nchw, nullptr, 2 * P, H, W, crop_size, ar, &elog, &dlog, &h2, &w2, st);
    if (rc) return rc;
    const int fh = (H - 1) / 4 + 1, fw = (W - 1) / 4 + 1;
    edge_dp_tail_kernel<<<dim3((fh * fw + 255) / 256, P), 256, 0, st>>>(elog, dlog, edge_out, dp_out, h2, w2, fh, fw);
    IRN_LAUNCH_CHECK("edge_dp_tail_kernel");
    return kOk;
}

extern "C" size_t irn_edge_displacement_ragged_workspace_bytes(int P, int crop_size) {
    return irn_edge_displacement_workspace_bytes(P, crop_size, crop_size, crop_size);
}

// EdgeDisplacement.forward for P images of any sizes <= crop_size in one batch: every image (and its flip) runs on the zero-padded
// crop_size canvas, as the reference pads each one (net/resnet50_irn.py:226), so each image's ceil(H/4) x ceil(W/4) corner of the
// fc x fc output is what irn_edge_displacement_forward returns for it alone; outside it edge = 1, dp = 0.
extern "C" int irn_edge_displacement_forward_ragged(const irn_net* net, const uint8_t* img_u8, size_t img_bytes, const int64_t* img_offsets,
                                                    const int32_t* sizes_hw, int P, int crop_size, const float* lut768, float* edge_out,
                                                    float* dp_out, void* workspace, size_t workspace_bytes, irn_stream_t stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    launch_counter() = 0;
    const char* fn = "irn_edge_displacement_forward_ragged";
    if (!net || net->kind != 1 || !img_u8 || !img_offsets || !sizes_hw || !lut768 || !edge_out || !dp_out || !workspace)
        return fail(kBadArg, "%s: bad argument", fn);
    if (P <= 0 || crop_size <= 0 || (crop_size % 16) != 0)
        return fail(kBadArg, "%s: need P > 0 and crop_size a positive multiple of 16; got P=%d crop=%d", fn, P, crop_size);
    for (int i = 0; i < P; ++i) {
        const int H = sizes_hw[2 * i], W = sizes_hw[2 * i + 1];
        if (H <= 0 || W <= 0 || H > crop_size || W > crop_size)
            return fail(kBadArg, "%s: image %d is %dx%d, need 0 < H,W <= crop_size %d", fn, i, H, W, crop_size);
        const int64_t off = img_offsets[i];
        if (off < 0 || (uint64_t)off > img_bytes || img_bytes - (uint64_t)off < (uint64_t)H * W * 3)
            return fail(kBadArg, "%s: image %d (%dx%dx3 bytes at offset %lld) lies outside the %zu-byte image buffer", fn, i, H, W,
                        (long long)off, img_bytes);
    }
    if (!is_device_ptr(img_u8) || !is_device_ptr(lut768) || !is_device_ptr(edge_out) || !is_device_ptr(dp_out) || !is_device_ptr(workspace))
        return fail(kBadArg, "%s: images, table, outputs and workspace must be device memory", fn);
    if (((uintptr_t)workspace & 255) != 0) return fail(kBadArg, "%s: workspace must be 256-byte aligned", fn);
    if (workspace_bytes < irn_edge_displacement_ragged_workspace_bytes(P, crop_size)) return fail(kWorkspace, "%s: workspace too small", fn);
    const RaggedBatch rg{img_u8, img_offsets, sizes_hw, lut768, P};
    Arena ar{(char*)workspace, workspace_bytes};
    float *elog, *dlog;
    int h2, w2;
    int rc = run_irn(net, nullptr, &rg, 2 * P, crop_size, crop_size, crop_size, ar, &elog, &dlog, &h2, &w2, st);
    if (rc) return rc;
    const int fc = (crop_size - 1) / 4 + 1;
    for (int i0 = 0; i0 < P; i0 += kRaggedChunk) {
        const int n = std::min(kRaggedChunk, P - i0);
        edge_dp_tail_ragged_kernel<<<dim3((fc * fc + 255) / 256, n), 256, 0, st>>>(elog, dlog, edge_out, dp_out, h2, w2, fc,
                                                                                   ragged_chunk(rg, i0, n), i0);
        IRN_LAUNCH_CHECK("edge_dp_tail_ragged_kernel");
    }
    return kOk;
}

// CAM.forward for P = B/2 pairs of different sizes on one Hc x Wc canvas (irn_resize_ragged_forward lays it out): pair p holds an
// image of hw[p] pixels at the top-left corner and zeros elsewhere.  Pair p's ceil(h/16) x ceil(w/16) corner of cam_out equals what
// irn_cam_forward returns for that pair alone; the rest is 0.
extern "C" int irn_cam_forward_ragged(const irn_net* net, const float* x_canvas, int B, int Hc, int Wc, const int32_t* hw, float* cam_out,
                                      void* workspace, size_t workspace_bytes, irn_stream_t stream_) {
    launch_counter() = 0;
    const char* fn = "irn_cam_forward_ragged";
    if (!net || net->kind != 0 || !x_canvas || !hw || !cam_out || !workspace) return fail(kBadArg, "%s: bad argument", fn);
    if (B <= 0 || (B & 1) || Hc <= 0 || Wc <= 0)
        return fail(kBadArg, "%s: B must be a positive even number (image + flipped image), got B=%d Hc=%d Wc=%d", fn, B, Hc, Wc);
    if (is_device_ptr(hw)) return fail(kBadArg, "%s: the extents must be host memory", fn);
    for (int p = 0; p < B / 2; ++p)
        if (hw[2 * p] <= 0 || hw[2 * p + 1] <= 0 || hw[2 * p] > Hc || hw[2 * p + 1] > Wc)
            return fail(kBadArg, "%s: pair %d is %dx%d, need 0 < h <= %d and 0 < w <= %d", fn, p, hw[2 * p], hw[2 * p + 1], Hc, Wc);
    if (!is_device_ptr(x_canvas) || !is_device_ptr(cam_out) || !is_device_ptr(workspace))
        return fail(kBadArg, "%s: canvas, output and workspace must be device memory", fn);
    if (((uintptr_t)workspace & 255) != 0) return fail(kBadArg, "%s: workspace must be 256-byte aligned", fn);
    if (workspace_bytes < irn_cam_workspace_bytes(B, Hc, Wc)) return fail(kWorkspace, "%s: workspace too small", fn);
    Arena ar{(char*)workspace, workspace_bytes};
    return run_cam(net, x_canvas, B, Hc, Wc, hw, cam_out, ar, (cudaStream_t)stream_);
}
