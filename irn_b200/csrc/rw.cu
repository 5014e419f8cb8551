// R3-R6: edge -> affinity -> random walk, as a 69-tap stencil iterated on the device.
//
// Reference: misc/indexing.py:91-167.  The reference densifies the affinities to an (hw)^2
// matrix on the CPU, column-normalises it and squares it exp_times times.  Here the same
// operator  y_j <- (sum_i a_ij^beta y_i) / s_j ,  s_j = 1 + sum_i a_ij^beta  (A symmetric)
// is applied n_iter = 2^exp_times times with the 34 half-plane weights per pixel kept in
// fp32 and the state / accumulator in fp64 (SURVEY.md D3: fp32 state misses the 1e-4 bar).
//
// HBM layout (workspace), row pitch wp = round_up(w, 4) so every row is 16-byte aligned for TMA:
//   W[img][34][h][wp] fp32   a^beta per half-plane offset, 0 when the destination leaves the image
//   inv_s[img][h][wp] fp64   1 / (1 + sum of the 68 incident weights)
//   y[2][chan][h][wp] fp64   ping-pong walk state
#include <mutex>
#include <type_traits>

#include "common.h"
#include "path_tables.h"
#include "tma.cuh"

namespace irn {

// ---------------------------------------------------------------- device path tables
constexpr int kMaxDst = 160;    // radius 10 has 152 destinations
constexpr int kMaxPts = 2304;

struct DevTables {
    int n_dst;
    int radius;
    short plane[kMaxDst];        // internal W plane of destination k
    signed char dy[kMaxDst], dx[kMaxDst];
    short pstart[kMaxDst + 1];
    signed char py[kMaxPts], px[kMaxPts];
};
__constant__ DevTables c_tab;

static std::mutex g_tab_mutex;
static int g_tab_radius[64] = {0};   // per device: radius currently resident in c_tab
static int g_tab_ndst[64] = {0};

// Internal plane order for radius 5, grouped by |dx| so the step kernel can stream one |dx| class
// of planes at a time through shared memory:  class c holds dx=+c (dy = 0..maxdy; dy=0 only exists
// for dx>0) then dx=-c (dy = 1..maxdy).  Class sizes 4,9,9,7,5 = 34.
__host__ __device__ constexpr int cls_base5(int c) { return c == 0 ? 0 : c == 1 ? 4 : c == 2 ? 13 : c == 3 ? 22 : c == 4 ? 29 : 34; }
__host__ __device__ constexpr int cls_maxdy5(int c) { return c <= 2 ? 4 : c == 3 ? 3 : 2; }
__host__ __device__ constexpr int plane5(int dy, int dx) {
    const int c = dx < 0 ? -dx : dx;
    if (c > 4 || dy < 0 || dy > cls_maxdy5(c)) return -1;
    if (dx == 0) return dy >= 1 ? dy - 1 : -1;
    if (dx > 0) return cls_base5(c) + dy;
    return dy >= 1 ? cls_base5(c) + cls_maxdy5(c) + dy : -1;
}
static_assert(plane5(1, 0) == 0 && plane5(0, 1) == 4 && plane5(4, 1) == 8 && plane5(1, -1) == 9 && plane5(4, -1) == 12 &&
                  plane5(0, 2) == 13 && plane5(3, -3) == 28 && plane5(0, 4) == 29 && plane5(2, -4) == 33 && plane5(3, 4) == -1 &&
                  plane5(4, 3) == -1 && plane5(0, 0) == -1 && plane5(0, -1) == -1,
              "radius-5 plane order");

static int upload_tables(int radius, cudaStream_t stream, int* n_dst_out) {
    int dev = 0;
    IRN_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(g_tab_mutex);
    if (dev < 64 && g_tab_radius[dev] == radius) {
        if (n_dst_out) *n_dst_out = g_tab_ndst[dev];
        return kOk;
    }
    PathTable t = build_path_table(radius);
    if ((int)t.dst.size() > kMaxDst || (int)t.points.size() > kMaxPts)
        return fail(kUnsupported, "radius %d: %zu destinations / %zu path points exceed the device table", radius,
                    t.dst.size(), t.points.size());
    static DevTables h;   // guarded by g_tab_mutex
    h.n_dst = (int)t.dst.size();
    h.radius = radius;
    for (int k = 0; k < h.n_dst; ++k) {
        const int dy = t.dst[k].first, dx = t.dst[k].second;
        h.plane[k] = (short)(radius == 5 ? plane5(dy, dx) : k);
        h.dy[k] = (signed char)dy;
        h.dx[k] = (signed char)dx;
        h.pstart[k] = (short)t.path_start[k];
    }
    h.pstart[h.n_dst] = (short)t.path_start[h.n_dst];
    for (size_t j = 0; j < t.points.size(); ++j) {
        h.py[j] = (signed char)t.points[j].first;
        h.px[j] = (signed char)t.points[j].second;
    }
    // Kernels launched earlier on ANY stream may still be reading the previous radius' table: a radius change is rare
    // (the hot path only uses 5), so wait for the whole device before overwriting the symbol.
    IRN_CUDA(cudaDeviceSynchronize());
    IRN_CUDA(cudaMemcpyToSymbolAsync(c_tab, &h, sizeof(h), 0, cudaMemcpyHostToDevice, stream));
    IRN_CUDA(cudaStreamSynchronize(stream));   // `h` is reused; happens once per (device, radius)
    if (dev < 64) {
        g_tab_radius[dev] = radius;
        g_tab_ndst[dev] = h.n_dst;
    }
    if (n_dst_out) *n_dst_out = h.n_dst;
    return kOk;
}

// ---------------------------------------------------------------- affinity
__device__ __forceinline__ double pow_weight(float a, double beta, int ibeta) {
    double b = (double)a;
    if (ibeta > 0) {   // exact repeated squaring in fp64, rounded once to fp32 by the caller
        double r = 1.0;
        int e = ibeta;
        while (e) {
            if (e & 1) r *= b;
            b *= b;
            e >>= 1;
        }
        return r;
    }
    return pow(b, beta);
}

constexpr int kAffTX = 32, kAffTY = 8;

// MODE 0: write a^beta into the internal plane order, row pitch `pitch` (walk workspace)
// MODE 1: write a in reference destination order, dense rows (irn_edge_to_affinity)
template <int MODE>
__global__ void __launch_bounds__(kAffTX* kAffTY)
rw_affinity_kernel(const float* __restrict__ edge, float* __restrict__ out, int h, int w, int pitch, double beta, int ibeta) {
    extern __shared__ float s_edge[];   // [(TY + R) x (TX + 2R)], R = radius - 1
    const int R = c_tab.radius - 1;
    const int SW = kAffTX + 2 * R;
    const int tiles_x = (w + kAffTX - 1) / kAffTX;
    const int x0 = (blockIdx.x % tiles_x) * kAffTX, y0 = (blockIdx.x / tiles_x) * kAffTY;
    const int img = blockIdx.y;
    const float* e = edge + (size_t)img * h * w;
    const int n = (kAffTY + R) * SW;
    for (int i = threadIdx.y * kAffTX + threadIdx.x; i < n; i += kAffTX * kAffTY) {
        const int yy = y0 + i / SW, xx = x0 - R + i % SW;
        s_edge[i] = (yy < h && xx >= 0 && xx < w) ? e[(size_t)yy * w + xx] : 1.0f;   // pad value 1.0 (misc/indexing.py:150)
    }
    __syncthreads();
    const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
    if (x >= w || y >= h) return;
    const int n_dst = c_tab.n_dst;
    const size_t plane_sz = (size_t)h * pitch;
    float* o = out + (size_t)img * n_dst * plane_sz + (size_t)y * pitch + x;
    for (int k = 0; k < n_dst; ++k) {
        float m = 0.f;
        for (int j = c_tab.pstart[k]; j < c_tab.pstart[k + 1]; ++j)
            m = fmaxf(m, s_edge[(threadIdx.y + c_tab.py[j]) * SW + threadIdx.x + R + c_tab.px[j]]);
        const float a = 1.0f - m;   // misc/indexing.py:106
        if (MODE == 0)
            o[(size_t)c_tab.plane[k] * plane_sz] = (float)pow_weight(a, beta, ibeta);   // misc/indexing.py:133
        else
            o[(size_t)k * plane_sz] = a;
    }
}

// ---------------------------------------------------------------- training-side affinity (SURVEY.md 8(f) N4)
// AffinityDisplacementLoss.to_affinity (net/resnet50_irn.py:162-175): the same gather + max over path points as
// edge_to_affinity, on the cropped source window of PathIndex (rows [0, h-rf), columns [rf, w-rf): every path stays inside the
// image), output [n_img, n_dst, (h-rf)*(w-2rf)].  `arg` records which path point held the maximum -- the FIRST one in path
// order, like max_pool2d -- so that the backward pass can route the gradient the way autograd does through
// max_pool2d + index_select.
__global__ void __launch_bounds__(kAffTX* kAffTY)
aff_train_fwd_kernel(const float* __restrict__ edge, float* __restrict__ aff, int* __restrict__ arg, int h, int w) {
    extern __shared__ float s_edge[];   // [(TY + R) x (TX + 2R)], R = radius - 1
    const int R = c_tab.radius - 1;
    const int ch = h - R, cw = w - 2 * R;
    const int SW = kAffTX + 2 * R;
    const int tiles_x = (cw + kAffTX - 1) / kAffTX;
    const int x0 = (blockIdx.x % tiles_x) * kAffTX, y0 = (blockIdx.x / tiles_x) * kAffTY;   // window coordinates
    const int img = blockIdx.y;
    const float* e = edge + (size_t)img * h * w;
    const int n = (kAffTY + R) * SW;
    for (int i = threadIdx.y * kAffTX + threadIdx.x; i < n; i += kAffTX * kAffTY) {
        const int yy = y0 + i / SW, xx = x0 + i % SW;          // image column of window column c is c + R; the tile starts R to its left
        s_edge[i] = (yy < h && xx < w) ? e[(size_t)yy * w + xx] : 0.f;
    }
    __syncthreads();
    const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
    if (x >= cw || y >= ch) return;
    const int n_dst = c_tab.n_dst;
    const size_t n_src = (size_t)ch * cw;
    const size_t o = (size_t)img * n_dst * n_src + (size_t)y * cw + x;
    for (int k = 0; k < n_dst; ++k) {
        float m = -INFINITY;
        int at = 0;
        for (int j = c_tab.pstart[k]; j < c_tab.pstart[k + 1]; ++j) {
            const int py = c_tab.py[j], px = c_tab.px[j];
            const float v = s_edge[(threadIdx.y + py) * SW + threadIdx.x + R + px];
            if (v > m || v != v) {      // strictly greater: the first maximum wins; NaN propagates (max_pool2d)
                m = v;
                at = (y + py) * w + x + R + px;
            }
        }
        aff[o + (size_t)k * n_src] = 1.0f - m;   // net/resnet50_irn.py:171
        if (arg) arg[o + (size_t)k * n_src] = at;
    }
}

// d aff / d edge: aff = 1 - edge[arg]  ->  grad_edge[arg] -= grad_aff (index_select's backward is the same scatter-add)
__global__ void aff_train_bwd_kernel(const float* __restrict__ grad_aff, const int* __restrict__ arg, float* __restrict__ grad_edge,
                                     size_t per_img, size_t hw, size_t total) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const size_t img = i / per_img;
    atomicAdd(grad_edge + img * hw + arg[i], -grad_aff[i]);
}

// inv_s[p] = 1 / (1 + sum_k W_k(p) + sum_k W_k(p - d_k))      (misc/indexing.py:124,135)
__global__ void rw_rowsum_kernel(const float* __restrict__ W, double* __restrict__ inv_s, int h, int w, int pitch) {
    const int img = blockIdx.y;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= h * w) return;
    const int y = p / w, x = p % w;
    const int n_dst = c_tab.n_dst;
    const size_t plane_sz = (size_t)h * pitch;
    const float* Wi = W + (size_t)img * n_dst * plane_sz;
    double s = 1.0;
    for (int k = 0; k < n_dst; ++k) {
        const float* Wk = Wi + (size_t)c_tab.plane[k] * plane_sz;
        s += (double)Wk[y * pitch + x];
        const int yy = y - c_tab.dy[k], xx = x - c_tab.dx[k];
        if (yy >= 0 && xx >= 0 && xx < w) s += (double)Wk[yy * pitch + xx];
    }
    inv_s[(size_t)img * plane_sz + (size_t)y * pitch + x] = 1.0 / s;
}

// y0 = x * (1 - edge) in fp32 (misc/indexing.py:162), widened to fp64
__global__ void rw_init_kernel(const float* __restrict__ x, const float* __restrict__ edge, double* __restrict__ y,
                               const int* __restrict__ chan_off, int h, int w, int pitch) {
    const int img = blockIdx.y;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    const int hw = h * w;
    if (p >= hw) return;
    const int yy = p / w, xx = p % w;
    const float om = 1.0f - edge[(size_t)img * hw + p];
    for (int c = chan_off[img]; c < chan_off[img + 1]; ++c)
        y[((size_t)c * h + yy) * pitch + xx] = (double)__fmul_rn(x[(size_t)c * hw + p], om);
}

__global__ void rw_finish_kernel(const double* __restrict__ y, float* __restrict__ out, int totc, int h, int w, int pitch) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)totc * h * w) return;
    const int xx = (int)(i % w);
    const size_t row = i / w;   // c*h + y
    out[i] = (float)y[row * pitch + xx];
}

// ---------------------------------------------------------------- generic step (any radius; validation / fallback)
// One thread per pixel, all channels; bounds-checked global loads, tables in constant memory.
__global__ void rw_step_generic_kernel(const float* __restrict__ W, const double* __restrict__ inv_s,
                                       const double* __restrict__ yin, double* __restrict__ yout,
                                       const int* __restrict__ chan_off, int h, int w, int pitch) {
    const int img = blockIdx.y;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= h * w) return;
    const int y = p / w, x = p % w;
    const int n_dst = c_tab.n_dst;
    const size_t plane_sz = (size_t)h * pitch;
    const float* Wi = W + (size_t)img * n_dst * plane_sz;
    const double is = inv_s[(size_t)img * plane_sz + (size_t)y * pitch + x];
    for (int c = chan_off[img]; c < chan_off[img + 1]; ++c) {
        const double* yc = yin + (size_t)c * plane_sz;
        double acc = yc[y * pitch + x];
        for (int k = 0; k < n_dst; ++k) {
            const float* Wk = Wi + (size_t)c_tab.plane[k] * plane_sz;
            const int dy = c_tab.dy[k], dx = c_tab.dx[k];
            const int yf = y + dy, xf = x + dx;
            if (yf < h && xf >= 0 && xf < w) acc = fma((double)Wk[y * pitch + x], yc[yf * pitch + xf], acc);
            const int yb = y - dy, xb = x - dx;
            if (yb >= 0 && xb >= 0 && xb < w) acc = fma((double)Wk[yb * pitch + xb], yc[yb * pitch + xb], acc);
        }
        yout[(size_t)c * plane_sz + (size_t)y * pitch + x] = acc * is;
    }
}

// ---------------------------------------------------------------- TMA step (radius 5)
template <int B, int E, class F>
__device__ __forceinline__ void static_for(F&& f) {
    if constexpr (B < E) {
        f(std::integral_constant<int, B>{});
        static_for<B + 1, E>(f);
    }
}

constexpr int kR = 4;                 // stencil reach for radius 5
constexpr int kTX = 32;               // tile width = one warp
constexpr int kPY = 4;                // rows per thread (register window), in the step and the fused kernel
constexpr int kWarps = 4;
constexpr int kTY = kPY * kWarps;     // 16
constexpr int kSW = kTX + 2 * kR;     // 40 columns staged (x0-4 .. x0+35)
constexpr int kYH = kTY + 2 * kR;     // 24 state rows staged (y0-4 .. y0+19)
constexpr int kWH = kTY + kR;         // 20 weight rows staged (y0-4 .. y0+15): mirrored taps only look up / left
constexpr int kMaxClsPlanes = 9;
constexpr int kWBufFloats = kMaxClsPlanes * kWH * kSW;   // 7200 floats = 28.8 KB per buffer

// fp32 -> fp64 widening of a non-negative finite weight with three integer-pipe ops instead of F2F.F64.F32
// (measured: the 68 conversions per pixel per step were the kernel's bottleneck).  Exact for normal
// values; +0 and sub-normals (< 1.2e-38) map to <= 2^-126, i.e. they stay numerically zero.
__device__ __forceinline__ double widen_weight(float f) {
    const uint32_t u = __float_as_uint(f);
    return __hiloint2double((int)((u >> 3) + 0x38000000u), (int)(u << 29));
}

// One tap of the radius-5 stencil, all compile-time: |dx| class, column offset dxc of the state value, window row r (relative
// to the thread's first row), output row j and the internal weight plane k the tap reads.
template <int CLS, int DXC, int R, int J, int K>
struct Tap5 {
    static constexpr int cls = CLS, dxc = DXC, r = R, j = J, k = K;
};

struct NoHook {
    template <class T>
    __device__ __forceinline__ void operator()(T) const {}
};

// The 69-tap update of PY consecutive rows x NC channels of one column, accumulated into acc (which holds the diagonal term).
// For every column offset dxc and window row r the state value y(r, dxc, c) is read ONCE and used by every (row j, tap) pair
// it takes part in:
//   forward tap  d = (r-j, dxc):   weight W_d(p_j)                        w_fwd(Tap5)
//   mirrored tap d = (j-r, -dxc):  weight W_d(p_j - d) = W_d at the cell being read   w_mir(Tap5)
// Taps are applied in one fixed order -- class 0..4, sign + then -, r = -kR .. PY+kR-1, j = 0..PY-1, forward before mirrored
// -- so every kernel that walks through this helper produces bit-identical results.  enter(CLS) / leave(CLS) run around each
// |dx| class (the step kernel waits for and refills its weight buffers there).
template <int PY, int NC, class YRead, class WFwd, class WMir, class Enter = NoHook, class Leave = NoHook>
__device__ __forceinline__ void stencil69(double (&acc)[PY][NC], YRead&& y, WFwd&& w_fwd, WMir&& w_mir, Enter&& enter = Enter{},
                                          Leave&& leave = Leave{}) {
    static_for<0, 5>([&](auto CLS) {
        constexpr int cls = decltype(CLS)::value;
        enter(CLS);
        static_for<0, (cls == 0 ? 1 : 2)>([&](auto SGN) {
            constexpr int dxc = decltype(SGN)::value == 0 ? cls : -cls;
            static_for<-kR, PY + kR>([&](auto RR) {
                constexpr int r = decltype(RR)::value;
                double v[NC];   // static_for, not #pragma unroll: a one-trip loop (NC = 1) made the fused kernel ~3 % slower
                static_for<0, NC>([&](auto C) { v[C] = y(r, dxc, C); });
                static_for<0, PY>([&](auto JJ) {
                    constexpr int j = decltype(JJ)::value;
                    constexpr int dy = r - j;
                    constexpr int kf = plane5(dy, dxc);
                    constexpr int kb = plane5(-dy, -dxc);
                    if constexpr (kf >= 0) {
                        const double wv = widen_weight(w_fwd(Tap5<cls, dxc, r, j, kf>{}));
                        static_for<0, NC>([&](auto C) { acc[j][C] = fma(wv, v[C], acc[j][C]); });
                    } else if constexpr (kb >= 0) {
                        const double wv = widen_weight(w_mir(Tap5<cls, dxc, r, j, kb>{}));
                        static_for<0, NC>([&](auto C) { acc[j][C] = fma(wv, v[C], acc[j][C]); });
                    }
                });
            });
        });
        leave(CLS);
    });
}

constexpr size_t rw_tma_smem_bytes(int ch) {
    return 128 /*alignment slack*/ + (size_t)ch * kYH * kSW * sizeof(double) + 2 * (size_t)kWBufFloats * sizeof(float) + 64;
}

struct RwMaps {
    CUtensorMap w[5];   // weights, one map per |dx| class (box depth = class size)
    CUtensorMap y[4];   // state being read, box depth 1..4 channels
};

// One walk step for CH channels of one 32x16 tile.  Thread = one column, kPY consecutive rows; state tile in shared memory.
// The 34 weight planes stream through two shared-memory buffers one |dx| class at a time (TMA,
// zero-filled outside the image, which is exactly the reference's "affinity 0 to anything outside").
// One channel chunk (CH = 1..4 channels of one image) of one tile: issue the TMA loads, run the five |dx| classes, store.
template <int CH>
__device__ __forceinline__ void rw_chunk(const RwMaps& maps, const double* __restrict__ inv_s, double* __restrict__ yout, double* s_y,
                                         float* s_w, uint64_t* bars, uint32_t& ph_y, uint32_t (&ph_w)[2], int img, int c0,
                                         int c_end, int x0, int y0, int h, int w, int pitch) {
    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const int x = x0 + lane;
    const int ty0 = warp * kPY;
    const int yb = y0 + ty0;
    const size_t plane_sz = (size_t)h * pitch;
        if (tid == 0) {
            mbar_arrive_expect_tx(&bars[0], (uint32_t)(CH * kYH * kSW * sizeof(double)));
            tma_load_3d(s_y, &maps.y[CH - 1], &bars[0], x0 - kR, y0 - kR, c0);
            mbar_arrive_expect_tx(&bars[1], (uint32_t)((cls_base5(1) - cls_base5(0)) * kWH * kSW * sizeof(float)));
            tma_load_3d(s_w, &maps.w[0], &bars[1], x0 - kR, y0 - kR, img * 34 + cls_base5(0));
            mbar_arrive_expect_tx(&bars[2], (uint32_t)((cls_base5(2) - cls_base5(1)) * kWH * kSW * sizeof(float)));
            tma_load_3d(s_w + kWBufFloats, &maps.w[1], &bars[2], x0 - kR, y0 - kR, img * 34 + cls_base5(1));
            // (an L2 tensor prefetch of classes 2..4 at this point was measured 8 % SLOWER: 54.3 vs 50.2 us/step at C=2)
        }
        mbar_wait(&bars[0], ph_y);
        ph_y ^= 1;

        double acc[kPY][CH];
#pragma unroll
        for (int j = 0; j < kPY; ++j)
#pragma unroll
            for (int c = 0; c < CH; ++c) acc[j][c] = s_y[(c * kYH + ty0 + j + kR) * kSW + lane + kR];   // diagonal weight 1

        stencil69(
            acc, [&](int r, int dxc, int c) { return s_y[(c * kYH + ty0 + r + kR) * kSW + lane + dxc + kR]; },
            [&](auto t) {   // buffer cls & 1 holds the planes of class cls
                using T = decltype(t);
                const float* wb = s_w + (T::cls & 1) * kWBufFloats;
                return wb[((T::k - cls_base5(T::cls)) * kWH + ty0 + T::j + kR) * kSW + lane + kR];
            },
            [&](auto t) {
                using T = decltype(t);
                const float* wb = s_w + (T::cls & 1) * kWBufFloats;
                return wb[((T::k - cls_base5(T::cls)) * kWH + ty0 + T::r + kR) * kSW + lane + T::dxc + kR];
            },
            [&](auto CLS) {
                constexpr int buf = decltype(CLS)::value & 1;
                mbar_wait(&bars[1 + buf], ph_w[buf]);
                ph_w[buf] ^= 1;
            },
            [&](auto CLS) {
                constexpr int cls = decltype(CLS)::value, buf = cls & 1;
                if constexpr (cls + 2 <= 4) {
                    __syncthreads();   // every thread is done reading buffer `buf`: refill it with class cls + 2
                    if (tid == 0) {
                        uint64_t* bar = &bars[1 + buf];
                        mbar_arrive_expect_tx(bar, (uint32_t)((cls_base5(cls + 3) - cls_base5(cls + 2)) * kWH * kSW * sizeof(float)));
                        tma_load_3d(s_w + buf * kWBufFloats, &maps.w[cls + 2], bar, x0 - kR, y0 - kR, img * 34 + cls_base5(cls + 2));
                    }
                }
            });

        if (x < w) {
#pragma unroll
            for (int j = 0; j < kPY; ++j) {
                if (yb + j < h) {
                    const double is = inv_s[(size_t)img * plane_sz + (size_t)(yb + j) * pitch + x];
#pragma unroll
                    for (int c = 0; c < CH; ++c)
                        if (c0 + c < c_end) yout[(size_t)(c0 + c) * plane_sz + (size_t)(yb + j) * pitch + x] = acc[j][c] * is;
                }
            }
        }
}

// Grid (tiles, images).  MAXCH sizes the state buffer; every image is processed with exactly its own channel count (chunks of
// at most MAXCH), so a C=1 image in a mixed batch does not pay for the widest image's channels.
template <int MAXCH>
__global__ void __launch_bounds__(kTX* kWarps)
rw_step_tma_kernel(const __grid_constant__ RwMaps maps, const double* __restrict__ inv_s, double* __restrict__ yout,
                   const int* __restrict__ chan_off, int h, int w, int pitch) {
    extern __shared__ __align__(128) unsigned char smem_raw[];   // TMA destinations need 128-byte alignment
    double* s_y = (double*)smem_raw;                                                 // [<=MAXCH][kYH][kSW]
    float* s_w = (float*)(smem_raw + (size_t)MAXCH * kYH * kSW * sizeof(double));   // [2][<=9][kWH][kSW]
    uint64_t* bars = (uint64_t*)(s_w + 2 * kWBufFloats);                            // [0]=y, [1],[2]=weight buffers

    const int tid = threadIdx.x;
    const int tiles_x = (w + kTX - 1) / kTX;
    const int x0 = (blockIdx.x % tiles_x) * kTX, y0 = (blockIdx.x / tiles_x) * kTY;
    const int img = blockIdx.y;
    const int c_begin = chan_off[img], c_end = chan_off[img + 1];
    if (c_begin >= c_end) return;

    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        mbar_init(&bars[2], 1);
        fence_mbar_init();
    }
    __syncthreads();
    uint32_t ph_y = 0, ph_w[2] = {0, 0};
    int c0 = c_begin;
    while (c0 < c_end) {
        const int n = c_end - c0 < MAXCH ? c_end - c0 : MAXCH;
        if (MAXCH >= 4 && n == 4) rw_chunk<4>(maps, inv_s, yout, s_y, s_w, bars, ph_y, ph_w, img, c0, c_end, x0, y0, h, w, pitch);
        else if (MAXCH >= 3 && n == 3) rw_chunk<3>(maps, inv_s, yout, s_y, s_w, bars, ph_y, ph_w, img, c0, c_end, x0, y0, h, w, pitch);
        else if (MAXCH >= 2 && n == 2) rw_chunk<2>(maps, inv_s, yout, s_y, s_w, bars, ph_y, ph_w, img, c0, c_end, x0, y0, h, w, pitch);
        else rw_chunk<1>(maps, inv_s, yout, s_y, s_w, bars, ph_y, ph_w, img, c0, c_end, x0, y0, h, w, pitch);
        c0 += n;
        __syncthreads();   // s_y / weight buffers are reused by the next channel chunk
    }
}

// ---------------------------------------------------------------- fused walk (radius 5, h,w <= 128): the production path
// All n_iter steps of one (image, channel) in ONE launch, one thread-block cluster per item:
//   * the cluster's CTAs own 8 consecutive rows each (cluster size = smallest of 1,2,4,8,16 covering h); every CTA keeps the
//     34 weight planes of its rows -- plus, for plane (dy,dx), the dy rows above that its mirrored taps read -- resident in
//     shared memory for the whole walk: (34*8 + 68) rows x 128 fp32 = 170 KB, loaded from HBM ONCE per item instead of
//     once per step (the step kernel above re-reads 2.2 MB of weights per image per step);
//   * the fp64 state lives in a double-buffered 16 x 136 shared tile (8 own rows + 4 halo rows either side, 4 zero columns
//     either side); each step writes the new rows locally and pushes the boundary rows into the neighbour CTAs' halo rows
//     through distributed shared memory, then ONE cluster barrier publishes them;
//   * HBM traffic per item = weights + 1/s + seeds in, fp32 result out; nothing per step.
constexpr int kFR = 8;                       // rows per CTA
constexpr int kFW = 128;                     // widest supported grid = weight row pitch in shared memory
constexpr int kFYP = kFW + 2 * kR;           // 136: state row pitch
constexpr int kFYR = kFR + 2 * kR;           // 16 state rows
constexpr int kFThreads = (kFW / 32) * (kFR / kPY) * 32;   // 256: one column and kPY rows per thread
constexpr int kFRegPlanes = 16;              // planes whose forward-tap weights live in registers

__host__ __device__ constexpr int plane_dy5(int k) {   // dy of internal plane k (inverse of plane5)
    if (k < 4) return k + 1;
    for (int c = 1; c <= 4; ++c) {
        const int base = cls_base5(c), m = cls_maxdy5(c);
        if (k < base + m + 1) return k - base;           // dx = +c, dy = 0..m
        if (k < base + 2 * m + 1) return k - base - m;   // dx = -c, dy = 1..m
    }
    return 0;
}
__host__ __device__ constexpr int wrow_base5(int k) {   // first shared-memory row of plane k: it stores rows r0-dy .. r0+7
    int s = 0;
    for (int i = 0; i < k; ++i) s += kFR + plane_dy5(i);
    return s;
}
constexpr int kFWRows = wrow_base5(34);      // 340
static_assert(kFWRows == 340 && plane_dy5(plane5(3, -2)) == 3 && plane_dy5(plane5(0, 4)) == 0 && plane_dy5(plane5(4, 0)) == 4, "fused weight layout");
constexpr size_t kFusedWBytes = 16 + (size_t)kFWRows * kFW * sizeof(float) + 16;   // 16 B of zeros either side: column -4 / +131 reads
constexpr size_t kFusedSmem = kFusedWBytes + 2 * (size_t)kFYR * kFYP * sizeof(double);

__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ uint32_t cluster_nctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster address of `local_smem_addr` in CTA `rank` of this cluster
__device__ __forceinline__ uint32_t cluster_map(uint32_t local_smem_addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(rank));
    return r;
}
__device__ __forceinline__ void st_cluster_f64(uint32_t addr, double v) {
    asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(addr), "d"(v) : "memory");
}

__global__ void __launch_bounds__(kFThreads, 1)
rw_fused_kernel(const float* __restrict__ W, const double* __restrict__ inv_s, const float* __restrict__ x,
                const float* __restrict__ edge, float* __restrict__ out, const int* __restrict__ chan_off, int totc, int h, int w,
                int pitch, int n_iter) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* s_w = (float*)(smem_raw + 16);
    double* s_y = (double*)(smem_raw + kFusedWBytes);   // [2][kFYR][kFYP]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int rank = (int)cluster_ctarank(), csize = (int)cluster_nctarank();
    const int n_clusters = gridDim.x / csize, cid = blockIdx.x / csize;
    const int per = (totc + n_clusters - 1) / n_clusters;
    const int c_lo = cid * per, c_hi = c_lo + per < totc ? c_lo + per : totc;
    const int r0 = rank * kFR;
    const bool active = r0 < h;            // CTAs below the image only take part in the barriers
    const int col = (warp & 3) * 32 + lane;
    const int ty0 = (warp >> 2) * kPY;
    const size_t plane_sz = (size_t)h * pitch;
    const size_t hw = (size_t)h * w;

    // zero the pads and both state buffers once: halo rows outside the image, pad columns and rows >= h stay zero for good
    if (tid < 4) {
        ((float*)smem_raw)[tid] = 0.f;
        ((float*)(smem_raw + kFusedWBytes - 16))[tid] = 0.f;
    }
    for (int i = tid; i < 2 * kFYR * kFYP; i += kFThreads) s_y[i] = 0.0;
    __syncthreads();
    cluster_sync_all();                    // nobody pushes halo rows into a buffer that is still being zeroed

    const uint32_t sy_addr = smem_u32(s_y);
    const uint32_t up_addr = rank > 0 ? cluster_map(sy_addr, (uint32_t)(rank - 1)) : 0u;
    const uint32_t dn_addr = rank + 1 < csize ? cluster_map(sy_addr, (uint32_t)(rank + 1)) : 0u;

    int cur_img = -1;
    float wf[kPY][kFRegPlanes];
    for (int c = c_lo; c < c_hi; ++c) {
        int img = 0;
        while (chan_off[img + 1] <= c) ++img;
        double val[kPY], is[kPY];
        if (active) {
            if (img != cur_img) {          // (the last step's barrier ordered every read of the previous weights before this)
                const float* Wi = W + (size_t)img * 34 * plane_sz;
                static_for<0, 34>([&](auto K) {
                    constexpr int k = decltype(K)::value;
                    constexpr int dyk = plane_dy5(k);
                    constexpr int rows = kFR + dyk;
                    float* dst = s_w + (size_t)wrow_base5(k) * kFW;
                    const float* src = Wi + (size_t)k * plane_sz;
                    for (int i = tid; i < rows * (kFW / 4); i += kFThreads) {
                        const int lr = i / (kFW / 4), c4 = (i % (kFW / 4)) * 4;
                        const int gr = r0 - dyk + lr;
                        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (gr >= 0 && gr < h && c4 < w) {
                            v = __ldg(reinterpret_cast<const float4*>(src + (size_t)gr * pitch + c4));   // pitch % 4 == 0
                            if (c4 + 1 >= w) v.y = 0.f;    // the pitch padding is uninitialised workspace
                            if (c4 + 2 >= w) v.z = 0.f;
                            if (c4 + 3 >= w) v.w = 0.f;
                        }
                        *reinterpret_cast<float4*>(dst + lr * kFW + c4) = v;
                    }
                });
            }
            if (img != cur_img) {          // forward-tap weights of this thread's pixels stay in registers for the whole walk:
                __syncthreads();           // shared memory then serves only the mirrored taps (half of the weight reads)
                static_for<0, kFRegPlanes>([&](auto K) {
                    constexpr int k = decltype(K)::value;
#pragma unroll
                    for (int j = 0; j < kPY; ++j) wf[j][k] = s_w[(wrow_base5(k) + plane_dy5(k) + ty0 + j) * kFW + col];
                });
            }
#pragma unroll
            for (int j = 0; j < kPY; ++j) {
                const int gr = r0 + ty0 + j;
                const bool in = gr < h && col < w;
                is[j] = in ? inv_s[(size_t)img * plane_sz + (size_t)gr * pitch + col] : 0.0;
                // y0 = x * (1 - edge) in fp32 (misc/indexing.py:162), widened
                val[j] = in ? (double)__fmul_rn(x[(size_t)c * hw + (size_t)gr * w + col], 1.0f - edge[(size_t)img * hw + (size_t)gr * w + col]) : 0.0;
            }
        }
        cur_img = img;

        for (int t = 0; t <= n_iter; ++t) {
            // publish val (y_t) into buffer t&1: own rows locally, boundary rows into the neighbours' halo rows
            if (active) {
                const uint32_t boff = (uint32_t)((t & 1) * kFYR * kFYP * sizeof(double));
                double* sn = s_y + (t & 1) * kFYR * kFYP;
#pragma unroll
                for (int j = 0; j < kPY; ++j) {
                    const int lr = ty0 + j;
                    sn[(kR + lr) * kFYP + kR + col] = val[j];
                    if (lr < kR) {
                        if (rank > 0) st_cluster_f64(up_addr + boff + (uint32_t)(((kFR + kR + lr) * kFYP + kR + col) * sizeof(double)), val[j]);
                    }
                    if (lr >= kFR - kR) {
                        if (rank + 1 < csize) st_cluster_f64(dn_addr + boff + (uint32_t)(((lr - (kFR - kR)) * kFYP + kR + col) * sizeof(double)), val[j]);
                    }
                }
            }
            cluster_sync_all();
            if (t == n_iter) break;
            if (active) {
                const double* sy = s_y + (t & 1) * kFYR * kFYP;
                double acc[kPY][1];
#pragma unroll
                for (int j = 0; j < kPY; ++j) acc[j][0] = val[j];   // diagonal weight 1
                stencil69(
                    acc, [&](int r, int dxc, int) { return sy[(kR + ty0 + r) * kFYP + kR + col + dxc]; },
                    [&](auto t) {   // W_k at the pixel itself: the register copy, or plane k's row (own row + dy)
                        using T = decltype(t);
                        if constexpr (T::k < kFRegPlanes) return wf[T::j][T::k];
                        else return s_w[(wrow_base5(T::k) + (T::r - T::j) + ty0 + T::j) * kFW + col];
                    },
                    [&](auto t) {   // W_k at the pixel being read, (row ty0+r, col+dxc): plane k stores it in row ty0+j
                        using T = decltype(t);
                        return s_w[(wrow_base5(T::k) + ty0 + T::j) * kFW + col + T::dxc];
                    });
#pragma unroll
                for (int j = 0; j < kPY; ++j) val[j] = acc[j][0] * is[j];
            }
        }
        if (active) {
#pragma unroll
            for (int j = 0; j < kPY; ++j) {
                const int gr = r0 + ty0 + j;
                if (gr < h && col < w) out[(size_t)c * hw + (size_t)gr * w + col] = (float)val[j];
            }
        }
    }
    cluster_sync_all();   // no CTA exits while a neighbour may still push into its shared memory
}

// ---------------------------------------------------------------- workspace carving
struct RwWorkspace {
    float* W;
    double* inv_s;
    double* y[2];
    int* chan_off;
    int pitch;
    size_t bytes;
};

static RwWorkspace carve(void* base, int n_img, int h, int w, int totc, int n_dst) {
    RwWorkspace ws;
    ws.pitch = (w + 3) / 4 * 4;
    const size_t plane_sz = (size_t)h * ws.pitch;
    char* p = (char*)base;
    size_t off = 0;
    ws.W = (float*)(p + off);
    off += align_up((size_t)n_img * n_dst * plane_sz * sizeof(float), 256);
    ws.inv_s = (double*)(p + off);
    off += align_up((size_t)n_img * plane_sz * sizeof(double), 256);
    for (int i = 0; i < 2; ++i) {
        ws.y[i] = (double*)(p + off);
        off += align_up((size_t)totc * plane_sz * sizeof(double), 256);
    }
    ws.chan_off = (int*)(p + off);
    off += align_up((size_t)(n_img + 1) * sizeof(int), 256);
    ws.bytes = off;
    return ws;
}

template <int MODE>
static int launch_affinity(const float* edge, float* out, int n_img, int h, int w, int pitch, int radius, double beta, int ibeta,
                           cudaStream_t stream) {
    const int R = radius - 1;
    dim3 grid(((w + kAffTX - 1) / kAffTX) * ((h + kAffTY - 1) / kAffTY), n_img), block(kAffTX, kAffTY);
    const size_t smem = (size_t)(kAffTY + R) * (kAffTX + 2 * R) * sizeof(float);
    rw_affinity_kernel<MODE><<<grid, block, smem, stream>>>(edge, out, h, w, pitch, beta, ibeta);
    IRN_LAUNCH_CHECK(MODE == 0 ? "rw_affinity_kernel<0>" : "rw_affinity_kernel<1>");
    return kOk;
}

template <int CH>
static int launch_tma_steps(const RwWorkspace& ws, int n_img, int totc, int h, int w, int n_iter, cudaStream_t stream) {
    const int pitch = ws.pitch;
    RwMaps maps[2];
    for (int b = 0; b < 2; ++b) {
        for (int c = 0; c < 5; ++c) {
            const uint64_t dims[3] = {(uint64_t)w, (uint64_t)h, (uint64_t)n_img * 34};
            const uint64_t strides[2] = {(uint64_t)pitch * sizeof(float), (uint64_t)pitch * h * sizeof(float)};
            const uint32_t box[3] = {(uint32_t)kSW, (uint32_t)kWH, (uint32_t)(cls_base5(c + 1) - cls_base5(c))};
            int rc = make_tensor_map(&maps[b].w[c], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, ws.W, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE);
            if (rc) return rc;
        }
        const uint64_t dims[3] = {(uint64_t)w, (uint64_t)h, (uint64_t)totc};
        const uint64_t strides[2] = {(uint64_t)pitch * sizeof(double), (uint64_t)pitch * h * sizeof(double)};
        for (int d = 1; d <= 4; ++d) {
            const uint32_t box[3] = {(uint32_t)kSW, (uint32_t)kYH, (uint32_t)d};
            int rc = make_tensor_map(&maps[b].y[d - 1], CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 3, ws.y[b], dims, strides, box, CU_TENSOR_MAP_SWIZZLE_NONE);
            if (rc) return rc;
        }
    }
    // three 4-warp CTAs per SM, two weight buffers each (measured faster than a persistent one-CTA-per-SM TMA ring: 50 against
    // 67 us/step at C = 2)
    const size_t smem = rw_tma_smem_bytes(CH);
    static DeviceOnce once;
    const int ds = once.slot();
    if (once.need(ds)) {
        IRN_CUDA(cudaFuncSetAttribute(rw_step_tma_kernel<CH>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        once.done[ds] = true;
    }
    dim3 grid(((w + kTX - 1) / kTX) * ((h + kTY - 1) / kTY), n_img);
    for (int it = 0; it < n_iter; ++it) {
        rw_step_tma_kernel<CH><<<grid, kTX * kWarps, smem, stream>>>(maps[it & 1], ws.inv_s, ws.y[(it + 1) & 1], ws.chan_off, h, w, pitch);
        IRN_LAUNCH_CHECK("rw_step_tma_kernel");
    }
    return kOk;
}

// Launches the fused walk; *n_clusters = 0 (and nothing launched) when the device cannot co-schedule a cluster of the needed
// size.
static int launch_fused(const RwWorkspace& ws, const float* x, const float* edge, float* out, int totc, int h, int w, int n_iter,
                        cudaStream_t stream, int* n_clusters) {
    *n_clusters = 0;
    const int need = (h + kFR - 1) / kFR;
    int cs = 1;
    while (cs < need) cs *= 2;
    static DeviceOnce once;
    const int ds = once.slot();
    if (once.need(ds)) {
        IRN_CUDA(cudaFuncSetAttribute(rw_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFusedSmem));
        IRN_CUDA(cudaFuncSetAttribute(rw_fused_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
        once.done[ds] = true;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)cs);
    cfg.blockDim = dim3(kFThreads);
    cfg.dynamicSmemBytes = kFusedSmem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)cs;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int max_clusters = 0;
    if (cudaOccupancyMaxActiveClusters(&max_clusters, rw_fused_kernel, &cfg) != cudaSuccess || max_clusters <= 0) {
        cudaGetLastError();   // not an error of this call: the caller decides what runs instead
        return kOk;
    }
    const int n = totc < max_clusters ? totc : max_clusters;
    cfg.gridDim = dim3((unsigned)(n * cs));
    const float* Wp = ws.W;
    const double* isp = ws.inv_s;
    const int* cop = ws.chan_off;
    int pitch = ws.pitch;
    IRN_CUDA(cudaLaunchKernelEx(&cfg, rw_fused_kernel, Wp, isp, x, edge, out, cop, totc, h, w, pitch, n_iter));
    IRN_LAUNCH_CHECK("rw_fused_kernel");
    *n_clusters = n;
    return kOk;
}

enum class WalkPath { kFused, kTmaSteps, kGeneric };

// Which kernel walks the batch, decided on the host before any CUDA call, so that a variant that cannot run as asked is
// refused before anything is launched.
static int choose_path(int variant, int radius, int h, int w, int n_img, const int32_t* chan_offsets, WalkPath* path) {
    if (variant == 1 || (variant == 0 && radius != 5)) {
        *path = WalkPath::kGeneric;
        return kOk;
    }
    if (radius != 5) return fail(kUnsupported, "irn_random_walk_variant: variant %d needs radius 5, got %d", variant, radius);
    const bool fits = h <= kFR * 16 && w <= kFW;
    if (variant == 4 && !fits) return fail(kUnsupported, "irn_random_walk: fused walk needs h <= %d, w <= %d", kFR * 16, kFW);
    if (variant != 0 || !fits) {
        *path = variant == 4 ? WalkPath::kFused : WalkPath::kTmaSteps;
        return kOk;
    }
    // Both kernels give bit-identical results; pick the faster one from a cost model fitted to H100 measurements
    // (tools/rw_micro.py, variants 2 and 4, 128x128 grids, 1-4 classes per image): the fused kernel walks one (image, class)
    // per cluster at ~3.0 us per step on the 7 clusters of 16 CTAs that fit; the per-step kernel shares the weight reads
    // between up to 4 classes of an image (~1.13 + 0.22 C us per image-chunk per step, ~10 us per step at least).
    // Single-class images favour the fused kernel, large batches of many-class images (instance path: classes x
    // instances) the per-step one.
    double step_us = 0.0;
    for (int i = 0; i < n_img; ++i) {
        int c = chan_offsets[i + 1] - chan_offsets[i];
        for (; c > 0; c -= 4) step_us += 1.13 + 0.22 * (c < 4 ? c : 4);
    }
    step_us *= (double)h * w / (128.0 * 128.0);
    if (step_us < 10.0) step_us = 10.0;
    const double fused_us = 3.0 * ((chan_offsets[n_img] + 6) / 7);
    *path = fused_us <= step_us ? WalkPath::kFused : WalkPath::kTmaSteps;
    return kOk;
}

// Optional device timing of the step kernels (bench.py roofline): events recorded on the caller's stream around the
// n_iter step launches of the most recent walk on this thread.
static thread_local bool g_rw_timing = false;
static thread_local cudaEvent_t g_rw_ev[2] = {nullptr, nullptr};
static thread_local int g_rw_timed_iters = 0;
static thread_local int g_rw_last_fused = 0;   // clusters of the last fused launch, 0 = ran step by step

// Records timing event `which` when timing is on: 0 before the walk's step launches, 1 after its `iters` steps.
static int record_timing(int which, cudaStream_t stream, int iters = 0) {
    if (!g_rw_timing) return kOk;
    if (!g_rw_ev[0]) {
        IRN_CUDA(cudaEventCreate(&g_rw_ev[0]));
        IRN_CUDA(cudaEventCreate(&g_rw_ev[1]));
    }
    IRN_CUDA(cudaEventRecord(g_rw_ev[which], stream));
    if (which == 1) g_rw_timed_iters = iters;
    return kOk;
}

static int walk_impl(const float* x, const float* edge, float* out, int n_img, const int32_t* chan_offsets, int h, int w,
                     int radius, double beta, int n_iter, void* workspace, size_t workspace_bytes, int variant,
                     cudaStream_t stream) {
    launch_counter() = 0;
    if (variant != 0 && variant != 1 && variant != 2 && variant != 4)
        return fail(kBadArg, "irn_random_walk_variant: unknown variant %d (0, 1, 2 or 4)", variant);
    if (!x || !edge || !out || !chan_offsets || !workspace) return fail(kBadArg, "irn_random_walk: null pointer");
    if (n_img <= 0 || h <= 0 || w <= 0 || n_iter < 0)
        return fail(kBadArg, "irn_random_walk: bad size (n_img=%d h=%d w=%d n_iter=%d)", n_img, h, w, n_iter);
    if (radius < 2 || radius > 10) return fail(kUnsupported, "irn_random_walk: radius %d outside [2,10]", radius);
    if (chan_offsets[0] != 0) return fail(kBadArg, "irn_random_walk: chan_offsets[0] must be 0");
    int max_c = 0;
    for (int i = 0; i < n_img; ++i) {
        if (chan_offsets[i + 1] < chan_offsets[i]) return fail(kBadArg, "irn_random_walk: chan_offsets not monotone at %d", i);
        max_c = chan_offsets[i + 1] - chan_offsets[i] > max_c ? chan_offsets[i + 1] - chan_offsets[i] : max_c;
    }
    const int totc = chan_offsets[n_img];
    if (totc == 0) return kOk;
    WalkPath path;
    int rc = choose_path(variant, radius, h, w, n_img, chan_offsets, &path);
    if (rc) return rc;
    if (((uintptr_t)workspace & 255) != 0) return fail(kBadArg, "irn_random_walk: workspace must be 256-byte aligned");
    int n_dst = 0;
    rc = upload_tables(radius, stream, &n_dst);
    if (rc) return rc;
    RwWorkspace ws = carve(workspace, n_img, h, w, totc, n_dst);
    if (ws.bytes > workspace_bytes) return fail(kWorkspace, "irn_random_walk: workspace %zu < required %zu bytes", workspace_bytes, ws.bytes);
    if ((size_t)n_img * n_dst >= (1u << 30) || (size_t)h * ws.pitch >= (1u << 30)) return fail(kUnsupported, "irn_random_walk: problem too large");

    const int pitch = ws.pitch;
    const size_t hw = (size_t)h * w;
    IRN_CUDA(cudaMemcpyAsync(ws.chan_off, chan_offsets, (size_t)(n_img + 1) * sizeof(int), cudaMemcpyHostToDevice, stream));
    const double rb = nearbyint(beta);
    const int ibeta = (rb == beta && beta >= 1 && beta <= 64) ? (int)rb : 0;
    rc = launch_affinity<0>(edge, ws.W, n_img, h, w, pitch, radius, beta, ibeta, stream);
    if (rc) return rc;
    dim3 pgrid((unsigned)((hw + 255) / 256), n_img);
    rw_rowsum_kernel<<<pgrid, 256, 0, stream>>>(ws.W, ws.inv_s, h, w, pitch);
    IRN_LAUNCH_CHECK("rw_rowsum_kernel");

    if (path == WalkPath::kFused) {
        int n_clusters = 0;
        rc = record_timing(0, stream);
        if (!rc) rc = launch_fused(ws, x, edge, out, totc, h, w, n_iter, stream, &n_clusters);
        if (rc) return rc;
        if (n_clusters > 0) {
            g_rw_last_fused = n_clusters;
            return record_timing(1, stream, n_iter > 0 ? n_iter : 1);
        }
        if (variant == 4) return fail(kUnsupported, "irn_random_walk: the device cannot co-schedule the fused walk's cluster");
        path = WalkPath::kTmaSteps;   // variant 0: the per-step kernel takes over
    }
    g_rw_last_fused = 0;

    rw_init_kernel<<<pgrid, 256, 0, stream>>>(x, edge, ws.y[0], ws.chan_off, h, w, pitch);
    IRN_LAUNCH_CHECK("rw_init_kernel");
    rc = record_timing(0, stream);
    if (rc) return rc;
    if (path == WalkPath::kGeneric) {
        for (int it = 0; it < n_iter; ++it) {
            rw_step_generic_kernel<<<pgrid, 256, 0, stream>>>(ws.W, ws.inv_s, ws.y[it & 1], ws.y[(it + 1) & 1], ws.chan_off, h, w, pitch);
            IRN_LAUNCH_CHECK("rw_step_generic_kernel");
        }
    } else {
        const int ch = max_c >= 4 ? 4 : max_c;
        if (ch == 1) rc = launch_tma_steps<1>(ws, n_img, totc, h, w, n_iter, stream);
        else if (ch == 2) rc = launch_tma_steps<2>(ws, n_img, totc, h, w, n_iter, stream);
        else if (ch == 3) rc = launch_tma_steps<3>(ws, n_img, totc, h, w, n_iter, stream);
        else rc = launch_tma_steps<4>(ws, n_img, totc, h, w, n_iter, stream);
        if (rc) return rc;
    }
    rc = record_timing(1, stream, n_iter);
    if (rc) return rc;
    const size_t n = (size_t)totc * hw;
    rw_finish_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(ws.y[n_iter & 1], out, totc, h, w, pitch);
    IRN_LAUNCH_CHECK("rw_finish_kernel");
    return kOk;
}

}  // namespace irn

using namespace irn;

extern "C" int irn_edge_to_affinity(const float* edge, float* aff, int n_img, int h, int w, int radius,
                                    irn_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    launch_counter() = 0;
    if (!edge || !aff || n_img <= 0 || h <= 0 || w <= 0) return fail(kBadArg, "irn_edge_to_affinity: bad argument");
    if (radius < 2 || radius > 10) return fail(kUnsupported, "irn_edge_to_affinity: radius %d outside [2,10]", radius);
    int rc = upload_tables(radius, stream, nullptr);
    if (rc) return rc;
    return launch_affinity<1>(edge, aff, n_img, h, w, w, radius, 1.0, 1, stream);
}

extern "C" int irn_to_affinity_forward(const float* edge, float* aff, int32_t* arg, int n_img, int h, int w, int radius,
                                       irn_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    launch_counter() = 0;
    if (!edge || !aff || n_img <= 0 || h <= 0 || w <= 0) return fail(kBadArg, "irn_to_affinity_forward: bad argument");
    if (radius < 2 || radius > 10) return fail(kUnsupported, "irn_to_affinity_forward: radius %d outside [2,10]", radius);
    const int R = radius - 1;
    const int ch = h - R, cw = w - 2 * R;
    if (ch <= 0 || cw <= 0) return fail(kBadArg, "irn_to_affinity_forward: grid %dx%d too small for radius %d", h, w, radius);
    if ((size_t)h * w >= (1u << 31)) return fail(kUnsupported, "irn_to_affinity_forward: grid too large");
    int rc = upload_tables(radius, stream, nullptr);
    if (rc) return rc;
    dim3 grid(((cw + kAffTX - 1) / kAffTX) * ((ch + kAffTY - 1) / kAffTY), n_img), block(kAffTX, kAffTY);
    const size_t smem = (size_t)(kAffTY + R) * (kAffTX + 2 * R) * sizeof(float);
    aff_train_fwd_kernel<<<grid, block, smem, stream>>>(edge, aff, arg, h, w);
    IRN_LAUNCH_CHECK("aff_train_fwd_kernel");
    return kOk;
}

extern "C" int irn_to_affinity_backward(const float* grad_aff, const int32_t* arg, float* grad_edge, int n_img, int h, int w,
                                        int radius, irn_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    launch_counter() = 0;
    if (!grad_aff || !arg || !grad_edge || n_img <= 0 || h <= 0 || w <= 0) return fail(kBadArg, "irn_to_affinity_backward: bad argument");
    if (radius < 2 || radius > 10) return fail(kUnsupported, "irn_to_affinity_backward: radius %d outside [2,10]", radius);
    const int R = radius - 1;
    const int ch = h - R, cw = w - 2 * R;
    if (ch <= 0 || cw <= 0) return fail(kBadArg, "irn_to_affinity_backward: grid %dx%d too small for radius %d", h, w, radius);
    int n_dst = 0;
    int rc = upload_tables(radius, stream, &n_dst);
    if (rc) return rc;
    const size_t per_img = (size_t)n_dst * ch * cw, total = per_img * n_img;
    IRN_CUDA(cudaMemsetAsync(grad_edge, 0, (size_t)n_img * h * w * sizeof(float), stream));
    aff_train_bwd_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(grad_aff, arg, grad_edge, per_img, (size_t)h * w, total);
    IRN_LAUNCH_CHECK("aff_train_bwd_kernel");
    return kOk;
}

extern "C" size_t irn_rw_workspace_bytes(int n_img, int h, int w, int total_channels, int radius) {
    if (n_img <= 0 || h <= 0 || w <= 0 || total_channels < 0 || radius < 2 || radius > 10) return 0;
    const int n_dst = radius == 5 ? 34 : (int)build_path_table(radius).dst.size();
    return carve(nullptr, n_img, h, w, total_channels, n_dst).bytes;
}

extern "C" int irn_rw_last_launch_count(void) { return launch_counter(); }

extern "C" int irn_rw_last_was_fused(void) { return g_rw_last_fused; }

extern "C" int irn_rw_set_timing(int enable) {
    g_rw_timing = enable != 0;
    return kOk;
}

// Average duration (ms) of one step-kernel launch of the last timed walk on this thread; blocks until it finished.
extern "C" int irn_rw_last_step_ms(float* ms_per_step, int* n_steps) {
    if (!ms_per_step || !g_rw_ev[0] || g_rw_timed_iters <= 0) return fail(kBadArg, "irn_rw_last_step_ms: no timed walk (call irn_rw_set_timing(1) first)");
    IRN_CUDA(cudaEventSynchronize(g_rw_ev[1]));
    float ms = 0.f;
    IRN_CUDA(cudaEventElapsedTime(&ms, g_rw_ev[0], g_rw_ev[1]));
    *ms_per_step = ms / (float)g_rw_timed_iters;
    if (n_steps) *n_steps = g_rw_timed_iters;
    return kOk;
}

extern "C" int irn_random_walk(const float* x, const float* edge, float* out, int n_img, const int32_t* chan_offsets,
                               int h, int w, int radius, double beta, int n_iter, void* workspace,
                               size_t workspace_bytes, irn_stream_t stream) {
    return walk_impl(x, edge, out, n_img, chan_offsets, h, w, radius, beta, n_iter, workspace, workspace_bytes, 0, (cudaStream_t)stream);
}

// variant: 0 = production (radius 5: the fused cluster kernel or the per-step TMA kernel, by the cost model in choose_path;
// other radii: the generic kernel), 1 = generic bounds-checked kernel (validation), 2 = per-step TMA kernel (radius 5) or
// kUnsupported, 4 = fused cluster kernel or kUnsupported; any other value is kBadArg
extern "C" int irn_random_walk_variant(const float* x, const float* edge, float* out, int n_img, const int32_t* chan_offsets,
                                       int h, int w, int radius, double beta, int n_iter, void* workspace,
                                       size_t workspace_bytes, int variant, irn_stream_t stream) {
    return walk_impl(x, edge, out, n_img, chan_offsets, h, w, radius, beta, n_iter, workspace, workspace_bytes, variant, (cudaStream_t)stream);
}
