// N3: fully connected CRF (mean field on two permutohedral lattices) and the cam_to_ir_label step.
// Reference: misc/imutils.py:156-170 (crf_inference_label through pydensecrf) and step/cam_to_ir_label.py:19-41.
// The arithmetic is the one oracle/crf.py states (Kraehenbuehl & Koltun 2011; Adams, Baek & Davis 2010, section 3): every
// floating-point operation below is written with an explicit _rn intrinsic so that no contraction changes a rounding, and the
// lattice keys, splat order, blur and slice order are the oracle's.  No floating-point atomics: the same inputs give the same
// bits on every run.
//
// Per call (a batch of n images of one size, N = H*W pixels):
//   build  per lattice (Gaussian d=2 over (x,y)/sxy, bilateral d=5 over (x,y)/sxy,(r,g,b)/srgb):
//          crf_elevate (one thread per pixel: elevate, rank, barycentrics, d+1 packed 64-bit vertex keys), a stable radix sort
//          of the (key, pair) list of every image, a scan of the run heads (vertex ids), crf_mark (vertex -> first pair, pair ->
//          vertex: a CSR of pairs per vertex in ascending pixel order), crf_neighbours (2(d+1) binary searches per vertex);
//          then norm = 1/sqrt(L(1) + 1e-20).  One host synchronisation reads the vertex counts and the error word.
//   iterate  G CRFs per image (G = 2 for the step: the fg and bg label maps share the image's lattices) as G*n_labels value
//          channels, in blocks of 8: crf_splat (per-vertex gather), d+1 crf_blur passes, crf_slice (slice, * norm, * compat,
//          + (-U) or + the previous term), then crf_softmax.  U comes from the label map (two values per image), never stored.
//   tail   crf_final: argmax over labels (first maximum), and for the step keys[] + the fg/bg combination into 0 / class / 255.
#include <cub/cub.cuh>

#include <cmath>
#include <vector>

#include "common.h"

namespace irn {
namespace crf {

constexpr int kMaxLabels = 32;   // per CRF; VOC needs 21
constexpr int kCB = 8;           // value channels per pass through the lattice

struct ImgParam {
    int n_labels;                // labels of each of the image's G CRFs
    int cam_off;                 // step: first high_res plane of the image
    float pe, ne;                // -log(gt_prob), -log((1-gt_prob)/(n_labels-1))
    int keys[kMaxLabels];        // step: class id of each label (entry 0 = background)
};

struct Lat {                     // one lattice of a batch; pairs are (pixel, remainder) = p*(D+1)+r, global index i*P + pair
    int N, P;
    const float* w;              // [n*P] barycentric weight of each pair
    const int* pvert;            // [n*P] vertex of each pair
    const int* csr;              // [n*P] pairs sorted by vertex, ascending pixel within a vertex
    const int* vstart;           // [V+1] first csr position of each vertex
    const int* nbr;              // [V*(D+1)*2] blur neighbours (-1 = none)
    const float* norm;           // [n*N]
};

template <int D>
struct Scale {
    float s[D];
};

template <int D>
__device__ __forceinline__ bool pack_key(const int* k, unsigned long long& key) {
    constexpr int B = 64 / D;
    constexpr long long off = 1LL << (B - 1);
    key = 0;
    bool ok = true;
#pragma unroll
    for (int c = 0; c < D; ++c) {
        const long long b = (long long)k[c] + off;
        ok &= b >= 0 && b < (1LL << B);
        key |= (unsigned long long)(b & ((1LL << B) - 1)) << (B * c);
    }
    return ok;
}

template <int D>
__global__ void crf_elevate(const uint8_t* __restrict__ img, int n, int H, int W, float sxy, float srgb, Scale<D> sf,
                            unsigned long long* __restrict__ keys, int* __restrict__ pairs, float* __restrict__ wts,
                            int* __restrict__ err) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int N = H * W;
    if (idx >= (long long)n * N) return;
    const int p = (int)(idx % N), x = p % W, y = p / W;
    float f[D];
    f[0] = __fdiv_rn((float)x, sxy);
    f[1] = __fdiv_rn((float)y, sxy);
    if constexpr (D == 5) {
#pragma unroll
        for (int c = 0; c < 3; ++c) f[2 + c] = __fdiv_rn((float)img[idx * 3 + c], srgb);
    }
    // elevation onto sum x = 0 (Adams et al. 3.1)
    float E[D + 1];
    float sm = 0.f;
#pragma unroll
    for (int j = D; j >= 1; --j) {
        const float cf = __fmul_rn(f[j - 1], sf.s[j - 1]);
        E[j] = __fsub_rn(sm, __fmul_rn((float)j, cf));
        sm = __fadd_rn(sm, cf);
    }
    E[0] = sm;
    const float down = (float)(1.0 / (D + 1)), dp1 = (float)(D + 1);
    int rem0[D + 1], rank[D + 1];
    float diff[D + 1];
    int sum = 0;
#pragma unroll
    for (int i = 0; i <= D; ++i) {
        const float v = __fmul_rn(E[i], down);
        const float up = __fmul_rn(ceilf(v), dp1), dn = __fmul_rn(floorf(v), dp1);
        const float r = __fsub_rn(up, E[i]) < __fsub_rn(E[i], dn) ? up : dn;
        rem0[i] = (int)r;
        diff[i] = __fsub_rn(E[i], r);
        sum += rem0[i];
        rank[i] = 0;
    }
    sum /= D + 1;
#pragma unroll
    for (int i = 0; i <= D; ++i)
#pragma unroll
        for (int j = i + 1; j <= D; ++j) {
            if (diff[i] < diff[j]) ++rank[i];
            else ++rank[j];
        }
    if (sum > 0) {
#pragma unroll
        for (int i = 0; i <= D; ++i) {
            if (rank[i] >= D + 1 - sum) { rem0[i] -= D + 1; rank[i] += sum - (D + 1); }
            else rank[i] += sum;
        }
    } else if (sum < 0) {
#pragma unroll
        for (int i = 0; i <= D; ++i) {
            if (rank[i] < -sum) { rem0[i] += D + 1; rank[i] += D + 1 + sum; }
            else rank[i] += sum;
        }
    }
    float b[D + 2];
#pragma unroll
    for (int i = 0; i < D + 2; ++i) b[i] = 0.f;
#pragma unroll
    for (int i = 0; i <= D; ++i) {
        const float v = __fmul_rn(__fsub_rn(E[i], (float)rem0[i]), down);
        b[D - rank[i]] = __fadd_rn(b[D - rank[i]], v);
        b[D - rank[i] + 1] = __fsub_rn(b[D - rank[i] + 1], v);
    }
    b[0] = __fadd_rn(b[0], __fadd_rn(1.f, b[D + 1]));
    const long long base = idx * (D + 1);
    bool ok = true;
#pragma unroll
    for (int r = 0; r <= D; ++r) {
        int k[D];
#pragma unroll
        for (int c = 0; c < D; ++c) k[c] = rem0[c] + (rank[c] <= D - r ? r : r - (D + 1));
        unsigned long long key;
        ok &= pack_key<D>(k, key);
        keys[base + r] = key;
        pairs[base + r] = (int)(base + r);
        wts[base + r] = b[r];
    }
    if (!ok) atomicOr(err, 1);
}

__global__ void crf_heads(const unsigned long long* __restrict__ keys, long long total, int P, int* __restrict__ head) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= total) return;
    head[k] = (k % P == 0 || keys[k] != keys[k - 1]) ? 1 : 0;
}

__global__ void crf_mark(const unsigned long long* __restrict__ keys, const int* __restrict__ csr, const int* __restrict__ vid,
                         long long total, int P, int n, int* __restrict__ vstart, unsigned long long* __restrict__ vkey,
                         int* __restrict__ pvert, int* __restrict__ voff) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= total) return;
    const int v = vid[k] - 1;
    if (k % P == 0 || keys[k] != keys[k - 1]) {
        vstart[v] = (int)k;
        vkey[v] = keys[k];
    }
    pvert[csr[k]] = v;
    if (k % P == 0) voff[k / P] = v;
    if (k == total - 1) {
        vstart[v + 1] = (int)total;
        voff[n] = v + 1;
    }
}

template <int D>
__global__ void crf_neighbours(const unsigned long long* __restrict__ vkey, const int* __restrict__ vstart,
                               const int* __restrict__ csr, const int* __restrict__ voff, int V, int P, int* __restrict__ nbr) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    constexpr int B = 64 / D;
    const int img = csr[vstart[v]] / P;
    const int lo0 = voff[img], hi0 = voff[img + 1];
    const unsigned long long key = vkey[v];
    int c[D];
#pragma unroll
    for (int i = 0; i < D; ++i) c[i] = (int)((key >> (B * i)) & ((1ULL << B) - 1)) - (1 << (B - 1));
#pragma unroll
    for (int j = 0; j <= D; ++j) {
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            const int sign = s == 0 ? 1 : -1;
            int k[D];
#pragma unroll
            for (int i = 0; i < D; ++i) k[i] = c[i] - sign + (i == j ? sign * (D + 1) : 0);
            unsigned long long nk;
            int found = -1;
            if (pack_key<D>(k, nk)) {
                int lo = lo0, hi = hi0;
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (vkey[mid] < nk) lo = mid + 1;
                    else hi = mid;
                }
                if (lo < hi0 && vkey[lo] == nk) found = lo;
            }
            nbr[((long long)v * (D + 1) + j) * 2 + s] = found;
        }
    }
}

// splat: per vertex, sum over its pairs (ascending pixel) of w * (norm * Q) -- or of w * 1 when Q is null (the normaliser)
template <int D>
__global__ void crf_splat(Lat L, int V, const float* __restrict__ Q, int CP, int blk, int G, const ImgParam* __restrict__ prm,
                          float* __restrict__ out) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    const int k0 = L.vstart[v], k1 = L.vstart[v + 1];
    float acc[kCB];
#pragma unroll
    for (int c = 0; c < kCB; ++c) acc[c] = 0.f;
    if (Q == nullptr) {
        for (int k = k0; k < k1; ++k) acc[0] = __fadd_rn(acc[0], L.w[L.csr[k]]);
    } else {
        const int img = L.csr[k0] / L.P;
        if (blk * kCB < G * prm[img].n_labels) {
            for (int k = k0; k < k1; ++k) {
                const int g = L.csr[k];
                const int p = (g - img * L.P) / (D + 1);
                const float w = L.w[g];
                const long long pix = (long long)img * L.N + p;
                const float nq = L.norm[pix];
                const float4* q = reinterpret_cast<const float4*>(Q + pix * CP + blk * kCB);
                const float4 a = q[0], b = q[1];
                const float qv[kCB] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
                for (int c = 0; c < kCB; ++c) acc[c] = __fadd_rn(acc[c], __fmul_rn(w, __fmul_rn(nq, qv[c])));
            }
        }
    }
    float4* o = reinterpret_cast<float4*>(out + (long long)v * kCB);
    o[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    o[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
}

// one blur pass along lattice direction j (Jacobi): v' = v + 0.5*(v[n1] + v[n2]), a missing neighbour counts as 0
template <int D>
__global__ void crf_blur(const int* __restrict__ nbr, int V, int j, const float* __restrict__ in, float* __restrict__ out) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    const int n1 = nbr[((long long)v * (D + 1) + j) * 2], n2 = nbr[((long long)v * (D + 1) + j) * 2 + 1];
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4* src = reinterpret_cast<const float4*>(in);
    float4* dst = reinterpret_cast<float4*>(out);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const float4 s = src[(long long)v * 2 + h];
        const float4 a = n1 >= 0 ? src[(long long)n1 * 2 + h] : z;
        const float4 b = n2 >= 0 ? src[(long long)n2 * 2 + h] : z;
        dst[(long long)v * 2 + h] = make_float4(__fadd_rn(s.x, __fmul_rn(0.5f, __fadd_rn(a.x, b.x))),
                                                __fadd_rn(s.y, __fmul_rn(0.5f, __fadd_rn(a.y, b.y))),
                                                __fadd_rn(s.z, __fmul_rn(0.5f, __fadd_rn(a.z, b.z))),
                                                __fadd_rn(s.w, __fmul_rn(0.5f, __fadd_rn(a.w, b.w))));
    }
}

__device__ __forceinline__ float neg_unary(const ImgParam& pr, const int* __restrict__ labels, int img, int G, int N, int p, int ch) {
    const int g = ch / pr.n_labels, l = ch - g * pr.n_labels;
    const int lab = labels[((long long)img * G + g) * N + p];
    return -(l == lab ? pr.pe : pr.ne);
}

// slice: L = sum_r (w_r * v[vertex_r]) * alpha.  mode 0: norm = 1/sqrt(L + 1e-20) (channel 0);  mode 1: T = -U + w*(norm*L);
// mode 2: T += w*(norm*L)
template <int D>
__global__ void crf_slice(Lat L, int n, const float* __restrict__ vals, int blk, int CP, int G, const ImgParam* __restrict__ prm,
                          const int* __restrict__ labels, float compat, int mode, float* __restrict__ norm_out,
                          float* __restrict__ T) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)n * L.N) return;
    const int img = (int)(idx / L.N), p = (int)(idx % L.N);
    const float alpha = (float)(1.0 / (1.0 + 1.0 / (1 << D)));
    int C = 0;
    if (mode != 0) {
        C = G * prm[img].n_labels;
        if (blk * kCB >= C) return;
    }
    float acc[kCB];
#pragma unroll
    for (int c = 0; c < kCB; ++c) acc[c] = 0.f;
    const long long base = idx * (D + 1);
#pragma unroll
    for (int r = 0; r <= D; ++r) {
        const int vert = L.pvert[base + r];
        const float w = L.w[base + r];
        const float4* src = reinterpret_cast<const float4*>(vals + (long long)vert * kCB);
        const float4 a = src[0], b = src[1];
        const float vv[kCB] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
        for (int c = 0; c < kCB; ++c) acc[c] = __fadd_rn(acc[c], __fmul_rn(__fmul_rn(w, vv[c]), alpha));
    }
    if (mode == 0) {
        norm_out[idx] = __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(acc[0], 1e-20f)));
        return;
    }
    const float nm = L.norm[idx];
    const ImgParam& pr = prm[img];
#pragma unroll
    for (int c = 0; c < kCB; ++c) {
        const int ch = blk * kCB + c;
        if (ch >= C) break;
        const float term = __fmul_rn(compat, __fmul_rn(nm, acc[c]));
        const float b0 = mode == 1 ? neg_unary(pr, labels, img, G, L.N, p, ch) : T[idx * CP + ch];
        T[idx * CP + ch] = __fadd_rn(b0, term);
    }
}

// Q = softmax(T) per CRF (from -U when T is null): max subtracted, exp in double rounded once, sequential sum, IEEE division.
// Padding channels [G*n_labels, CP) are written as 0.
__global__ void crf_softmax(int n, int N, int CP, int G, const ImgParam* __restrict__ prm, const int* __restrict__ labels,
                            const float* __restrict__ T, float* __restrict__ Q) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)n * N) return;
    const int img = (int)(idx / N), p = (int)(idx % N);
    const ImgParam& pr = prm[img];
    const int nl = pr.n_labels;
    float* q = Q + idx * CP;
    for (int g = 0; g < G; ++g) {
        float m = -INFINITY;
        for (int l = 0; l < nl; ++l) {
            const int ch = g * nl + l;
            const float x = T ? T[idx * CP + ch] : neg_unary(pr, labels, img, G, N, p, ch);
            m = fmaxf(m, x);
        }
        float s = 0.f;
        for (int l = 0; l < nl; ++l) {
            const int ch = g * nl + l;
            const float x = T ? T[idx * CP + ch] : neg_unary(pr, labels, img, G, N, p, ch);
            const float e = (float)exp((double)__fsub_rn(x, m));
            q[ch] = e;
            s = __fadd_rn(s, e);
        }
        for (int l = 0; l < nl; ++l) q[g * nl + l] = __fdiv_rn(q[g * nl + l], s);
    }
    for (int ch = G * nl; ch < CP; ++ch) q[ch] = 0.f;
}

// tail: argmax per CRF (first maximum wins).  Generic: labels_out int32 [n][G][N], q_out fp32 [n][n_labels][N] (G == 1).
// Step (conf != null): fg = keys[argmax Q_fg], bg = keys[argmax Q_bg]; conf = fg, 255 where fg == 0, 0 where fg + bg == 0.
__global__ void crf_final(int n, int N, int CP, int G, const ImgParam* __restrict__ prm, const float* __restrict__ Q,
                          int* __restrict__ labels_out, float* __restrict__ q_out, uint8_t* __restrict__ conf) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)n * N) return;
    const int img = (int)(idx / N), p = (int)(idx % N);
    const ImgParam& pr = prm[img];
    const int nl = pr.n_labels;
    const float* q = Q + idx * CP;
    int arg[2] = {0, 0};
    for (int g = 0; g < G; ++g) {
        float best = q[g * nl];
        for (int l = 1; l < nl; ++l) {
            const float v = q[g * nl + l];
            if (v > best) { best = v; arg[g] = l; }
        }
        if (labels_out) labels_out[((long long)img * G + g) * N + p] = arg[g];
    }
    if (q_out)
        for (int l = 0; l < nl; ++l) q_out[((long long)img * nl + l) * N + p] = q[l];
    if (conf) {
        const int fg = pr.keys[arg[0]], bg = pr.keys[arg[1]];
        int c = fg;
        if (fg == 0) c = 255;
        if (bg + fg == 0) c = 0;
        conf[idx] = (uint8_t)c;
    }
}

// step: the confident fg / bg label maps, argmax over [thres, cam_0, ..., cam_{K-1}] (first maximum wins)
__global__ void crf_conf_labels(int n, int N, const float* __restrict__ high, const ImgParam* __restrict__ prm, float fg, float bg,
                                int* __restrict__ labels) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)n * N) return;
    const int img = (int)(idx / N), p = (int)(idx % N);
    const ImgParam& pr = prm[img];
    const float thr[2] = {fg, bg};
    for (int g = 0; g < 2; ++g) {
        float best = thr[g];
        int arg = 0;
        for (int k = 0; k + 1 < pr.n_labels; ++k) {
            const float v = high[((long long)pr.cam_off + k) * N + p];
            if (v > best) { best = v; arg = k + 1; }
        }
        labels[((long long)img * 2 + g) * N + p] = arg;
    }
}

__global__ void crf_check_labels(const int* __restrict__ labels, long long total, int n_labels, int* __restrict__ err) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < total && (labels[k] < 0 || labels[k] >= n_labels)) atomicOr(err, 2);
}

// ------------------------------------------------------------------------------------------------------------------------
// host side

struct Layout {
    size_t q, t, lab, prm, info, region, cub;            // offsets
    size_t lat[2][6];                                     // w, pvert, csr, vstart, nbr, norm
    size_t sk_in, sk_out, sp_in, shead, svid, svkey, scub;   // build scratch, aliased into the value region
    size_t vals[2];
    size_t total;
};

inline int dims(int i) { return i == 0 ? 2 : 5; }

static size_t cub_bytes(long long P, long long nP) {
    size_t a = 0, b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, a, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (const int*)nullptr,
                                    (int*)nullptr, (int)P, 0, 64);
    cub::DeviceScan::InclusiveSum(nullptr, b, (const int*)nullptr, (int*)nullptr, (int)nP);
    return a > b ? a : b;
}

static Layout layout(int n, int H, int W, int G, int max_labels) {
    Layout L{};
    const long long N = (long long)H * W, nN = n * N;
    const int CP = (G * max_labels + kCB - 1) / kCB * kCB;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
    L.q = take(nN * CP * 4);
    L.t = take(nN * CP * 4);
    L.lab = take(nN * G * 4);
    L.prm = take(sizeof(ImgParam) * n);
    L.info = take(4 * (1 + 2 * (n + 1)));
    for (int li = 0; li < 2; ++li) {
        const int D = dims(li);
        const long long nP = nN * (D + 1);
        L.lat[li][0] = take(nP * 4);
        L.lat[li][1] = take(nP * 4);
        L.lat[li][2] = take(nP * 4);
        L.lat[li][3] = take((nP + 1) * 4);
        L.lat[li][4] = take(nP * (D + 1) * 2 * 4);
        L.lat[li][5] = take(nN * 4);
    }
    const long long nP5 = nN * 6;
    // region: the vertex value ping-pong buffers; before that, the scratch of the lattice builds
    size_t vb = align_up(nP5 * kCB * 4, 256);
    size_t s = 0;
    auto stake = [&](size_t bytes) { size_t r = s; s = align_up(s + bytes, 256); return r; };
    L.sk_in = stake(nP5 * 8);
    L.sk_out = stake(nP5 * 8);
    L.sp_in = stake(nP5 * 4);
    L.shead = stake(nP5 * 4);
    L.svid = stake(nP5 * 4);
    L.svkey = stake(nP5 * 8);
    L.scub = stake(cub_bytes(N * 6, nP5));
    L.region = o;
    L.vals[0] = o;
    L.vals[1] = o + vb;
    L.total = o + (2 * vb > s ? 2 * vb : s);
    return L;
}

static int check_device_ptr(const void* p, const char* what) {
    if (!p) return fail(kBadArg, "irn crf: %s is NULL", what);
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return fail(kBadArg, "irn crf: %s is not a device pointer", what);
    }
    if (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged)
        return fail(kBadArg, "irn crf: %s is not a device pointer (host memory; there is no CPU path)", what);
    return kOk;
}

struct Timing {
    bool on = false;
    cudaEvent_t ev[4] = {};
    bool valid = false;
};
static thread_local Timing g_timing;

static inline unsigned grid_of(long long n, int b) { return (unsigned)((n + b - 1) / b); }

struct Run {
    int n, H, W, G, CP, t;
    float wg, wb, sxy_g, sxy_b, srgb;
};

template <int D>
static int build_lattice(const Run& R, const uint8_t* img, char* ws, const Layout& Lo, int li, float sxy, float srgb, int* err_dev,
                         int* voff_dev, cudaStream_t st) {
    const long long N = (long long)R.H * R.W, nN = R.n * N, P = N * (D + 1), nP = nN * (D + 1);
    Scale<D> sf;
    for (int i = 0; i < D; ++i) sf.s[i] = (float)((D + 1) * std::sqrt(2.0 / 3.0) / std::sqrt((double)(i + 1) * (i + 2)));
    auto* k_in = (unsigned long long*)(ws + Lo.region + Lo.sk_in);
    auto* k_out = (unsigned long long*)(ws + Lo.region + Lo.sk_out);
    int* p_in = (int*)(ws + Lo.region + Lo.sp_in);
    int* head = (int*)(ws + Lo.region + Lo.shead);
    int* vid = (int*)(ws + Lo.region + Lo.svid);
    auto* vkey = (unsigned long long*)(ws + Lo.region + Lo.svkey);
    void* tmp = ws + Lo.region + Lo.scub;
    size_t tmp_bytes = cub_bytes(P, nP);
    float* w = (float*)(ws + Lo.lat[li][0]);
    int* pvert = (int*)(ws + Lo.lat[li][1]);
    int* csr = (int*)(ws + Lo.lat[li][2]);
    int* vstart = (int*)(ws + Lo.lat[li][3]);
    crf_elevate<D><<<grid_of(nN, 128), 128, 0, st>>>(img, R.n, R.H, R.W, sxy, srgb, sf, k_in, p_in, w, err_dev);
    IRN_LAUNCH_CHECK("crf_elevate");
    for (int i = 0; i < R.n; ++i) {    // stable LSD radix sort: equal keys keep ascending pixel order
        IRN_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, k_in + i * P, k_out + i * P, p_in + i * P, csr + i * P, (int)P, 0,
                                                 (64 / D) * D, st));
        launch_counter()++;
    }
    crf_heads<<<grid_of(nP, 256), 256, 0, st>>>(k_out, nP, (int)P, head);
    IRN_LAUNCH_CHECK("crf_heads");
    IRN_CUDA(cub::DeviceScan::InclusiveSum(tmp, tmp_bytes, head, vid, (int)nP, st));
    crf_mark<<<grid_of(nP, 256), 256, 0, st>>>(k_out, csr, vid, nP, (int)P, R.n, vstart, vkey, pvert, voff_dev);
    IRN_LAUNCH_CHECK("crf_mark");
    return kOk;
}

template <int D>
static Lat lat_view(const Run& R, char* ws, const Layout& Lo, int li) {
    Lat L;
    L.N = R.H * R.W;
    L.P = L.N * (D + 1);
    L.w = (const float*)(ws + Lo.lat[li][0]);
    L.pvert = (const int*)(ws + Lo.lat[li][1]);
    L.csr = (const int*)(ws + Lo.lat[li][2]);
    L.vstart = (const int*)(ws + Lo.lat[li][3]);
    L.nbr = (const int*)(ws + Lo.lat[li][4]);
    L.norm = (const float*)(ws + Lo.lat[li][5]);
    return L;
}

template <int D>
static int finish_lattice(const Run& R, char* ws, const Layout& Lo, int li, int V, const int* voff_dev, cudaStream_t st) {
    Lat L = lat_view<D>(R, ws, Lo, li);
    auto* vkey = (const unsigned long long*)(ws + Lo.region + Lo.svkey);
    crf_neighbours<D><<<grid_of(V, 128), 128, 0, st>>>(vkey, L.vstart, L.csr, voff_dev, V, L.P, (int*)L.nbr);
    IRN_LAUNCH_CHECK("crf_neighbours");
    return kOk;
}

// L(.) of one channel block through lattice li; mode as crf_slice
template <int D>
static int filter(const Run& R, char* ws, const Layout& Lo, int li, int V, const float* Q, int blk, const ImgParam* prm,
                  const int* labels, float compat, int mode, float* T, cudaStream_t st) {
    Lat L = lat_view<D>(R, ws, Lo, li);
    float* a = (float*)(ws + Lo.vals[0]);
    float* b = (float*)(ws + Lo.vals[1]);
    crf_splat<D><<<grid_of(V, 128), 128, 0, st>>>(L, V, Q, R.CP, blk, R.G, prm, a);
    IRN_LAUNCH_CHECK("crf_splat");
    for (int j = 0; j <= D; ++j) {
        crf_blur<D><<<grid_of(V, 256), 256, 0, st>>>(L.nbr, V, j, a, b);
        IRN_LAUNCH_CHECK("crf_blur");
        float* s = a;
        a = b;
        b = s;
    }
    crf_slice<D><<<grid_of((long long)R.n * L.N, 128), 128, 0, st>>>(L, R.n, a, blk, R.CP, R.G, prm, labels, compat, mode,
                                                                     (float*)L.norm, T);
    IRN_LAUNCH_CHECK("crf_slice");
    return kOk;
}

// the whole CRF once the label maps [n][G][N] are in the workspace and the per-image parameters are uploaded
static int run_crf(const Run& R, const uint8_t* img, char* ws, const Layout& Lo, const std::vector<ImgParam>& prm_host,
                   int* labels_out, float* q_out, uint8_t* conf, int32_t* counts_host, cudaStream_t st) {
    const long long N = (long long)R.H * R.W, nN = R.n * N;
    const ImgParam* prm = (const ImgParam*)(ws + Lo.prm);
    const int* labels = (const int*)(ws + Lo.lab);
    float* Q = (float*)(ws + Lo.q);
    float* T = (float*)(ws + Lo.t);
    int* info = (int*)(ws + Lo.info);
    int* voff[2] = {info + 1, info + 1 + (R.n + 1)};
    Timing& tm = g_timing;
    if (tm.on) IRN_CUDA(cudaEventRecord(tm.ev[0], st));
    int rc = build_lattice<2>(R, img, ws, Lo, 0, R.sxy_g, 1.f, info, voff[0], st);
    if (rc) return rc;
    // the second build reuses the sort scratch: the first lattice's vertex keys are consumed by its neighbour search first
    std::vector<int> host(1 + 2 * (R.n + 1));
    IRN_CUDA(cudaMemcpyAsync(host.data(), info, 4 * (1 + (R.n + 1)), cudaMemcpyDeviceToHost, st));
    IRN_CUDA(cudaStreamSynchronize(st));
    if (host[0] & 2) return fail(kBadArg, "irn_dense_crf: a label is outside [0, n_labels)");
    if (host[0] & 1) return fail(kUnsupported, "irn crf: a lattice coordinate exceeds the 32-bit key packing range (image too large for sxy)");
    const int Vg = host[R.n + 1];
    rc = finish_lattice<2>(R, ws, Lo, 0, Vg, voff[0], st);
    if (rc) return rc;
    rc = build_lattice<5>(R, img, ws, Lo, 1, R.sxy_b, R.srgb, info, voff[1], st);
    if (rc) return rc;
    IRN_CUDA(cudaMemcpyAsync(host.data(), info, 4 * host.size(), cudaMemcpyDeviceToHost, st));
    IRN_CUDA(cudaStreamSynchronize(st));
    if (host[0] & 1) return fail(kUnsupported, "irn crf: a lattice coordinate exceeds the 12-bit key packing range of the bilateral lattice");
    const int Vb = host[2 * (R.n + 1)];
    rc = finish_lattice<5>(R, ws, Lo, 1, Vb, voff[1], st);
    if (rc) return rc;
    if (counts_host)
        for (int i = 0; i < R.n; ++i) {
            counts_host[2 * i] = host[1 + i + 1] - host[1 + i];
            counts_host[2 * i + 1] = host[1 + (R.n + 1) + i + 1] - host[1 + (R.n + 1) + i];
        }
    rc = filter<2>(R, ws, Lo, 0, Vg, nullptr, 0, prm, labels, 0.f, 0, nullptr, st);
    if (rc) return rc;
    rc = filter<5>(R, ws, Lo, 1, Vb, nullptr, 0, prm, labels, 0.f, 0, nullptr, st);
    if (rc) return rc;
    crf_softmax<<<grid_of(nN, 128), 128, 0, st>>>(R.n, (int)N, R.CP, R.G, prm, labels, nullptr, Q);
    IRN_LAUNCH_CHECK("crf_softmax");
    if (tm.on) IRN_CUDA(cudaEventRecord(tm.ev[1], st));
    const int nb = R.CP / kCB;
    for (int it = 0; it < R.t; ++it) {
        for (int blk = 0; blk < nb; ++blk) {
            rc = filter<2>(R, ws, Lo, 0, Vg, Q, blk, prm, labels, R.wg, 1, T, st);
            if (rc) return rc;
            rc = filter<5>(R, ws, Lo, 1, Vb, Q, blk, prm, labels, R.wb, 2, T, st);
            if (rc) return rc;
        }
        crf_softmax<<<grid_of(nN, 128), 128, 0, st>>>(R.n, (int)N, R.CP, R.G, prm, labels, T, Q);
        IRN_LAUNCH_CHECK("crf_softmax");
    }
    if (tm.on) IRN_CUDA(cudaEventRecord(tm.ev[2], st));
    crf_final<<<grid_of(nN, 128), 128, 0, st>>>(R.n, (int)N, R.CP, R.G, prm, Q, labels_out, q_out, conf);
    IRN_LAUNCH_CHECK("crf_final");
    if (tm.on) {
        IRN_CUDA(cudaEventRecord(tm.ev[3], st));
        tm.valid = true;
    }
    return kOk;
}

static int common_checks(int n, int H, int W, const uint8_t* img, void* ws, size_t ws_bytes, size_t need) {
    if (n <= 0 || H <= 0 || W <= 0) return fail(kBadArg, "irn crf: bad sizes n=%d H=%d W=%d", n, H, W);
    if ((long long)n * H * W * 6 >= (1LL << 31)) return fail(kUnsupported, "irn crf: batch too large (%d x %dx%d): split it", n, H, W);
    if (int rc = check_device_ptr(img, "images")) return rc;
    if (int rc = check_device_ptr(ws, "workspace")) return rc;
    if (ws_bytes < need) return fail(kWorkspace, "irn crf: workspace %zu bytes < %zu", ws_bytes, need);
    return kOk;
}

}  // namespace crf
}  // namespace irn

using namespace irn;
using namespace irn::crf;

extern "C" size_t irn_crf_workspace_bytes(int n, int H, int W, int n_groups, int max_labels) {
    if (n <= 0 || H <= 0 || W <= 0 || n_groups < 1 || n_groups > 2 || max_labels < 1 || max_labels > kMaxLabels) return 0;
    return layout(n, H, W, n_groups, max_labels).total;
}

extern "C" int irn_crf_max_labels(void) { return kMaxLabels; }

extern "C" int irn_crf_set_timing(int enable) {
    Timing& tm = g_timing;
    if (enable && !tm.ev[0])
        for (auto& e : tm.ev) IRN_CUDA(cudaEventCreate(&e));
    tm.on = enable != 0;
    tm.valid = false;
    return kOk;
}

extern "C" int irn_crf_last_ms(float* ms3) {
    Timing& tm = g_timing;
    if (!tm.valid) return fail(kBadArg, "irn_crf_last_ms: no timed call");
    IRN_CUDA(cudaEventSynchronize(tm.ev[3]));
    for (int i = 0; i < 3; ++i) IRN_CUDA(cudaEventElapsedTime(ms3 + i, tm.ev[i], tm.ev[i + 1]));
    return kOk;
}

extern "C" int irn_dense_crf(const uint8_t* img, const int32_t* labels, int n, int H, int W, int n_labels, int t, double gt_prob,
                             float gauss_sxy, float gauss_compat, float bil_sxy, float bil_srgb, float bil_compat, int32_t* labels_out,
                             float* q_out, int32_t* vertex_counts, void* workspace, size_t workspace_bytes, irn_stream_t stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    launch_counter() = 0;
    if (n_labels < 1 || n_labels > kMaxLabels)
        return fail(kUnsupported, "irn_dense_crf: n_labels=%d outside [1, %d]", n_labels, kMaxLabels);
    if (t < 0 || !(gt_prob > 0.0 && gt_prob < 1.0) || !(gauss_sxy > 0.f) || !(bil_sxy > 0.f) || !(bil_srgb > 0.f))
        return fail(kBadArg, "irn_dense_crf: bad parameters t=%d gt_prob=%g sxy=%g/%g srgb=%g", t, gt_prob, gauss_sxy, bil_sxy, bil_srgb);
    const size_t need = irn_crf_workspace_bytes(n, H, W, 1, n_labels);
    if (int rc = common_checks(n, H, W, img, workspace, workspace_bytes, need)) return rc;
    if (int rc = check_device_ptr(labels, "labels")) return rc;
    if (!labels_out && !q_out) return fail(kBadArg, "irn_dense_crf: no output");
    if (labels_out)
        if (int rc = check_device_ptr(labels_out, "labels_out")) return rc;
    if (q_out)
        if (int rc = check_device_ptr(q_out, "q_out")) return rc;
    Layout Lo = layout(n, H, W, 1, n_labels);
    char* ws = (char*)workspace;
    Run R{n, H, W, 1, (n_labels + kCB - 1) / kCB * kCB, t, gauss_compat, bil_compat, gauss_sxy, bil_sxy, bil_srgb};
    std::vector<ImgParam> prm(n);
    const double pe = -std::log((double)gt_prob);
    const double ne = n_labels > 1 ? -std::log((1.0 - (double)gt_prob) / (n_labels - 1)) : pe;
    for (auto& p : prm) {
        p = ImgParam{};
        p.n_labels = n_labels;
        p.pe = (float)pe;
        p.ne = (float)ne;
    }
    const long long N = (long long)H * W;
    IRN_CUDA(cudaMemsetAsync(ws + Lo.info, 0, 4, st));
    IRN_CUDA(cudaMemcpyAsync(ws + Lo.prm, prm.data(), sizeof(ImgParam) * n, cudaMemcpyHostToDevice, st));
    IRN_CUDA(cudaMemcpyAsync(ws + Lo.lab, labels, 4 * n * N, cudaMemcpyDeviceToDevice, st));
    crf_check_labels<<<grid_of(n * N, 256), 256, 0, st>>>((const int*)(ws + Lo.lab), n * N, n_labels, (int*)(ws + Lo.info));
    IRN_LAUNCH_CHECK("crf_check_labels");
    return run_crf(R, img, ws, Lo, prm, labels_out, q_out, nullptr, vertex_counts, st);
}

extern "C" int irn_ir_label(const uint8_t* img, const float* high_res, const int32_t* keys_host, const int32_t* counts_host, int n,
                            int H, int W, float conf_fg_thres, float conf_bg_thres, uint8_t* out, int32_t* vertex_counts,
                            void* workspace, size_t workspace_bytes, irn_stream_t stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    launch_counter() = 0;
    if (!counts_host) return fail(kBadArg, "irn_ir_label: counts is NULL");
    int max_labels = 1, total_k = 0;
    for (int i = 0; i < n; ++i) {
        if (counts_host[i] < 0 || counts_host[i] + 1 > kMaxLabels)
            return fail(kUnsupported, "irn_ir_label: image %d has %d classes (at most %d)", i, counts_host[i], kMaxLabels - 1);
        max_labels = counts_host[i] + 1 > max_labels ? counts_host[i] + 1 : max_labels;
        total_k += counts_host[i];
    }
    const size_t need = irn_crf_workspace_bytes(n, H, W, 2, max_labels);
    if (int rc = common_checks(n, H, W, img, workspace, workspace_bytes, need)) return rc;
    if (total_k > 0)
        if (int rc = check_device_ptr(high_res, "high_res")) return rc;
    if (int rc = check_device_ptr(out, "out")) return rc;
    if (total_k > 0 && !keys_host) return fail(kBadArg, "irn_ir_label: keys is NULL");
    Layout Lo = layout(n, H, W, 2, max_labels);
    char* ws = (char*)workspace;
    Run R{n, H, W, 2, (2 * max_labels + kCB - 1) / kCB * kCB, 10, 3.f, 10.f, 3.f, 50.f, 5.f};
    std::vector<ImgParam> prm(n);
    int off = 0;
    for (int i = 0; i < n; ++i) {
        ImgParam& p = prm[i];
        p = ImgParam{};
        p.n_labels = counts_host[i] + 1;
        p.cam_off = off;
        const double pe = -std::log(0.7);
        p.pe = (float)pe;
        p.ne = (float)(p.n_labels > 1 ? -std::log((1.0 - 0.7) / (p.n_labels - 1)) : pe);
        p.keys[0] = 0;                                   // np.pad(keys + 1, (1, 0))
        for (int k = 0; k < counts_host[i]; ++k) p.keys[k + 1] = keys_host[off + k] + 1;
        off += counts_host[i];
    }
    const long long N = (long long)H * W;
    IRN_CUDA(cudaMemsetAsync(ws + Lo.info, 0, 4, st));
    IRN_CUDA(cudaMemcpyAsync(ws + Lo.prm, prm.data(), sizeof(ImgParam) * n, cudaMemcpyHostToDevice, st));
    crf_conf_labels<<<grid_of(n * N, 128), 128, 0, st>>>(n, (int)N, high_res, (const ImgParam*)(ws + Lo.prm), conf_fg_thres,
                                                         conf_bg_thres, (int*)(ws + Lo.lab));
    IRN_LAUNCH_CHECK("crf_conf_labels");
    return run_crf(R, img, ws, Lo, prm, nullptr, nullptr, out, vertex_counts, st);
}
