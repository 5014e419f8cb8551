// N3: fully connected CRF (mean field on two permutohedral lattices) and the cam_to_ir_label step.
// Reference: misc/imutils.py:156-170 (crf_inference_label through pydensecrf) and step/cam_to_ir_label.py:19-41.
// The arithmetic is the one oracle/crf.py states (Kraehenbuehl & Koltun 2011; Adams, Baek & Davis 2010, section 3): every
// floating-point operation below is written with an explicit _rn intrinsic so that no contraction changes a rounding, and the
// lattice keys, splat order, blur and slice order are the oracle's.  No floating-point atomics: the same inputs give the same
// bits on every run.
//
// Per call (a batch of n images of any sizes, image i of N_i = H_i*W_i pixels; pixels, pairs, label maps and outputs of the images
// packed back to back in batch order, so a batch of one size is the [n,H,W] stack):
//   build  per lattice (Gaussian d=2 over (x,y)/sxy, bilateral d=5 over (x,y)/sxy,(r,g,b)/srgb):
//          crf_elevate (one thread per pixel: elevate, rank, barycentrics, d+1 packed 64-bit vertex keys), a stable radix sort
//          of the (key, pair) list of every image, a scan of the run heads (vertex ids), crf_mark (vertex -> first pair, pair ->
//          vertex: a CSR of pairs per vertex in ascending pixel order), crf_neighbours (2(d+1) binary searches per vertex);
//          then norm = 1/sqrt(L(1) + 1e-20).  One host synchronisation reads the vertex counts and the error word.
//   iterate  G CRFs per image (G = 2 for the step: the fg and bg label maps share the image's lattices) as G*n_labels value
//          channels, in blocks of 8: crf_splat (per-vertex gather), d+1 crf_blur passes, crf_slice (slice, * norm, * compat,
//          + (-U) or + the previous term), then crf_softmax.  U comes from the label map (two values per image), never stored.
//   tail   crf_final: argmax over labels (first maximum), and for the step keys[] + the fg/bg combination into 0 / class / 255.
//
// Image geometry comes from per-image descriptors (ImgParam: H_i, W_i, first pixel, first high_res element), uploaded once per call
// with the pixel offsets off[0..n] (off[n] = total pixels).  Image i's pairs in a lattice of dimension D start at off[i]*(D+1), so a
// global pixel, pair or (through the per-image vertex offsets) vertex index finds its image by a binary search over n+1 offsets:
// at most ceil(log2(n+1)) steps on a few hundred L1-resident bytes, no table to size per block shape, no per-image launches, and the
// kernels keep their one-thread-per-pixel / per-vertex grids over the whole batch.  A batch of one size (Batch::N) divides by N
// instead, as the one-size kernels did.
#include <cub/cub.cuh>

#include <cmath>
#include <cstring>
#include <vector>

#include "common.h"

namespace irn {
namespace crf {

constexpr int kMaxLabels = IRN_CAM_MAX_CLASSES + 1;   // per CRF: background + every class of a CAM plan (VOC 21, COCO 81)
constexpr int kCB = 8;           // value channels per pass through the lattice

struct ImgParam {
    int n_labels;                // labels of each of the image's G CRFs
    int H, W;                    // the image's size
    int pix;                     // its first pixel in the batch (= off[i])
    long long cam;               // step: its first high_res element (planes [K_i,H_i,W_i], images back to back)
    float pe, ne;                // -log(gt_prob), -log((1-gt_prob)/(n_labels-1))
    int keys[kMaxLabels];        // step: class id of each label (entry 0 = background)
};

struct Batch {
    int n;
    int N;                       // the pixels of every image when all have one size, else 0
    const int* off;              // [n+1] first pixel of each image, off[n] = total pixels
    const ImgParam* prm;         // [n]
};

// the image holding element x of a strictly increasing offset table t[0..n] (pixels: off; vertices: voff)
__device__ __forceinline__ int image_of(const int* __restrict__ t, int n, long long x) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (t[mid] <= x) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// the image of pixel p: a division when the batch has one size (no dependent loads on the per-iteration kernels' critical path),
// else the search over the pixel offsets
__device__ __forceinline__ int image_of_pixel(const Batch& B, long long p) {
    return B.N ? (int)p / B.N : image_of(B.off, B.n, p);      // p < 2^31: a batch's pairs have 32-bit indices
}

// pair k of a lattice with D1 = D+1 pairs per pixel is the first pair of an image
__device__ __forceinline__ bool image_start(const Batch& B, long long k, int D1, int* img) {
    if (k % D1) return false;
    const long long p = k / D1;
    *img = image_of_pixel(B, p);
    return B.off[*img] == p;
}

struct Lat {                     // one lattice of a batch; pairs are (pixel, remainder): global pixel g*(D+1)+r
    const float* w;              // [nP] barycentric weight of each pair
    const int* pvert;            // [nP] vertex of each pair
    const int* csr;              // [nP] pairs sorted by vertex, ascending pixel within a vertex
    const int* vstart;           // [V+1] first csr position of each vertex
    const int* nbr;              // [V*(D+1)*2] blur neighbours (-1 = none)
    const float* norm;           // [nN]
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
__global__ void crf_elevate(const uint8_t* __restrict__ img, Batch B, long long nN, float sxy, float srgb, Scale<D> sf,
                            unsigned long long* __restrict__ keys, int* __restrict__ pairs, float* __restrict__ wts,
                            int* __restrict__ err) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= nN) return;
    const int im = image_of_pixel(B, idx);
    const int W = B.prm[im].W;
    const int p = (int)(idx - B.off[im]), x = p % W, y = p / W;
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

// a vertex starts at every change of key and at every image's first pair: the sorted (key, pair) lists are per image
__global__ void crf_heads(const unsigned long long* __restrict__ keys, long long total, int D1, Batch B, int* __restrict__ head) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= total) return;
    int img;
    head[k] = (k == 0 || keys[k] != keys[k - 1] || image_start(B, k, D1, &img)) ? 1 : 0;
}

__global__ void crf_mark(const unsigned long long* __restrict__ keys, const int* __restrict__ csr, const int* __restrict__ vid,
                         long long total, int D1, Batch B, int* __restrict__ vstart, unsigned long long* __restrict__ vkey,
                         int* __restrict__ pvert, int* __restrict__ voff) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= total) return;
    const int v = vid[k] - 1;
    int img = 0;
    const bool first = image_start(B, k, D1, &img);
    if (first || keys[k] != keys[k - 1]) {
        vstart[v] = (int)k;
        vkey[v] = keys[k];
    }
    pvert[csr[k]] = v;
    if (first) voff[img] = v;
    if (k == total - 1) {
        vstart[v + 1] = (int)total;
        voff[B.n] = v + 1;
    }
}

template <int D>
__global__ void crf_neighbours(const unsigned long long* __restrict__ vkey, const int* __restrict__ voff, int n, int V,
                               int* __restrict__ nbr) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    constexpr int B = 64 / D;
    const int img = image_of(voff, n, v);
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
__global__ void crf_splat(Lat L, int V, const float* __restrict__ Q, int CP, int blk, int G, Batch B, float* __restrict__ out) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    const int k0 = L.vstart[v], k1 = L.vstart[v + 1];
    float acc[kCB];
#pragma unroll
    for (int c = 0; c < kCB; ++c) acc[c] = 0.f;
    if (Q == nullptr) {
        for (int k = k0; k < k1; ++k) acc[0] = __fadd_rn(acc[0], L.w[L.csr[k]]);
    } else {
        const int img = image_of_pixel(B, L.csr[k0] / (D + 1));
        if (blk * kCB < G * B.prm[img].n_labels) {
            for (int k = k0; k < k1; ++k) {
                const unsigned g = (unsigned)L.csr[k];
                const float w = L.w[g];
                const long long pix = g / (D + 1);
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

// what -U and the label maps need of one image, read once into registers (the kernels' stores could alias the descriptor block)
struct ImgUnary {
    int n_labels, pix, N;
    float pe, ne;
};

__device__ __forceinline__ ImgUnary unary_of(const ImgParam& pr) { return ImgUnary{pr.n_labels, pr.pix, pr.H * pr.W, pr.pe, pr.ne}; }

// the image's map of CRF g among G is [H_i,W_i] at G*pix + g*N_i (the batch's maps are [n][G][N_i], images back to back)
__device__ __forceinline__ long long label_at(const ImgUnary& u, int G, int g, long long idx) {
    return (long long)G * u.pix + (long long)g * u.N + (idx - u.pix);
}

__device__ __forceinline__ float neg_unary(const ImgUnary& u, const int* __restrict__ labels, int G, long long idx, int ch) {
    const int g = ch / u.n_labels, l = ch - g * u.n_labels;
    const int lab = labels[label_at(u, G, g, idx)];
    return -(l == lab ? u.pe : u.ne);
}

// slice: L = sum_r (w_r * v[vertex_r]) * alpha.  mode 0: norm = 1/sqrt(L + 1e-20) (channel 0);  mode 1: T = -U + w*(norm*L);
// mode 2: T += w*(norm*L)
template <int D>
__global__ void crf_slice(Lat L, long long nN, const float* __restrict__ vals, int blk, int CP, int G, Batch B,
                          const int* __restrict__ labels, float compat, int mode, float* __restrict__ norm_out,
                          float* __restrict__ T) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= nN) return;
    const float alpha = (float)(1.0 / (1.0 + 1.0 / (1 << D)));
    int C = 0;
    ImgUnary u{};
    if (mode != 0) {
        u = unary_of(B.prm[image_of_pixel(B, idx)]);
        C = G * u.n_labels;
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
#pragma unroll
    for (int c = 0; c < kCB; ++c) {
        const int ch = blk * kCB + c;
        if (ch >= C) break;
        const float term = __fmul_rn(compat, __fmul_rn(nm, acc[c]));
        const float b0 = mode == 1 ? neg_unary(u, labels, G, idx, ch) : T[idx * CP + ch];
        T[idx * CP + ch] = __fadd_rn(b0, term);
    }
}

// Q = softmax(T) per CRF (from -U when T is null): max subtracted, exp in double rounded once, sequential sum, IEEE division.
// Padding channels [G*n_labels, CP) are written as 0.
__global__ void crf_softmax(Batch B, long long nN, int CP, int G, const int* __restrict__ labels, const float* __restrict__ T,
                            float* __restrict__ Q) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= nN) return;
    const ImgUnary u = unary_of(B.prm[image_of_pixel(B, idx)]);
    const int nl = u.n_labels;
    float* q = Q + idx * CP;
    for (int g = 0; g < G; ++g) {
        float m = -INFINITY;
        for (int l = 0; l < nl; ++l) {
            const int ch = g * nl + l;
            const float x = T ? T[idx * CP + ch] : neg_unary(u, labels, G, idx, ch);
            m = fmaxf(m, x);
        }
        float s = 0.f;
        for (int l = 0; l < nl; ++l) {
            const int ch = g * nl + l;
            const float x = T ? T[idx * CP + ch] : neg_unary(u, labels, G, idx, ch);
            const float e = (float)exp((double)__fsub_rn(x, m));
            q[ch] = e;
            s = __fadd_rn(s, e);
        }
        for (int l = 0; l < nl; ++l) q[g * nl + l] = __fdiv_rn(q[g * nl + l], s);
    }
    for (int ch = G * nl; ch < CP; ++ch) q[ch] = 0.f;
}

// tail: argmax per CRF (first maximum wins).  Generic: labels_out int32 [n][G][N_i], q_out fp32 [n][n_labels][N_i] (G == 1; one
// n_labels for the batch), images back to back.
// Step (conf != null): fg = keys[argmax Q_fg], bg = keys[argmax Q_bg]; conf = fg, 255 where fg == 0, 0 where fg + bg == 0.
__global__ void crf_final(Batch B, long long nN, int CP, int G, const float* __restrict__ Q, int* __restrict__ labels_out,
                          float* __restrict__ q_out, uint8_t* __restrict__ conf) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= nN) return;
    const ImgParam& pr = B.prm[image_of_pixel(B, idx)];
    const ImgUnary u = unary_of(pr);
    const int nl = u.n_labels;
    const float* q = Q + idx * CP;
    int arg[2] = {0, 0};
    for (int g = 0; g < G; ++g) {
        float best = q[g * nl];
        for (int l = 1; l < nl; ++l) {
            const float v = q[g * nl + l];
            if (v > best) { best = v; arg[g] = l; }
        }
        if (labels_out) labels_out[label_at(u, G, g, idx)] = arg[g];
    }
    if (q_out)
        for (int l = 0; l < nl; ++l) q_out[label_at(u, nl, l, idx)] = q[l];
    if (conf) {
        const int fg = pr.keys[arg[0]], bg = pr.keys[arg[1]];
        int c = fg;
        if (fg == 0) c = 255;
        if (bg + fg == 0) c = 0;
        conf[idx] = (uint8_t)c;
    }
}

// step: the confident fg / bg label maps, argmax over [thres, cam_0, ..., cam_{K-1}] (first maximum wins)
__global__ void crf_conf_labels(Batch B, long long nN, const float* __restrict__ high, float fg, float bg, int* __restrict__ labels) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= nN) return;
    const ImgParam& pr = B.prm[image_of_pixel(B, idx)];
    const ImgUnary u = unary_of(pr);
    const long long cam = pr.cam, p = idx - u.pix;
    const float thr[2] = {fg, bg};
    for (int g = 0; g < 2; ++g) {
        float best = thr[g];
        int arg = 0;
        for (int k = 0; k + 1 < u.n_labels; ++k) {
            const float v = high[cam + (long long)k * u.N + p];
            if (v > best) { best = v; arg = k + 1; }
        }
        labels[label_at(u, 2, g, idx)] = arg;
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

// a batch's images on the host: sizes, pixel offsets (off[n] = total pixels), the largest image
struct Sizes {
    int n = 0;
    std::vector<int> hw;         // [n][2]
    std::vector<int> off;        // [n+1]
    long long nN = 0, maxN = 0;
};

// n images of sizes hw [n][2], or all H x W when hw is NULL.  0; 1: image *bad has a size <= 0 (or n <= 0: *bad = -1);
// 2: 6 pairs per pixel overflow the 32-bit pair indices
static int fill_sizes(int n, const int32_t* hw, int H, int W, Sizes& S, int* bad) {
    *bad = -1;
    if (n <= 0) return 1;
    S.n = n;
    S.hw.resize(2 * (size_t)n);
    S.off.resize((size_t)n + 1);
    S.nN = S.maxN = 0;
    for (int i = 0; i < n; ++i) {
        const int h = hw ? hw[2 * i] : H, w = hw ? hw[2 * i + 1] : W;
        if (h <= 0 || w <= 0) {
            *bad = i;
            return 1;
        }
        S.hw[2 * i] = h;
        S.hw[2 * i + 1] = w;
        const long long N = (long long)h * w;
        if ((S.nN + N) * 6 >= (1LL << 31)) return 2;
        S.off[i] = (int)S.nN;
        S.nN += N;
        S.maxN = N > S.maxN ? N : S.maxN;
    }
    S.off[n] = (int)S.nN;
    return 0;
}

// workspace: value buffers and lattices over the batch's pixels, CUB sort scratch for its largest image
static Layout layout(const Sizes& S, int G, int max_labels) {
    Layout L{};
    const int n = S.n;
    const long long nN = S.nN;
    const int CP = (G * max_labels + kCB - 1) / kCB * kCB;
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
    L.q = take(nN * CP * 4);
    L.t = take(nN * CP * 4);
    L.lab = take(nN * G * 4);
    L.prm = take(sizeof(ImgParam) * n + 4 * (n + 1));   // the descriptors, then the pixel offsets
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
    L.scub = stake(cub_bytes(S.maxN * 6, nP5));
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
    const Sizes* S;
    int G, CP, t;
    float wg, wb, sxy_g, sxy_b, srgb;
};

static Batch batch_view(const Run& R, char* ws, const Layout& Lo) {
    const Sizes& S = *R.S;
    const int N = S.maxN * S.n == S.nN ? (int)S.maxN : 0;
    return Batch{S.n, N, (const int*)(ws + Lo.prm + sizeof(ImgParam) * S.n), (const ImgParam*)(ws + Lo.prm)};
}

template <int D>
static int build_lattice(const Run& R, const uint8_t* img, char* ws, const Layout& Lo, int li, float sxy, float srgb, int* err_dev,
                         int* voff_dev, cudaStream_t st) {
    const Sizes& S = *R.S;
    const long long nN = S.nN, nP = nN * (D + 1);
    const Batch B = batch_view(R, ws, Lo);
    Scale<D> sf;
    for (int i = 0; i < D; ++i) sf.s[i] = (float)((D + 1) * std::sqrt(2.0 / 3.0) / std::sqrt((double)(i + 1) * (i + 2)));
    auto* k_in = (unsigned long long*)(ws + Lo.region + Lo.sk_in);
    auto* k_out = (unsigned long long*)(ws + Lo.region + Lo.sk_out);
    int* p_in = (int*)(ws + Lo.region + Lo.sp_in);
    int* head = (int*)(ws + Lo.region + Lo.shead);
    int* vid = (int*)(ws + Lo.region + Lo.svid);
    auto* vkey = (unsigned long long*)(ws + Lo.region + Lo.svkey);
    void* tmp = ws + Lo.region + Lo.scub;
    size_t tmp_bytes = cub_bytes(S.maxN * (D + 1), nP);
    float* w = (float*)(ws + Lo.lat[li][0]);
    int* pvert = (int*)(ws + Lo.lat[li][1]);
    int* csr = (int*)(ws + Lo.lat[li][2]);
    int* vstart = (int*)(ws + Lo.lat[li][3]);
    crf_elevate<D><<<grid_of(nN, 128), 128, 0, st>>>(img, B, nN, sxy, srgb, sf, k_in, p_in, w, err_dev);
    IRN_LAUNCH_CHECK("crf_elevate");
    for (int i = 0; i < S.n; ++i) {    // stable LSD radix sort of each image's pairs: equal keys keep ascending pixel order
        const long long a = (long long)S.off[i] * (D + 1), P = ((long long)S.off[i + 1] - S.off[i]) * (D + 1);
        IRN_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, k_in + a, k_out + a, p_in + a, csr + a, (int)P, 0, (64 / D) * D, st));
        launch_counter()++;
    }
    crf_heads<<<grid_of(nP, 256), 256, 0, st>>>(k_out, nP, D + 1, B, head);
    IRN_LAUNCH_CHECK("crf_heads");
    IRN_CUDA(cub::DeviceScan::InclusiveSum(tmp, tmp_bytes, head, vid, (int)nP, st));
    crf_mark<<<grid_of(nP, 256), 256, 0, st>>>(k_out, csr, vid, nP, D + 1, B, vstart, vkey, pvert, voff_dev);
    IRN_LAUNCH_CHECK("crf_mark");
    return kOk;
}

static Lat lat_view(char* ws, const Layout& Lo, int li) {
    Lat L;
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
    Lat L = lat_view(ws, Lo, li);
    auto* vkey = (const unsigned long long*)(ws + Lo.region + Lo.svkey);
    crf_neighbours<D><<<grid_of(V, 128), 128, 0, st>>>(vkey, voff_dev, R.S->n, V, (int*)L.nbr);
    IRN_LAUNCH_CHECK("crf_neighbours");
    return kOk;
}

// L(.) of one channel block through lattice li; mode as crf_slice
template <int D>
static int filter(const Run& R, char* ws, const Layout& Lo, int li, int V, const float* Q, int blk, const int* labels, float compat,
                  int mode, float* T, cudaStream_t st) {
    Lat L = lat_view(ws, Lo, li);
    const Batch B = batch_view(R, ws, Lo);
    float* a = (float*)(ws + Lo.vals[0]);
    float* b = (float*)(ws + Lo.vals[1]);
    crf_splat<D><<<grid_of(V, 128), 128, 0, st>>>(L, V, Q, R.CP, blk, R.G, B, a);
    IRN_LAUNCH_CHECK("crf_splat");
    for (int j = 0; j <= D; ++j) {
        crf_blur<D><<<grid_of(V, 256), 256, 0, st>>>(L.nbr, V, j, a, b);
        IRN_LAUNCH_CHECK("crf_blur");
        float* s = a;
        a = b;
        b = s;
    }
    crf_slice<D><<<grid_of(R.S->nN, 128), 128, 0, st>>>(L, R.S->nN, a, blk, R.CP, R.G, B, labels, compat, mode, (float*)L.norm, T);
    IRN_LAUNCH_CHECK("crf_slice");
    return kOk;
}

// the whole CRF once the label maps [n][G][N_i] are in the workspace and the per-image descriptors are uploaded
static int run_crf(const Run& R, const uint8_t* img, char* ws, const Layout& Lo, int* labels_out, float* q_out, uint8_t* conf,
                   int32_t* counts_host, cudaStream_t st) {
    const int n = R.S->n;
    const long long nN = R.S->nN;
    const Batch B = batch_view(R, ws, Lo);
    const int* labels = (const int*)(ws + Lo.lab);
    float* Q = (float*)(ws + Lo.q);
    float* T = (float*)(ws + Lo.t);
    int* info = (int*)(ws + Lo.info);
    int* voff[2] = {info + 1, info + 1 + (n + 1)};
    Timing& tm = g_timing;
    if (tm.on) IRN_CUDA(cudaEventRecord(tm.ev[0], st));
    int rc = build_lattice<2>(R, img, ws, Lo, 0, R.sxy_g, 1.f, info, voff[0], st);
    if (rc) return rc;
    // the second build reuses the sort scratch: the first lattice's vertex keys are consumed by its neighbour search first
    std::vector<int> host(1 + 2 * (n + 1));
    IRN_CUDA(cudaMemcpyAsync(host.data(), info, 4 * (1 + (n + 1)), cudaMemcpyDeviceToHost, st));
    IRN_CUDA(cudaStreamSynchronize(st));
    if (host[0] & 2) return fail(kBadArg, "irn_dense_crf: a label is outside [0, n_labels)");
    if (host[0] & 1) return fail(kUnsupported, "irn crf: a lattice coordinate exceeds the 32-bit key packing range (image too large for sxy)");
    const int Vg = host[n + 1];
    rc = finish_lattice<2>(R, ws, Lo, 0, Vg, voff[0], st);
    if (rc) return rc;
    rc = build_lattice<5>(R, img, ws, Lo, 1, R.sxy_b, R.srgb, info, voff[1], st);
    if (rc) return rc;
    IRN_CUDA(cudaMemcpyAsync(host.data(), info, 4 * host.size(), cudaMemcpyDeviceToHost, st));
    IRN_CUDA(cudaStreamSynchronize(st));
    if (host[0] & 1) return fail(kUnsupported, "irn crf: a lattice coordinate exceeds the 12-bit key packing range of the bilateral lattice");
    const int Vb = host[2 * (n + 1)];
    rc = finish_lattice<5>(R, ws, Lo, 1, Vb, voff[1], st);
    if (rc) return rc;
    if (counts_host)
        for (int i = 0; i < n; ++i) {
            counts_host[2 * i] = host[1 + i + 1] - host[1 + i];
            counts_host[2 * i + 1] = host[1 + (n + 1) + i + 1] - host[1 + (n + 1) + i];
        }
    rc = filter<2>(R, ws, Lo, 0, Vg, nullptr, 0, labels, 0.f, 0, nullptr, st);
    if (rc) return rc;
    rc = filter<5>(R, ws, Lo, 1, Vb, nullptr, 0, labels, 0.f, 0, nullptr, st);
    if (rc) return rc;
    crf_softmax<<<grid_of(nN, 128), 128, 0, st>>>(B, nN, R.CP, R.G, labels, nullptr, Q);
    IRN_LAUNCH_CHECK("crf_softmax");
    if (tm.on) IRN_CUDA(cudaEventRecord(tm.ev[1], st));
    const int nb = R.CP / kCB;
    for (int it = 0; it < R.t; ++it) {
        for (int blk = 0; blk < nb; ++blk) {
            rc = filter<2>(R, ws, Lo, 0, Vg, Q, blk, labels, R.wg, 1, T, st);
            if (rc) return rc;
            rc = filter<5>(R, ws, Lo, 1, Vb, Q, blk, labels, R.wb, 2, T, st);
            if (rc) return rc;
        }
        crf_softmax<<<grid_of(nN, 128), 128, 0, st>>>(B, nN, R.CP, R.G, labels, T, Q);
        IRN_LAUNCH_CHECK("crf_softmax");
    }
    if (tm.on) IRN_CUDA(cudaEventRecord(tm.ev[2], st));
    crf_final<<<grid_of(nN, 128), 128, 0, st>>>(B, nN, R.CP, R.G, Q, labels_out, q_out, conf);
    IRN_LAUNCH_CHECK("crf_final");
    if (tm.on) {
        IRN_CUDA(cudaEventRecord(tm.ev[3], st));
        tm.valid = true;
    }
    return kOk;
}

// sizes (as fill_sizes), the packed image bytes (img_bytes < 0: not given, the one-size entry points) and the pointers every call takes
static int common_checks(int n, const int32_t* hw, int H, int W, Sizes& S, const uint8_t* img, long long img_bytes, void* ws) {
    int bad;
    const int rc = fill_sizes(n, hw, H, W, S, &bad);
    if (rc == 1 && (hw == nullptr || bad < 0)) return fail(kBadArg, "irn crf: bad sizes n=%d H=%d W=%d", n, H, W);
    if (rc == 1) return fail(kBadArg, "irn crf: image %d has size %dx%d", bad, hw[2 * bad], hw[2 * bad + 1]);
    if (rc == 2) return fail(kUnsupported, "irn crf: batch too large (%d images): split it", n);
    if (img_bytes >= 0 && img_bytes != 3 * S.nN)
        return fail(kBadArg, "irn crf: %lld image bytes for images of %lld pixels in all (want 3 bytes per pixel)", img_bytes, S.nN);
    if (int e = check_device_ptr(img, "images")) return e;
    if (int e = check_device_ptr(ws, "workspace")) return e;
    return kOk;
}

// the descriptors and pixel offsets of the batch, in one upload
static int upload_params(const Sizes& S, std::vector<ImgParam>& prm, char* ws, const Layout& Lo, cudaStream_t st) {
    std::vector<char> blob(sizeof(ImgParam) * S.n + 4 * (S.n + 1));
    for (int i = 0; i < S.n; ++i) {
        prm[i].H = S.hw[2 * i];
        prm[i].W = S.hw[2 * i + 1];
        prm[i].pix = S.off[i];
    }
    std::memcpy(blob.data(), prm.data(), sizeof(ImgParam) * S.n);
    std::memcpy(blob.data() + sizeof(ImgParam) * S.n, S.off.data(), 4 * (S.n + 1));
    IRN_CUDA(cudaMemsetAsync(ws + Lo.info, 0, 4, st));
    IRN_CUDA(cudaMemcpyAsync(ws + Lo.prm, blob.data(), blob.size(), cudaMemcpyHostToDevice, st));
    return kOk;
}

static int dense_crf(const char* fn, const uint8_t* img, long long img_bytes, int n, const int32_t* hw, int H, int W,
                     const int32_t* labels, int n_labels, int t, double gt_prob, float gauss_sxy, float gauss_compat, float bil_sxy,
                     float bil_srgb, float bil_compat, int32_t* labels_out, float* q_out, int32_t* vertex_counts, void* workspace,
                     size_t workspace_bytes, cudaStream_t st) {
    launch_counter() = 0;
    if (n_labels < 1 || n_labels > kMaxLabels) return fail(kUnsupported, "%s: n_labels=%d outside [1, %d]", fn, n_labels, kMaxLabels);
    if (t < 0 || !(gt_prob > 0.0 && gt_prob < 1.0) || !(gauss_sxy > 0.f) || !(bil_sxy > 0.f) || !(bil_srgb > 0.f))
        return fail(kBadArg, "%s: bad parameters t=%d gt_prob=%g sxy=%g/%g srgb=%g", fn, t, gt_prob, gauss_sxy, bil_sxy, bil_srgb);
    Sizes S;
    if (int rc = common_checks(n, hw, H, W, S, img, img_bytes, workspace)) return rc;
    const Layout Lo = layout(S, 1, n_labels);
    if (workspace_bytes < Lo.total) return fail(kWorkspace, "irn crf: workspace %zu bytes < %zu", workspace_bytes, Lo.total);
    if (int rc = check_device_ptr(labels, "labels")) return rc;
    if (!labels_out && !q_out) return fail(kBadArg, "%s: no output", fn);
    if (labels_out)
        if (int rc = check_device_ptr(labels_out, "labels_out")) return rc;
    if (q_out)
        if (int rc = check_device_ptr(q_out, "q_out")) return rc;
    char* ws = (char*)workspace;
    const Run R{&S, 1, (n_labels + kCB - 1) / kCB * kCB, t, gauss_compat, bil_compat, gauss_sxy, bil_sxy, bil_srgb};
    std::vector<ImgParam> prm(S.n);
    const double pe = -std::log((double)gt_prob);
    const double ne = n_labels > 1 ? -std::log((1.0 - (double)gt_prob) / (n_labels - 1)) : pe;
    for (auto& p : prm) {
        p = ImgParam{};
        p.n_labels = n_labels;
        p.pe = (float)pe;
        p.ne = (float)ne;
    }
    if (int rc = upload_params(S, prm, ws, Lo, st)) return rc;
    IRN_CUDA(cudaMemcpyAsync(ws + Lo.lab, labels, 4 * S.nN, cudaMemcpyDeviceToDevice, st));
    crf_check_labels<<<grid_of(S.nN, 256), 256, 0, st>>>((const int*)(ws + Lo.lab), S.nN, n_labels, (int*)(ws + Lo.info));
    IRN_LAUNCH_CHECK("crf_check_labels");
    return run_crf(R, img, ws, Lo, labels_out, q_out, nullptr, vertex_counts, st);
}

static int ir_label(const char* fn, const uint8_t* img, long long img_bytes, int n, const int32_t* hw, int H, int W, const float* high_res,
                    long long high_res_elems, const int32_t* keys_host, const int32_t* counts_host, float conf_fg_thres,
                    float conf_bg_thres, uint8_t* out, int32_t* vertex_counts, void* workspace, size_t workspace_bytes, cudaStream_t st) {
    launch_counter() = 0;
    if (!counts_host) return fail(kBadArg, "%s: counts is NULL", fn);
    int max_labels = 1, total_k = 0;
    for (int i = 0; i < n; ++i) {
        if (counts_host[i] < 0 || counts_host[i] + 1 > kMaxLabels)
            return fail(kUnsupported, "%s: image %d has %d classes (at most %d)", fn, i, counts_host[i], kMaxLabels - 1);
        max_labels = counts_host[i] + 1 > max_labels ? counts_host[i] + 1 : max_labels;
        total_k += counts_host[i];
    }
    Sizes S;
    if (int rc = common_checks(n, hw, H, W, S, img, img_bytes, workspace)) return rc;
    const Layout Lo = layout(S, 2, max_labels);
    if (workspace_bytes < Lo.total) return fail(kWorkspace, "irn crf: workspace %zu bytes < %zu", workspace_bytes, Lo.total);
    if (high_res_elems >= 0) {
        long long want = 0;
        for (int i = 0; i < n; ++i) want += (long long)counts_host[i] * S.hw[2 * i] * S.hw[2 * i + 1];
        if (high_res_elems != want)
            return fail(kBadArg, "%s: %lld high_res values for planes of %lld values in all", fn, high_res_elems, want);
    }
    if (total_k > 0)
        if (int rc = check_device_ptr(high_res, "high_res")) return rc;
    if (int rc = check_device_ptr(out, "out")) return rc;
    if (total_k > 0 && !keys_host) return fail(kBadArg, "%s: keys is NULL", fn);
    char* ws = (char*)workspace;
    const Run R{&S, 2, (2 * max_labels + kCB - 1) / kCB * kCB, 10, 3.f, 10.f, 3.f, 50.f, 5.f};
    std::vector<ImgParam> prm(S.n);
    int off = 0;
    long long cam = 0;
    for (int i = 0; i < n; ++i) {
        ImgParam& p = prm[i];
        p = ImgParam{};
        p.n_labels = counts_host[i] + 1;
        p.cam = cam;
        const double pe = -std::log(0.7);
        p.pe = (float)pe;
        p.ne = (float)(p.n_labels > 1 ? -std::log((1.0 - 0.7) / (p.n_labels - 1)) : pe);
        p.keys[0] = 0;                                   // np.pad(keys + 1, (1, 0))
        for (int k = 0; k < counts_host[i]; ++k) p.keys[k + 1] = keys_host[off + k] + 1;
        off += counts_host[i];
        cam += (long long)counts_host[i] * S.hw[2 * i] * S.hw[2 * i + 1];
    }
    if (int rc = upload_params(S, prm, ws, Lo, st)) return rc;
    crf_conf_labels<<<grid_of(S.nN, 128), 128, 0, st>>>(batch_view(R, ws, Lo), S.nN, high_res, conf_fg_thres, conf_bg_thres,
                                                        (int*)(ws + Lo.lab));
    IRN_LAUNCH_CHECK("crf_conf_labels");
    return run_crf(R, img, ws, Lo, nullptr, nullptr, out, vertex_counts, st);
}

static size_t ws_bytes_of(int n, const int32_t* hw, int H, int W, int n_groups, int max_labels) {
    Sizes S;
    int bad;
    if (n_groups < 1 || n_groups > 2 || max_labels < 1 || max_labels > kMaxLabels || fill_sizes(n, hw, H, W, S, &bad) != 0) return 0;
    return layout(S, n_groups, max_labels).total;
}

}  // namespace crf
}  // namespace irn

using namespace irn;
using namespace irn::crf;

extern "C" size_t irn_crf_workspace_bytes(int n, int H, int W, int n_groups, int max_labels) {
    return ws_bytes_of(n, nullptr, H, W, n_groups, max_labels);
}

extern "C" size_t irn_crf_ragged_workspace_bytes(int n, const int32_t* sizes_hw, int n_groups, int max_labels) {
    if (!sizes_hw) return 0;
    return ws_bytes_of(n, sizes_hw, 0, 0, n_groups, max_labels);
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
                             float* q_out, int32_t* vertex_counts, void* workspace, size_t workspace_bytes, irn_stream_t stream) {
    return dense_crf("irn_dense_crf", img, -1, n, nullptr, H, W, labels, n_labels, t, gt_prob, gauss_sxy, gauss_compat, bil_sxy,
                     bil_srgb, bil_compat, labels_out, q_out, vertex_counts, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int irn_dense_crf_ragged(const uint8_t* img, size_t img_bytes, const int32_t* sizes_hw, int n, const int32_t* labels,
                                    int n_labels, int t, double gt_prob, float gauss_sxy, float gauss_compat, float bil_sxy,
                                    float bil_srgb, float bil_compat, int32_t* labels_out, float* q_out, int32_t* vertex_counts,
                                    void* workspace, size_t workspace_bytes, irn_stream_t stream) {
    if (!sizes_hw) return fail(kBadArg, "irn_dense_crf_ragged: sizes is NULL");
    return dense_crf("irn_dense_crf_ragged", img, (long long)img_bytes, n, sizes_hw, 0, 0, labels, n_labels, t, gt_prob, gauss_sxy,
                     gauss_compat, bil_sxy, bil_srgb, bil_compat, labels_out, q_out, vertex_counts, workspace, workspace_bytes,
                     (cudaStream_t)stream);
}

extern "C" int irn_ir_label(const uint8_t* img, const float* high_res, const int32_t* keys_host, const int32_t* counts_host, int n,
                            int H, int W, float conf_fg_thres, float conf_bg_thres, uint8_t* out, int32_t* vertex_counts,
                            void* workspace, size_t workspace_bytes, irn_stream_t stream) {
    return ir_label("irn_ir_label", img, -1, n, nullptr, H, W, high_res, -1, keys_host, counts_host, conf_fg_thres, conf_bg_thres, out,
                    vertex_counts, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int irn_ir_label_ragged(const uint8_t* img, size_t img_bytes, const int32_t* sizes_hw, int n, const float* high_res,
                                   size_t high_res_elems, const int32_t* keys_host, const int32_t* counts_host, float conf_fg_thres,
                                   float conf_bg_thres, uint8_t* out, int32_t* vertex_counts, void* workspace, size_t workspace_bytes,
                                   irn_stream_t stream) {
    if (!sizes_hw) return fail(kBadArg, "irn_ir_label_ragged: sizes is NULL");
    return ir_label("irn_ir_label_ragged", img, (long long)img_bytes, n, sizes_hw, 0, 0, high_res, (long long)high_res_elems, keys_host,
                    counts_host, conf_fg_thres, conf_bg_thres, out, vertex_counts, workspace, workspace_bytes, (cudaStream_t)stream);
}
