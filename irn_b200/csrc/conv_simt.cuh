// SIMT fp32 implicit-GEMM convolution (NHWC) and the small glue kernels of the network path.
// This is the exact-fp32 path: every conv the wgmma kernel (conv_wgmma.cuh) does not cover runs
// here, and it is the on-device cross-check for the tensor-core path.
//
// Reference semantics restated (SURVEY.md App. E): cross-correlation, zero padding, no bias;
// FixedBatchNorm (net/resnet50.py:11-14) is folded into (weights, bias) at plan creation.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace irn {

struct ConvGeom {
    int B, H, W, Cin;        // input NHWC
    int Ho, Wo, Cout;        // output NHWC
    int k, stride, pad;
};

constexpr int kBM = 128, kBN = 64, kBK = 16;

// out[m][n] = act( sum_k A[m][k] * Wt[k][n] + bias[n] + residual[m][n] ),  m = (b,oy,ox), k = (r,s,c)
// Wt: [k*k*Cin][Cout] row-major.  VEC: Cin % 16 == 0 (a 16-wide k slice never straddles a filter tap).
template <bool VEC>
__global__ void __launch_bounds__(256)
conv_simt_kernel(const float* __restrict__ in, const float* __restrict__ wt, const float* __restrict__ bias,
                 const float* __restrict__ residual, float* __restrict__ out, ConvGeom g, int relu) {
    __shared__ __align__(16) float As[kBK][kBM + 4];
    __shared__ __align__(16) float Bs[kBK][kBN];
    const int tid = threadIdx.x;
    const int M = g.B * g.Ho * g.Wo;
    const int K = g.k * g.k * g.Cin;
    const int m0 = blockIdx.x * kBM, n0 = blockIdx.y * kBN;

    // A-load role: thread loads 8 consecutive k for one row
    const int a_row = tid >> 1, a_k0 = (tid & 1) * 8;
    const int am = m0 + a_row;
    int ab = 0, aoy = 0, aox = 0;
    const bool a_valid = am < M;
    if (a_valid) {
        ab = am / (g.Ho * g.Wo);
        const int rem = am % (g.Ho * g.Wo);
        aoy = rem / g.Wo;
        aox = rem % g.Wo;
    }
    // B-load role: thread loads 4 consecutive n for one k
    const int b_k = tid >> 4, b_n = (tid & 15) * 4;

    // compute role: 8 rows x 4 cols
    const int tm = (tid >> 4) * 8, tn = (tid & 15) * 4;
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < K; k0 += kBK) {
        // ---- A tile
        float av[8];
        if (VEC) {
            const int kk = k0 + a_k0;            // whole 8-slice lies in one tap
            const int tap = kk / g.Cin, c = kk % g.Cin;
            const int r = tap / g.k, s = tap % g.k;
            const int iy = aoy * g.stride - g.pad + r, ix = aox * g.stride - g.pad + s;
            if (a_valid && iy >= 0 && iy < g.H && ix >= 0 && ix < g.W) {
                const float4* p = reinterpret_cast<const float4*>(in + (((size_t)ab * g.H + iy) * g.W + ix) * g.Cin + c);
                const float4 v0 = __ldg(p), v1 = __ldg(p + 1);
                av[0] = v0.x; av[1] = v0.y; av[2] = v0.z; av[3] = v0.w;
                av[4] = v1.x; av[5] = v1.y; av[6] = v1.z; av[7] = v1.w;
            } else {
#pragma unroll
                for (int i = 0; i < 8; ++i) av[i] = 0.f;
            }
        } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int kk = k0 + a_k0 + i;
                float v = 0.f;
                if (a_valid && kk < K) {
                    const int tap = kk / g.Cin, c = kk % g.Cin;
                    const int r = tap / g.k, s = tap % g.k;
                    const int iy = aoy * g.stride - g.pad + r, ix = aox * g.stride - g.pad + s;
                    if (iy >= 0 && iy < g.H && ix >= 0 && ix < g.W) v = __ldg(in + (((size_t)ab * g.H + iy) * g.W + ix) * g.Cin + c);
                }
                av[i] = v;
            }
        }
        // ---- B tile
        float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
        {
            const int kk = k0 + b_k, n = n0 + b_n;
            if (kk < K) {
                if (n + 3 < g.Cout && (g.Cout & 3) == 0) {
                    bv = __ldg(reinterpret_cast<const float4*>(wt + (size_t)kk * g.Cout + n));
                } else {
                    float t[4] = {0.f, 0.f, 0.f, 0.f};
                    for (int j = 0; j < 4; ++j)
                        if (n + j < g.Cout) t[j] = __ldg(wt + (size_t)kk * g.Cout + n + j);
                    bv = make_float4(t[0], t[1], t[2], t[3]);
                }
            }
        }
        __syncthreads();   // previous tile fully consumed
#pragma unroll
        for (int i = 0; i < 8; ++i) As[a_k0 + i][a_row] = av[i];
        *reinterpret_cast<float4*>(&Bs[b_k][b_n]) = bv;
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < kBK; ++kk) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[kk][tm]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[kk][tm + 4]);
            const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tn]);
            const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
        }
    }
    // ---- epilogue
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int m = m0 + tm + i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tn + j;
            if (n >= g.Cout) continue;
            float v = acc[i][j];
            if (bias) v += bias[n];
            if (residual) v += residual[(size_t)m * g.Cout + n];
            if (relu) v = fmaxf(v, 0.f);
            out[(size_t)m * g.Cout + n] = v;
        }
    }
}

// NCHW fp32 -> NHWC fp32, optionally zero-padding to (Hp, Wp) on the right/bottom
// (EdgeDisplacement pads its input to crop_size, net/resnet50_irn.py:226).
__global__ void nchw_to_nhwc_pad_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int C, int H, int W,
                                        int Hp, int Wp) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t total = (size_t)B * Hp * Wp * C;
    if (i >= total) return;
    const int c = (int)(i % C);
    size_t r = i / C;
    const int x = (int)(r % Wp);
    r /= Wp;
    const int y = (int)(r % Hp);
    const int b = (int)(r / Hp);
    out[i] = (y < H && x < W) ? in[(((size_t)b * C + c) * H + y) * W + x] : 0.f;
}

// NCHW fp32 [B,3,H,W] -> zero-haloed NHWC4 [B, Hin+6, Win+8, 4] for the tensor-core stem: pixel (y,x) lands at
// (y+3, x+3), channel 3 and everything outside the real HxW image is 0 (conv zero padding + IRNet's crop padding).
__global__ void nchw_to_nhwc4_halo_kernel(const float* __restrict__ in, float4* __restrict__ out, int B, int H, int W, int Hp, int Wp) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t total = (size_t)B * Hp * Wp;
    if (i >= total) return;
    const int px = (int)(i % Wp);
    const int py = (int)((i / Wp) % Hp);
    const int b = (int)(i / ((size_t)Wp * Hp));
    const int x = px - 3, y = py - 3;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (x >= 0 && x < W && y >= 0 && y < H) {
        const size_t plane = (size_t)H * W;
        const float* p = in + (size_t)b * 3 * plane + (size_t)y * W + x;
        v.x = p[0];
        v.y = p[plane];
        v.z = p[2 * plane];
    }
    out[i] = v;
}

// MaxPool2d(3, stride 2, pad 1), -inf padding (net/resnet50.py:66).  NHWC, C % 4 == 0.
__global__ void maxpool3s2_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int H, int W, int C, int Ho, int Wo) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int C4 = C >> 2;
    const size_t total = (size_t)B * Ho * Wo * C4;
    if (i >= total) return;
    const int c4 = (int)(i % C4);
    size_t r = i / C4;
    const int ox = (int)(r % Wo);
    r /= Wo;
    const int oy = (int)(r % Ho);
    const int b = (int)(r / Ho);
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    for (int dy = -1; dy <= 1; ++dy) {
        const int iy = 2 * oy + dy;
        if (iy < 0 || iy >= H) continue;
        for (int dx = -1; dx <= 1; ++dx) {
            const int ix = 2 * ox + dx;
            if (ix < 0 || ix >= W) continue;
            const float4 v = __ldg(reinterpret_cast<const float4*>(in + (((size_t)b * H + iy) * W + ix) * C) + c4);
            m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
        }
    }
    reinterpret_cast<float4*>(out + (((size_t)b * Ho + oy) * Wo + ox) * C)[c4] = m;
}

// 1x1 conv with few outputs (N <= 32): one warp per pixel, lanes stride over Cin.
//   w: [N][Cin];  y[pix][n] = sum_c x[pix][c] * w[n][c] (+ bias[n]) (- shift[n])
template <int N>
__device__ __forceinline__ void smalln_dot(const float* __restrict__ x, const float* __restrict__ w, int Cin, int lane, float (&acc)[N]) {
#pragma unroll
    for (int n = 0; n < N; ++n) acc[n] = 0.f;
    for (int c = lane; c < Cin; c += 32) {
        const float a = __ldg(x + c);
#pragma unroll
        for (int n = 0; n < N; ++n) acc[n] = fmaf(a, __ldg(w + (size_t)n * Cin + c), acc[n]);
    }
#pragma unroll
    for (int n = 0; n < N; ++n)
#pragma unroll
        for (int o = 16; o; o >>= 1) acc[n] += __shfl_xor_sync(0xffffffffu, acc[n], o);
}

template <int N>
__global__ void conv1x1_smalln_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                      const float* __restrict__ shift, float* __restrict__ y, size_t n_pix, int Cin) {
    const size_t pix = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (pix >= n_pix) return;
    float acc[N];
    smalln_dot<N>(x + pix * Cin, w, Cin, lane, acc);
    if (lane == 0) {
#pragma unroll
        for (int n = 0; n < N; ++n) {
            float v = acc[n];
            if (bias) v += bias[n];
            if (shift) v -= shift[n];
            y[pix * N + n] = v;
        }
    }
}

// CAM head (net/resnet50_cam.py:65-68): relu(conv1x1 2048->20) of sample 2p at (y,x) plus the same of the
// flipped sample 2p+1 at (y, w-1-x).  feat NHWC [2P,h,w,Cin] -> out NCHW-like [P,20,h,w].
__global__ void cam_head_kernel(const float* __restrict__ feat, const float* __restrict__ w, float* __restrict__ out, int P, int h,
                                int wd, int Cin) {
    const size_t wid = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const size_t n_pix = (size_t)P * h * wd;
    if (wid >= n_pix) return;
    const int x = (int)(wid % wd);
    const int y = (int)((wid / wd) % h);
    const int p = (int)(wid / ((size_t)wd * h));
    float a0[20], a1[20];
    smalln_dot<20>(feat + ((((size_t)(2 * p) * h + y) * wd) + x) * Cin, w, Cin, lane, a0);
    smalln_dot<20>(feat + ((((size_t)(2 * p + 1) * h + y) * wd) + (wd - 1 - x)) * Cin, w, Cin, lane, a1);
    if (lane == 0) {
#pragma unroll
        for (int n = 0; n < 20; ++n) out[(((size_t)p * 20 + n) * h + y) * wd + x] = fmaxf(a0[n], 0.f) + fmaxf(a1[n], 0.f);
    }
}

// CAM head tail for the tensor-core path: y = relu(classifier(x)) is already in t NHWC [2P,h,w,C] (first 20 channels real);
// out[p,n,y,x] = t[2p,y,x,n] + t[2p+1,y,w-1-x,n]      (net/resnet50_cam.py:68)
__global__ void cam_flip_add_kernel(const float* __restrict__ t, float* __restrict__ out, int P, int h, int w, int C) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)P * 20 * h * w) return;
    const int x = (int)(i % w);
    const int y = (int)((i / w) % h);
    const int n = (int)((i / ((size_t)w * h)) % 20);
    const int p = (int)(i / ((size_t)w * h * 20));
    const float a = t[(((size_t)(2 * p) * h + y) * w + x) * C + n];
    const float b = t[(((size_t)(2 * p + 1) * h + y) * w + (w - 1 - x)) * C + n];
    out[i] = a + b;
}

// GroupNorm statistics, pass 1: per (sample, group) sum and sum of squares in fp64.  grid (slices, B), 256 threads;
// thread t owns channel t % C of every (256/C)-th pixel of its slice, so global reads are fully coalesced; the
// per-channel partials are folded per group through shared-memory atomics, then one atomicAdd per group per block.
// x NHWC [B,HW,C], C in {32,64,128,256}; sums[(b*G+g)*2 + {0,1}] must be zeroed beforehand.
__global__ void __launch_bounds__(256)
gn_partial_kernel(const float* __restrict__ x, double* __restrict__ sums, int HW, int C, int G) {
    __shared__ double sh[32][2];
    const int b = blockIdx.y;
    const int c = threadIdx.x % C, prow = threadIdx.x / C, pstep = 256 / C;
    const int per = (HW + gridDim.x - 1) / gridDim.x;
    const int p0 = blockIdx.x * per, p1 = min(p0 + per, HW);
    if (threadIdx.x < 32) sh[threadIdx.x][0] = sh[threadIdx.x][1] = 0.0;
    __syncthreads();
    double s = 0.0, ss = 0.0;
    for (int p = p0 + prow; p < p1; p += pstep) {
        const double v = (double)x[((size_t)b * HW + p) * C + c];
        s += v;
        ss += v * v;
    }
    const int cpg = C / G;            // 8 or 16 consecutive lanes share a group (C >= 32, so a warp never wraps channels)
    for (int o = 1; o < cpg; o <<= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        ss += __shfl_xor_sync(0xffffffffu, ss, o);
    }
    const int g = c / cpg;
    if ((c % cpg) == 0) {
        atomicAdd(&sh[g][0], s);
        atomicAdd(&sh[g][1], ss);
    }
    __syncthreads();
    if (threadIdx.x < G) {
        atomicAdd(&sums[(size_t)(b * G + threadIdx.x) * 2], sh[threadIdx.x][0]);
        atomicAdd(&sums[(size_t)(b * G + threadIdx.x) * 2 + 1], sh[threadIdx.x][1]);
    }
}

// GroupNorm affine -> bilinear upsample by `up` (align_corners=False) -> ReLU, written into a channel slice
// of a concat buffer, cropped to (Hd, Wd)   (net/resnet50_irn.py:23-93,117-131: conv -> GN -> Upsample -> ReLU).
// One thread = 4 consecutive channels (same group: groups hold >= 8 channels); coff and Cd are multiples of 4.
__global__ void gn_up_relu_kernel(const float* __restrict__ x, const double* __restrict__ sums, const float* __restrict__ gamma,
                                  const float* __restrict__ beta, float* __restrict__ dst, int B, int H, int W, int C, int G, int up,
                                  int Hd, int Wd, int Cd, int coff) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int C4 = C >> 2;
    const size_t total = (size_t)B * Hd * Wd * C4;
    if (i >= total) return;
    const int c = (int)(i % C4) * 4;
    size_t r = i / C4;
    const int X = (int)(r % Wd);
    r /= Wd;
    const int Y = (int)(r % Hd);
    const int b = (int)(r / Hd);
    const int g = c / (C / G);
    // biased variance over the (C/G)*H*W elements of the group, eps inside the sqrt (torch GroupNorm)
    const double cnt = (double)H * W * (C / G);
    const double mu = sums[2 * (b * G + g)] / cnt;
    double var = sums[2 * (b * G + g) + 1] / cnt - mu * mu;
    var = var < 0.0 ? 0.0 : var;
    const float mean = (float)mu, rstd = (float)(1.0 / sqrt(var + 1e-5));
    const float4 ga = *reinterpret_cast<const float4*>(gamma + c), be = *reinterpret_cast<const float4*>(beta + c);
    const float* xb = x + (size_t)b * H * W * C + c;
    auto norm = [&](const float4 v) {
        float4 o;
        o.x = (v.x - mean) * rstd * ga.x + be.x;
        o.y = (v.y - mean) * rstd * ga.y + be.y;
        o.z = (v.z - mean) * rstd * ga.z + be.z;
        o.w = (v.w - mean) * rstd * ga.w + be.w;
        return o;
    };
    auto ld = [&](int yy, int xx) { return norm(__ldg(reinterpret_cast<const float4*>(xb + ((size_t)yy * W + xx) * C))); };
    float4 v;
    if (up == 1) {
        v = ld(Y, X);
    } else {
        const float inv = 1.0f / (float)up;
        float sy = ((float)Y + 0.5f) * inv - 0.5f, sx = ((float)X + 0.5f) * inv - 0.5f;
        sy = sy < 0.f ? 0.f : sy;
        sx = sx < 0.f ? 0.f : sx;
        int y0 = (int)sy, x0 = (int)sx;
        y0 = y0 > H - 1 ? H - 1 : y0;
        x0 = x0 > W - 1 ? W - 1 : x0;
        const int y1 = y0 + (y0 < H - 1), x1 = x0 + (x0 < W - 1);
        const float ly = sy - (float)y0, lx = sx - (float)x0;
        const float4 v00 = ld(y0, x0), v01 = ld(y0, x1), v10 = ld(y1, x0), v11 = ld(y1, x1);
        v.x = (1.f - ly) * ((1.f - lx) * v00.x + lx * v01.x) + ly * ((1.f - lx) * v10.x + lx * v11.x);
        v.y = (1.f - ly) * ((1.f - lx) * v00.y + lx * v01.y) + ly * ((1.f - lx) * v10.y + lx * v11.y);
        v.z = (1.f - ly) * ((1.f - lx) * v00.z + lx * v01.z) + ly * ((1.f - lx) * v10.z + lx * v11.z);
        v.w = (1.f - ly) * ((1.f - lx) * v00.w + lx * v01.w) + ly * ((1.f - lx) * v10.w + lx * v11.w);
    }
    v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
    *reinterpret_cast<float4*>(dst + (((size_t)b * Hd + Y) * Wd + X) * Cd + coff + c) = v;
}

// EdgeDisplacement tail (net/resnet50_irn.py:228-234) for pair p = blockIdx.y: crop to (fh,fw);
// edge = sigmoid(e[2p]/2 + flip(e[2p+1])/2); dp = dp[2p]
//   e NHWC [2P,Hf,Wf,1], d NHWC [2P,Hf,Wf,2]  ->  edge [P,fh,fw], dp [P,2,fh,fw]
__global__ void edge_dp_tail_kernel(const float* __restrict__ e, const float* __restrict__ d, float* __restrict__ edge,
                                    float* __restrict__ dp, int Hf, int Wf, int fh, int fw) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int p = blockIdx.y;
    if (i >= fh * fw) return;
    const int y = i / fw, x = i % fw;
    const size_t plane = (size_t)Hf * Wf;
    const float* e0 = e + (size_t)(2 * p) * plane;
    const float* e1 = e0 + plane;
    const float* d0 = d + (size_t)(2 * p) * plane * 2;
    const float a = e0[(size_t)y * Wf + x] / 2.f + e1[(size_t)y * Wf + (fw - 1 - x)] / 2.f;
    edge[(size_t)p * fh * fw + i] = 1.f / (1.f + expf(-a));
    dp[((size_t)p * 2) * fh * fw + i] = d0[((size_t)y * Wf + x) * 2];
    dp[((size_t)p * 2 + 1) * fh * fw + i] = d0[((size_t)y * Wf + x) * 2 + 1];
}

}  // namespace irn
