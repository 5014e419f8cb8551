// wgmma implicit-GEMM convolution for sm_90a: NHWC fp32 activations in and out, split-precision tensor-core arithmetic.
//
//   out[b,oy,ox,n] = act( oscale[n] * sum_{r,s,c} in[b, oy*st-pad+r, ox*st-pad+s, c] * w[n,(r,s,c)] + bias[n] + residual )
//
// Every product is evaluated as  a*w ~= a_hi*w_hi + a_lo*w_hi + a_hi*w_lo  with one of two operand splits (w split on the host):
//   3xTF32 (F16 = false)  a_hi = tf32(a) (round to nearest), a_lo = a - a_hi; wgmma kind tf32, K = 8 per instruction,
//                         32-channel k-blocks
//   f16x3  (F16 = true)   a_hi = fp16(a) (truncated), a_lo = fp16(a - a_hi); the weights are pre-scaled per output channel by a
//                         power of two (undone exactly by `oscale`); K = 16 per instruction, 64-channel k-blocks: half the tensor
//                         time of 3xTF32.  Activations beyond +-65504 saturate (ResNet-50 activations stay far below).
// fp16 and tf32 carry the same 11 significant bits, so both splits keep ~22 bits per operand; plain TF32 misses the 1e-4 CAM
// parity bar by ~20x.
//
// GEMM tile per CTA: M = 8x16 output pixels (128 rows), N = BN in {64, 128} output channels, K walked in k-blocks per filter tap.
//   warpgroup 0      one thread issues TMA: activations as 4-D boxes {32 ch, 16 px, 8 rows, 1 image} (zero fill outside the image =
//                    padding, element strides = stride-2 convs), the weight planes hi / lo as 2-D boxes {128 B of k, BN rows}; all
//                    SWIZZLE_128B, which is the canonical K-major layout wgmma reads from shared memory
//   warpgroups 1, 2  consumers, 64 tile rows each: split their rows of the activation k-block into hi / lo planes in shared
//                    memory, then 4 k-steps x 3 wgmma (A and B from shared memory) into a register accumulator; epilogue
// Accumulation: the tensor core's fp32 accumulate truncates, so the products of one k-block go into a fresh accumulator that is
// then added to the running sum in IEEE fp32: the truncation error is that of 12 MMAs into one partial sum instead of one per
// MMA of the whole reduction.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>

#include "tma.cuh"

namespace irn {

constexpr int kTcTW = 16, kTcTH = 8;          // spatial tile: 128 output pixels
constexpr int kTcBK = 32;                     // 3xTF32: fp32 channels per k-block = 128 bytes = one swizzle atom row
constexpr int kBfBK = 64;                     // f16x3: channels per k-block = 128 bytes of fp16
constexpr int kWgThreads = 384;               // producer warpgroup + two consumer warpgroups

struct TcMaps {
    CUtensorMap a;      // input  {Cin, W, H, B}
    CUtensorMap b_hi;   // weights {K, Cout}
    CUtensorMap b_lo;
    CUtensorMap a2;     // f16x3 only: second input of a K-concatenated 1x1 conv (TcArgs::kb_split); unused otherwise
};

struct TcArgs {
    const float* bias;
    const float* residual;
    float* out;
    int B, Ho, Wo, Cout, Cin, ksize, stride, pad, relu;
    int tiles_x, tiles_y;
    int kb_split = 1 << 30;          // f16x3 only: k-blocks [kb_split, KB) read input `a2` (pixel stride `stride2`): the projection
    int stride2 = 1;                 // shortcut of a bottleneck fused into conv3's reduction (nets.cu, Block::c3ds)
    const float* oscale = nullptr;   // f16x3 only: per-output-channel factor undoing the weights' power-of-two pre-scale
    int stem = 0;                    // 1: 7x7/s2 stem over the zero-haloed NHWC4 input, k-blocks = filter rows (nets.cu, launch_*_stem)
};

template <bool F16, int BN>
struct WgCfg {
    static constexpr int kBK = F16 ? kBfBK : kTcBK;
    static constexpr int kARaw = F16 ? 32768 : 16384;     // fp32 activations: 128 rows x 128 B per 32 channels
    static constexpr int kALo = F16 ? 0 : 16384;          // 3xTF32: lo plane (the hi plane overwrites the raw tile in place)
    static constexpr int kBBytes = BN * 128;              // one weight plane
    static constexpr int kStageBytes = kARaw + kALo + 2 * kBBytes;
    static constexpr int kSplitBytes = F16 ? 32768 : 0;   // f16x3: fp16 hi | lo planes of the current k-block (128 rows x 128 B each)
    static constexpr int kMaxSmem = 227 * 1024;
    static constexpr int kFit = (kMaxSmem - 1024 - 256 - kSplitBytes) / kStageBytes;
    static constexpr int kStages = kFit > 4 ? 4 : kFit;
    static constexpr size_t kSmem = 1024 + (size_t)kStages * kStageBytes + kSplitBytes + 256;
    static_assert(kStages >= 2, "shared memory holds at least two stages");
    static_assert(BN == 64 || BN == 128, "N tile 64 or 128");
};

#ifdef __CUDACC__
// K-major SWIZZLE_128B operand: 8-row groups of 1024 B (stride byte offset), leading byte offset unused for swizzled K-major
__device__ __forceinline__ uint64_t wg_desc(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_fence_regs(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// D(64 x N, fp32 registers) (+)= A(64 x K, smem desc) * B(N x K, smem desc)^T; scale_d = 0 overwrites D
template <bool F16, int N>
__device__ __forceinline__ void wg_mma(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d);

template <> __device__ __forceinline__ void wg_mma<false, 64>(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, %32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d));
}

template <> __device__ __forceinline__ void wg_mma<false, 128>(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d));
}

template <> __device__ __forceinline__ void wg_mma<true, 64>(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d));
}

template <> __device__ __forceinline__ void wg_mma<true, 128>(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d));
}

// tf32 "hi" part of an fp32 value: round to nearest (ties away, like cvt.rna.tf32.f32) on the 13 dropped mantissa bits; the "lo"
// part x - hi is exact in fp32 (<= 13 significant bits) and the tensor core keeps its top 11 bits (error 2^-21 |x|)
__device__ __forceinline__ float tf32_hi(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u); }

// (a, b) -> packed fp16 pair {low half = hi(a), high half = hi(b)} and the packed pair of the residuals.  hi(x) = x truncated to 11
// significant bits (round-toward-zero conversion); the same value rebuilt in fp32 by a mask gives the residual x - hi(x), exact in
// fp32 and rounded once, to 11 bits, by its own conversion: |error| <= 2^-21 |x| for 2^-14 <= |x| <= 65504.
__device__ __forceinline__ void f16_split2(float a, float b, uint32_t& hi, uint32_t& lo) {
    asm("cvt.rz.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(b), "f"(a));      // upper half <- first source operand
    const float ha = __uint_as_float(__float_as_uint(a) & 0xFFFFE000u), hb = __uint_as_float(__float_as_uint(b) & 0xFFFFE000u);
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(b - hb), "f"(a - ha));
}

template <bool F16, int BN>
__global__ void __launch_bounds__(kWgThreads, 1)
conv_wg_kernel(const __grid_constant__ TcMaps maps, const TcArgs args) {
    using Cfg = WgCfg<F16, BN>;
    constexpr int S = Cfg::kStages;
    constexpr int R = BN / 2;                       // accumulator registers per thread (64 x BN per warpgroup)
    extern __shared__ unsigned char wg_smem_raw[];
    unsigned char* smem = wg_smem_raw + ((1024u - (smem_u32(wg_smem_raw) & 1023u)) & 1023u);   // swizzle atoms need 1 KB alignment
    unsigned char* split_buf = smem + S * Cfg::kStageBytes;
    uint64_t* bars = (uint64_t*)(split_buf + Cfg::kSplitBytes);
    uint64_t* full = bars;          // [S] TMA landed
    uint64_t* empty = bars + S;     // [S] both consumer warpgroups finished reading the stage

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_tiles = args.Cout / BN;
    // 1-D grid, N tile fastest: the CTAs that share an activation tile run at the same time and read it from L2
    const int tile = blockIdx.x / n_tiles;
    const int ox0 = (tile % args.tiles_x) * kTcTW;
    const int oy0 = ((tile / args.tiles_x) % args.tiles_y) * kTcTH;
    const int b = tile / (args.tiles_x * args.tiles_y);
    const int n0 = (blockIdx.x % n_tiles) * BN;
    const int cblocks = args.Cin / Cfg::kBK;
    const int KB = (!F16 && args.stem) ? args.ksize : args.ksize * args.ksize * cblocks;

    if (threadIdx.x == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 8);
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ---- producer
        if (threadIdx.x == 0) {
            tma_prefetch_desc(&maps.a);
            tma_prefetch_desc(&maps.b_hi);
            tma_prefetch_desc(&maps.b_lo);
            if (F16 && args.kb_split < KB) tma_prefetch_desc(&maps.a2);
            for (int kb = 0; kb < KB; ++kb) {
                const int s = kb % S;
                mbar_wait(&empty[s], ((kb / S) & 1) ^ 1);
                unsigned char* st = smem + s * Cfg::kStageBytes;
                unsigned char* wb = st + Cfg::kARaw + Cfg::kALo;
                mbar_arrive_expect_tx(&full[s], (uint32_t)(Cfg::kARaw + 2 * Cfg::kBBytes));
                if (args.stem) {
                    // the 32 floats of a box row are the 8 taps x 4 channels of ONE filter row for one output pixel (overlapping
                    // windows); 3xTF32: k-block = filter row kb, f16x3: filter rows 2 kb and 2 kb + 1 (row 7 carries zero weights)
                    const int row = F16 ? 2 * kb : kb;
                    tma_load_4d(st, &maps.a, &full[s], 0, ox0, oy0 * 2 + row, b);
                    if (F16) tma_load_4d(st + 16384, &maps.a, &full[s], 0, ox0, oy0 * 2 + row + 1, b);
                } else {
                    // K-concatenated 1x1 conv: k-blocks from kb_split on come from the second input (its own pixel stride, no padding)
                    const bool second = F16 && kb >= args.kb_split;
                    const CUtensorMap* am = second ? &maps.a2 : &maps.a;
                    const int tap = second ? 0 : kb / cblocks, cb = second ? kb - args.kb_split : kb % cblocks;
                    const int r = tap / args.ksize, ss = tap % args.ksize;
                    const int x = second ? ox0 * args.stride2 : ox0 * args.stride - args.pad + ss;
                    const int y = second ? oy0 * args.stride2 : oy0 * args.stride - args.pad + r;
                    tma_load_4d(st, am, &full[s], cb * Cfg::kBK, x, y, b);
                    if (F16) tma_load_4d(st + 16384, am, &full[s], cb * Cfg::kBK + 32, x, y, b);
                }
                tma_load_2d(wb, &maps.b_hi, &full[s], kb * Cfg::kBK, n0);
                tma_load_2d(wb + Cfg::kBBytes, &maps.b_lo, &full[s], kb * Cfg::kBK, n0);
            }
        }
        return;
    }

    // ---- consumers: warpgroup g takes tile rows [64 g, 64 g + 64)
    const int g = (threadIdx.x >> 7) - 1;
    const int t = threadIdx.x & 127;
    float acc[R], part[R];
#pragma unroll
    for (int i = 0; i < R; ++i) acc[i] = 0.f;

    for (int kb = 0; kb < KB; ++kb) {
        const int s = kb % S;
        unsigned char* st = smem + s * Cfg::kStageBytes;
        mbar_wait(&full[s], (kb / S) & 1);
        uint32_t a_hi, a_lo;
        if (F16) {
            // 64 rows x 8 chunks of 8 channels: raw fp32 (two 32-channel halves, swizzled 16-byte chunks) -> fp16 hi / lo planes
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int i = t + 128 * j;
                const int row = 64 * g + (i >> 3), c = i & 7, key = row & 7;
                const float4* src = reinterpret_cast<const float4*>(st + (c >> 2) * 16384 + row * 128);
                const float4 v0 = src[(2 * (c & 3)) ^ key], v1 = src[(2 * (c & 3) + 1) ^ key];
                uint4 h, l;
                f16_split2(v0.x, v0.y, h.x, l.x);
                f16_split2(v0.z, v0.w, h.y, l.y);
                f16_split2(v1.x, v1.y, h.z, l.z);
                f16_split2(v1.z, v1.w, h.w, l.w);
                const int off = row * 128 + ((c ^ key) << 4);
                *reinterpret_cast<uint4*>(split_buf + off) = h;
                *reinterpret_cast<uint4*>(split_buf + 16384 + off) = l;
            }
            a_hi = smem_u32(split_buf);
            a_lo = a_hi + 16384;
        } else {
            // element-wise, so the swizzle does not matter: hi over the raw tile, lo into its own plane at the same offset
            float4* a = reinterpret_cast<float4*>(st + g * 8192);
            float4* lo = reinterpret_cast<float4*>(st + 16384 + g * 8192);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float4 v = a[t + 128 * j];
                float4 h, l;
                h.x = tf32_hi(v.x); h.y = tf32_hi(v.y); h.z = tf32_hi(v.z); h.w = tf32_hi(v.w);
                l.x = v.x - h.x; l.y = v.y - h.y; l.z = v.z - h.z; l.w = v.w - h.w;
                a[t + 128 * j] = h;
                lo[t + 128 * j] = l;
            }
            a_hi = smem_u32(st);
            a_lo = a_hi + 16384;
        }
        fence_proxy_async();            // generic-proxy writes -> visible to the tensor core (async proxy)
        named_bar_sync(1 + g, 128);     // the whole warpgroup's rows are split
        a_hi += (uint32_t)(g * 8192);
        a_lo += (uint32_t)(g * 8192);
        const uint32_t b_hi = smem_u32(st + Cfg::kARaw + Cfg::kALo), b_lo = b_hi + Cfg::kBBytes;
        wg_fence_regs(part);
        wg_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {   // 32 bytes of k per instruction inside the 128-byte swizzle row
            const uint64_t da_hi = wg_desc(a_hi + 32 * k), da_lo = wg_desc(a_lo + 32 * k);
            const uint64_t db_hi = wg_desc(b_hi + 32 * k), db_lo = wg_desc(b_lo + 32 * k);
            wg_mma<F16, BN>(part, da_hi, db_hi, k != 0 ? 1u : 0u);
            wg_mma<F16, BN>(part, da_lo, db_hi, 1u);
            wg_mma<F16, BN>(part, da_hi, db_lo, 1u);
        }
        wg_commit();
        wg_wait_all();
        wg_fence_regs(part);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
#pragma unroll
        for (int i = 0; i < R; ++i) acc[i] += part[i];
    }

    // ---- epilogue: fragment (j, h) of thread (warp w, lane l) = tile row 64 g + 16 w + l/4 + 8 h, channels 8 j + 2 (l % 4) + {0, 1}
    const int wq = warp & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = 64 * g + 16 * wq + (lane >> 2) + 8 * h;
        const int oy = oy0 + row / kTcTW, ox = ox0 + row % kTcTW;
        if (oy >= args.Ho || ox >= args.Wo) continue;
        const size_t base = (((size_t)b * args.Ho + oy) * args.Wo + ox) * args.Cout + n0 + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int n = n0 + 8 * j + 2 * (lane & 3);
            float2 o = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            if (F16 && args.oscale) {
                // a power of two: the product is exact, so a contracted multiply-add rounds once like the add alone
                const float2 sc = __ldg(reinterpret_cast<const float2*>(args.oscale + n));
                o.x *= sc.x; o.y *= sc.y;
            }
            if (args.bias) {
                const float2 bi = __ldg(reinterpret_cast<const float2*>(args.bias + n));
                o.x += bi.x; o.y += bi.y;
            }
            if (args.residual) {
                const float2 rv = __ldg(reinterpret_cast<const float2*>(args.residual + base + 8 * j));
                o.x += rv.x; o.y += rv.y;
            }
            if (args.relu) {
                o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f);
            }
            *reinterpret_cast<float2*>(args.out + base + 8 * j) = o;
        }
    }
}
#endif  // __CUDACC__

}  // namespace irn
