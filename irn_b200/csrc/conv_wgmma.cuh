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
// Work item: M = 8x16 output pixels (128 rows) x N = BN in {64, 128} output channels, K walked in k-blocks per filter tap.  CTAs are
// persistent (grid = co-resident CTAs): each walks the work items with stride gridDim.x through one shared-memory ring.
//   warpgroup 0      one thread issues TMA: activations as 4-D boxes {32 ch, 16 px, 8 rows, 1 image} (zero fill outside the image =
//                    padding, element strides = stride-2 convs), the weight planes hi / lo as 2-D boxes {128 B of k, BN rows}; all
//                    SWIZZLE_128B, which is the canonical K-major layout wgmma reads from shared memory.  It runs on into the next
//                    work item while the consumers finish the current one.  setmaxnreg gives its registers to the consumers.
//   warpgroups 1, 2  consumers, 64 tile rows each: per k-step each thread loads its A fragment (fp32) straight from the swizzled
//                    TMA tile, splits it in registers into hi / lo, and issues 3 wgmma with A from registers and B from shared
//                    memory; the next k-step is loaded and split while those run.  Epilogue from the register accumulator.
// Accumulation: the tensor core's fp32 accumulate truncates, so the products of one k-block go into a fresh accumulator that is
// then added to the running sum in IEEE fp32: the truncation error is that of 12 MMAs into one partial sum instead of one per
// MMA of the whole reduction.  Two such partial accumulators alternate, so one k-block is added while the next one's MMAs run.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <type_traits>

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
    int stem = 0;                    // 1: 7x7/s2 stem over the zero-haloed NHWC4 input, k-blocks = filter rows (nets.cu, run_stem)
};

template <bool F16, int BN>
struct WgCfg {
    static constexpr int kBK = F16 ? kBfBK : kTcBK;
    static constexpr int kARaw = F16 ? 32768 : 16384;     // fp32 activations: 128 rows x 128 B per 32 channels
    static constexpr int kBBytes = BN * 128;              // one weight plane
    static constexpr int kStageBytes = kARaw + 2 * kBBytes;
    static constexpr int kMaxSmem = 227 * 1024;
    static constexpr int kBarBytes = 256;                 // full[S] + empty[S] mbarriers
    static constexpr int kStages = (kMaxSmem - 1024 - kBarBytes) / kStageBytes;   // f16x3: 3 (BN 128) / 4; 3xTF32: 4 / 7
    static constexpr size_t kSmem = 1024 + (size_t)kStages * kStageBytes + kBarBytes;
    static_assert(kStages >= 2, "shared memory holds at least two stages");
    static_assert(2 * kStages * 8 <= kBarBytes, "barrier area holds full[S] and empty[S]");
    static_assert(BN == 64 || BN == 128, "N tile 64 or 128");
};
constexpr int kWgProducerRegs = 40, kWgConsumerRegs = 232;   // setmaxnreg: 128 x 40 + 256 x 232 <= 64K registers

#ifdef __CUDACC__
// K-major SWIZZLE_128B operand: 8-row groups of 1024 B (stride byte offset), leading byte offset unused for swizzled K-major
__device__ __forceinline__ uint64_t wg_desc(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void wg_fence_regs(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D(64 x N, fp32 registers) (+)= A(64 x K, registers: this thread's fragment) * B(N x K, smem desc)^T; scale_d = 0 overwrites D
template <bool F16, int N>
__device__ __forceinline__ void wg_mma(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d);

template <> __device__ __forceinline__ void wg_mma<false, 64>(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}

template <> __device__ __forceinline__ void wg_mma<false, 128>(float (&d)[64], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, {%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}

template <> __device__ __forceinline__ void wg_mma<true, 64>(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}

template <> __device__ __forceinline__ void wg_mma<true, 128>(float (&d)[64], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
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

// The fp32 values of this thread's wgmma A fragment for k-step k (0..3) of a k-block, in register order.  `row` points at byte
// (tile row 64 g + 16 w + lane/4, in-chunk offset) of the stage's fp32 tile, the other row of the fragment is 8 rows (1 KB)
// further; key = row & 7 is the SWIZZLE_128B key of both.
//   f16x3   k-step = 16 channels, v[0..7]: {row, row + 8, row (+8 ch), row + 8 (+8 ch)} x channels 2 (lane%4) + {0, 1}; 4 LDS.64
//   3xTF32  k-step = 8 channels,  v[0..3]: {row, row + 8, row (+4 ch), row + 8 (+4 ch)} at channel lane%4; 4 LDS.32
template <bool F16>
__device__ __forceinline__ void wg_load_frag(const unsigned char* row, int k, int key, int t4, float (&v)[8]) {
    if (F16) {
        const unsigned char* box = row + (k >> 1) * 16384;       // channels 0-31 | 32-63 of the k-block
        const int c = 4 * (k & 1) + (t4 >> 1);                    // 16-byte chunk of the first channel pair
        const float2 x0 = *reinterpret_cast<const float2*>(box + ((c ^ key) << 4));
        const float2 x1 = *reinterpret_cast<const float2*>(box + 1024 + ((c ^ key) << 4));
        const float2 x2 = *reinterpret_cast<const float2*>(box + (((c + 2) ^ key) << 4));
        const float2 x3 = *reinterpret_cast<const float2*>(box + 1024 + (((c + 2) ^ key) << 4));
        v[0] = x0.x; v[1] = x0.y; v[2] = x1.x; v[3] = x1.y; v[4] = x2.x; v[5] = x2.y; v[6] = x3.x; v[7] = x3.y;
    } else {
        const int c = 2 * k;
        v[0] = *reinterpret_cast<const float*>(row + ((c ^ key) << 4));
        v[1] = *reinterpret_cast<const float*>(row + 1024 + ((c ^ key) << 4));
        v[2] = *reinterpret_cast<const float*>(row + (((c + 1) ^ key) << 4));
        v[3] = *reinterpret_cast<const float*>(row + 1024 + (((c + 1) ^ key) << 4));
    }
}

// fragment values -> the hi and lo A operand registers (f16x3: packed fp16 pairs; 3xTF32: tf32 in fp32 bit patterns)
template <bool F16>
__device__ __forceinline__ void wg_split_frag(const float (&v)[8], uint32_t (&hi)[4], uint32_t (&lo)[4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if (F16) {
            f16_split2(v[2 * i], v[2 * i + 1], hi[i], lo[i]);
        } else {
            const float h = tf32_hi(v[i]);
            hi[i] = __float_as_uint(h);
            lo[i] = __float_as_uint(v[i] - h);
        }
    }
}

template <bool F16, int BN>
__global__ void __launch_bounds__(kWgThreads, 1)
conv_wg_kernel(const __grid_constant__ TcMaps maps, const TcArgs args) {
    using Cfg = WgCfg<F16, BN>;
    constexpr int S = Cfg::kStages;
    constexpr int R = BN / 2;                       // accumulator registers per thread (64 x BN per warpgroup)
    extern __shared__ unsigned char wg_smem_raw[];
    unsigned char* smem = wg_smem_raw + ((1024u - (smem_u32(wg_smem_raw) & 1023u)) & 1023u);   // swizzle atoms need 1 KB alignment
    uint64_t* bars = (uint64_t*)(smem + S * Cfg::kStageBytes);
    uint64_t* full = bars;          // [S] TMA landed
    uint64_t* empty = bars + S;     // [S] both consumer warpgroups finished reading the stage

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // work item = (spatial tile, N tile), N tile fastest: the CTAs that share an activation tile run at the same time and read it
    // from L2.  Persistent CTAs walk the items with stride gridDim.x.
    const int n_tiles = args.Cout / BN;
    const int n_items = args.tiles_x * args.tiles_y * args.B * n_tiles;
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
        // ---- producer: the ring's stage / phase run on across work items, so the next item's loads overlap this one's epilogue
        setmaxnreg_dec<kWgProducerRegs>();
        if (threadIdx.x == 0) {
            tma_prefetch_desc(&maps.a);
            tma_prefetch_desc(&maps.b_hi);
            tma_prefetch_desc(&maps.b_lo);
            if (F16 && args.kb_split < KB) tma_prefetch_desc(&maps.a2);
            int s = 0;
            uint32_t ph = 0;
            for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
                const int tile = item / n_tiles;
                const int ox0 = (tile % args.tiles_x) * kTcTW;
                const int oy0 = ((tile / args.tiles_x) % args.tiles_y) * kTcTH;
                const int b = tile / (args.tiles_x * args.tiles_y);
                const int n0 = (item % n_tiles) * BN;
                for (int kb = 0; kb < KB; ++kb) {
                    mbar_wait(&empty[s], ph ^ 1);
                    unsigned char* st = smem + s * Cfg::kStageBytes;
                    unsigned char* wb = st + Cfg::kARaw;
                    mbar_arrive_expect_tx(&full[s], (uint32_t)Cfg::kStageBytes);
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
                    if (++s == S) { s = 0; ph ^= 1; }
                }
            }
        }
        return;
    }

    // ---- consumers: warpgroup g takes tile rows [64 g, 64 g + 64)
    setmaxnreg_inc<kWgConsumerRegs>();
    const int g = (threadIdx.x >> 7) - 1, wq = warp & 3;
    const int key = lane >> 2, t4 = lane & 3;
    const int frag_off = (64 * g + 16 * wq + key) * 128 + (F16 ? 8 * (t4 & 1) : 4 * t4);
    // The k-blocks of a work item run in pairs: the first accumulates into part[0], the second into part[1].  Each k-step is one
    // wgmma group whose A registers are fa[k & 1]; waiting before k-step k until at most one group is in flight frees fa[k & 1], so
    // the fragments of k-step k are loaded and split while the MMAs of k-step k - 1 run.  At k-step 1 of the second k-block that
    // wait also completes the first, whose part is added to acc (and its stage released) while the second k-block's MMAs run.
    // Only the pair's last part waits for an empty pipe.  (The promotion reads part[0] after a wait issued in the same pair: ptxas
    // serialises every wgmma when an accumulator it cannot prove retired, such as one carried over a loop back edge, is read.)
    float acc[R], part[2][R];
    uint32_t fa[2][2][4];           // [k & 1][hi, lo]
    int s = 0, s_prev = 0;
    uint32_t ph = 0;
    // add part[p] to acc (k-block order) and release the stage of the k-block it holds; its MMAs have completed
    auto promote = [&](auto P) {
        constexpr int p = decltype(P)::value;
        wg_fence_regs(part[p]);
#pragma unroll
        for (int i = 0; i < R; ++i) acc[i] += part[p][i];
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s_prev]);
    };
    auto kblock = [&](auto P) {
        constexpr int p = decltype(P)::value;
        mbar_wait(&full[s], ph);
        unsigned char* st = smem + s * Cfg::kStageBytes;
        const unsigned char* frag = st + frag_off;
        const uint32_t b_hi = smem_u32(st + Cfg::kARaw), b_lo = b_hi + Cfg::kBBytes;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            float v[8];
            wg_load_frag<F16>(frag, k, key, t4, v);
            wg_wait<1>();
            if (p == 1 && k == 1) promote(std::integral_constant<int, 0>());
            wg_split_frag<F16>(v, fa[k & 1][0], fa[k & 1][1]);
            if (k == 0) wg_fence_regs(part[p]);
            wg_fence();
            const uint64_t db_hi = wg_desc(b_hi + 32 * k), db_lo = wg_desc(b_lo + 32 * k);   // 32 bytes of k per instruction
            wg_mma<F16, BN>(part[p], fa[k & 1][0], db_hi, k != 0 ? 1u : 0u);
            wg_mma<F16, BN>(part[p], fa[k & 1][1], db_hi, 1u);
            wg_mma<F16, BN>(part[p], fa[k & 1][0], db_lo, 1u);
            wg_commit();
        }
        s_prev = s;
        if (++s == S) { s = 0; ph ^= 1; }
    };

    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int tile = item / n_tiles;
        const int ox0 = (tile % args.tiles_x) * kTcTW;
        const int oy0 = ((tile / args.tiles_x) % args.tiles_y) * kTcTH;
        const int b = tile / (args.tiles_x * args.tiles_y);
        const int n0 = (item % n_tiles) * BN;
#pragma unroll
        for (int i = 0; i < R; ++i) acc[i] = 0.f;
        int kb = 0;
        for (; kb + 1 < KB; kb += 2) {
            kblock(std::integral_constant<int, 0>());
            kblock(std::integral_constant<int, 1>());
            wg_wait<0>();
            promote(std::integral_constant<int, 1>());
        }
        if (kb < KB) {
            kblock(std::integral_constant<int, 0>());
            wg_wait<0>();
            promote(std::integral_constant<int, 0>());
        }

        // ---- epilogue: fragment (j, h) of thread (warp w, lane l) = tile row 64 g + 16 w + l/4 + 8 h, channels 8 j + 2 (l % 4) + {0, 1}
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
}
#endif  // __CUDACC__

}  // namespace irn
