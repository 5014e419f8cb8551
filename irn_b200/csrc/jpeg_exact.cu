// Exact JPEG decode on the device: baseline Huffman-coded streams of any sizes in one call, uint8 RGB written at caller-given
// offsets, bit-identical to libjpeg-turbo's default decompression as PIL returns it (np.asarray(Image.open(f).convert("RGB"))).
// The arithmetic (islow IDCT, fancy chroma up-sampling, 16-bit YCbCr tables) is restated from ITU-T T.81 and pinned against PIL
// by the oracle, oracle/jpeg.py, whose docstring lists every choice that decides a pixel.
//
// Host work is header parsing only; the entropy-coded segments are uploaded as they are in the files.  Four stages on the device:
//   1. unstuff: per byte, "kept" (not the 00 of FF 00, not part of an RSTn marker) and "is RSTn" flags, one CUB exclusive scan over
//      both packed in 64 bits, then a scatter that writes the kept bytes and the start of every restart interval;
//   2. entropy decode: one CTA per image, one thread per restart interval, Huffman lookup tables in shared memory, int16
//      coefficients per block (natural order) into per-component block planes padded to whole MCUs;
//   3. dequantise + islow IDCT: 8 threads per block (one column in pass 1, one row in pass 2), samples into per-component planes;
//   4. up-sampling + YCbCr->RGB: one thread per output pixel, written at the image's output offset.
// Errors in the entropy-coded data (a marker other than RSTn / stuffing, a missing or surplus restart marker, an invalid Huffman
// code, an AC run past the block, a read past the interval's end) set bits of the image's status word and stop that interval.
#include <cub/cub.cuh>

#include <cstring>
#include <vector>

#include "common.h"

namespace irn {
namespace jx {

constexpr int kMaxComp = 3;

struct Huff {                   // one Huffman table as it appears in a DHT segment
    uint8_t counts[16];
    uint8_t vals[256];
};

struct Desc {                   // one image, built on the host, read by every stage
    int H, W, nc, hs, vs, restart;
    int mcux, mcuy, n_int;      // MCU grid, restart intervals
    int bw[kMaxComp], bh[kMaxComp];     // block grid per component (whole MCUs)
    long long blk0;             // first block of this image in the coefficient buffer (components back to back)
    long long pix0;             // first byte of this image in the plane buffer (components back to back, each bw*8 x bh*8)
    long long raw0;             // first byte of this image's entropy-coded segment in the raw buffer
    long long raw_len;
    long long seg0;             // first entry of this image in the interval-start table (n_int + 1 entries)
    long long out0;             // output byte offset
    uint16_t q[kMaxComp][64];   // natural order
    Huff dc[kMaxComp], ac[kMaxComp];
};

enum : int { kStMarker = 1, kStRestart = 2, kStCode = 4, kStOverrun = 8, kStRun = 16 };

// ------------------------------------------------------------------------------------------------------------------------------
// host: header parse (the one place that knows the supported set; oracle/jpeg.py parse() is its restatement)

struct Header {
    int H = 0, W = 0, nc = 0, hs = 1, vs = 1, restart = 0;
    uint16_t q[kMaxComp][64];
    Huff dc[kMaxComp], ac[kMaxComp];
    size_t scan_start = 0, scan_end = 0;
};

// zig-zag index -> natural (row-major) index
#define IRN_JPEG_ZIGZAG                                                                                                          \
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28, 35, 42, \
        49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63
static const uint8_t kZigzag[64] = {IRN_JPEG_ZIGZAG};
__constant__ uint8_t kZigzagDev[64] = {IRN_JPEG_ZIGZAG};

static bool huff_ok(const Huff& h) {      // the counts fit the canonical code space
    unsigned code = 0;
    for (int l = 1; l <= 16; ++l) {
        code += h.counts[l - 1];
        if (code > (1u << l)) return false;
        code <<= 1;
    }
    return true;
}

static int parse(const uint8_t* d, size_t len, Header& hd) {
    hd = Header{};
    if (!d || len < 4 || d[0] != 0xFF || d[1] != 0xD8) return fail(kBadArg, "jpeg: no SOI marker");
    struct Comp { int id, h, v, tq; } comps[4] = {};
    int nc = 0, H = 0, W = 0, adobe = -1, td[4] = {}, ta[4] = {};
    bool jfif = false, have_sof = false, have_q[4] = {}, have_h[2][4] = {};
    uint16_t qt[4][64];
    Huff ht[2][4];
    size_t p = 2;
    for (;;) {
        if (p >= len || d[p] != 0xFF) return fail(kBadArg, "jpeg: truncated header or missing marker at byte %zu", p);
        while (p < len && d[p] == 0xFF) ++p;
        if (p + 3 > len) return fail(kBadArg, "jpeg: truncated header");
        const int m = d[p++];
        if (m == 0xD8 || m == 0xD9 || (m >= 0xD0 && m <= 0xD7) || m == 0x01) return fail(kBadArg, "jpeg: unexpected marker FF%02X", m);
        const size_t L = (size_t(d[p]) << 8) | d[p + 1];
        if (L < 2 || p + L > len) return fail(kBadArg, "jpeg: truncated marker segment FF%02X", m);
        const uint8_t* s = d + p + 2;
        const size_t sl = L - 2;
        if (m == 0xC0 || m == 0xC1) {
            if (sl < 6) return fail(kBadArg, "jpeg: short SOF");
            if (s[0] != 8) return fail(kUnsupported, "jpeg: %d-bit samples", s[0]);
            H = (s[1] << 8) | s[2];
            W = (s[3] << 8) | s[4];
            nc = s[5];
            if (sl < 6 + 3 * size_t(nc)) return fail(kBadArg, "jpeg: short SOF");
            if (H == 0) return fail(kUnsupported, "jpeg: height defined by DNL");
            if (W == 0 || nc == 0) return fail(kBadArg, "jpeg: zero width or no components");
            if (nc != 1 && nc != 3) return fail(kUnsupported, "jpeg: %d components", nc);
            for (int i = 0; i < nc; ++i) comps[i] = {s[6 + 3 * i], s[7 + 3 * i] >> 4, s[7 + 3 * i] & 15, s[8 + 3 * i]};
            have_sof = true;
        } else if (m == 0xCC) {
            return fail(kUnsupported, "jpeg: arithmetic coding");
        } else if (m >= 0xC2 && m <= 0xCF && m != 0xC4 && m != 0xC8) {
            return fail(kUnsupported, "jpeg: SOF%d (only baseline / extended sequential Huffman)", m - 0xC0);
        } else if (m == 0xC4) {
            for (size_t q = 0; q < sl;) {
                if (q + 17 > sl) return fail(kBadArg, "jpeg: short DHT");
                const int tc = s[q] >> 4, th = s[q] & 15;
                int nv = 0;
                for (int i = 0; i < 16; ++i) nv += s[q + 1 + i];
                if (tc > 1 || th > 3 || nv > 256 || q + 17 + nv > sl) return fail(kBadArg, "jpeg: bad DHT");
                Huff& h = ht[tc][th];
                memset(&h, 0, sizeof(h));
                memcpy(h.counts, s + q + 1, 16);
                memcpy(h.vals, s + q + 17, nv);
                if (!huff_ok(h)) return fail(kBadArg, "jpeg: bad Huffman table");
                have_h[tc][th] = true;
                q += 17 + nv;
            }
        } else if (m == 0xDB) {
            for (size_t q = 0; q < sl;) {
                const int pq = s[q] >> 4, tq = s[q] & 15;
                const size_t n = 64 * (pq + 1);
                if (pq > 1 || tq > 3 || q + 1 + n > sl) return fail(kBadArg, "jpeg: bad DQT");
                for (int k = 0; k < 64; ++k)
                    qt[tq][kZigzag[k]] = pq ? uint16_t((s[q + 1 + 2 * k] << 8) | s[q + 2 + 2 * k]) : s[q + 1 + k];
                have_q[tq] = true;
                q += 1 + n;
            }
        } else if (m == 0xDD) {
            if (sl < 2) return fail(kBadArg, "jpeg: short DRI");
            hd.restart = (s[0] << 8) | s[1];
        } else if (m == 0xE0) {
            jfif = jfif || (sl >= 5 && !memcmp(s, "JFIF\0", 5));
        } else if (m == 0xEE) {
            if (sl >= 12 && !memcmp(s, "Adobe", 5)) adobe = s[11];
        } else if (m == 0xDC) {
            return fail(kUnsupported, "jpeg: DNL");
        } else if (m == 0xDA) {
            if (!have_sof) return fail(kBadArg, "jpeg: SOS before SOF");
            if (sl < 1 || sl < 4 + 2 * size_t(s[0])) return fail(kBadArg, "jpeg: short SOS");
            const int ns = s[0];
            if (ns != nc) return fail(kUnsupported, "jpeg: more than one scan (non-interleaved components)");
            for (int i = 0; i < ns; ++i) {
                if (s[1 + 2 * i] != comps[i].id) return fail(kUnsupported, "jpeg: more than one scan (non-interleaved components)");
                td[i] = s[2 + 2 * i] >> 4;
                ta[i] = s[2 + 2 * i] & 15;
                if (td[i] > 3 || ta[i] > 3) return fail(kBadArg, "jpeg: bad Huffman table selector");
            }
            if (s[1 + 2 * ns] != 0 || s[2 + 2 * ns] != 63 || s[3 + 2 * ns] != 0)
                return fail(kBadArg, "jpeg: bad spectral selection in a sequential scan");
            hd.scan_start = p + L;
            break;
        }
        p += L;
    }
    if (nc == 3) {
        hd.hs = comps[0].h;
        hd.vs = comps[0].v;
        const bool luma_ok = (hd.hs == 1 && hd.vs == 1) || (hd.hs == 2 && hd.vs == 1) || (hd.hs == 2 && hd.vs == 2);
        for (int i = 1; i < 3; ++i)
            if (comps[i].h != 1 || comps[i].v != 1) return fail(kUnsupported, "jpeg: chroma sampling %dx%d", comps[i].h, comps[i].v);
        if (!luma_ok) return fail(kUnsupported, "jpeg: luma sampling %dx%d", hd.hs, hd.vs);
        if (adobe == 0 || (adobe < 0 && !jfif && comps[0].id == 'R' && comps[1].id == 'G' && comps[2].id == 'B'))
            return fail(kUnsupported, "jpeg: RGB colour space");
    }
    for (int i = 0; i < nc; ++i) {
        if (comps[i].h < 1 || comps[i].h > 4 || comps[i].v < 1 || comps[i].v > 4) return fail(kBadArg, "jpeg: bad sampling factor");
        if (comps[i].tq > 3 || !have_q[comps[i].tq] || !have_h[0][td[i]] || !have_h[1][ta[i]])
            return fail(kBadArg, "jpeg: component %d refers to a missing table", comps[i].id);
        memcpy(hd.q[i], qt[comps[i].tq], sizeof(hd.q[i]));
        hd.dc[i] = ht[0][td[i]];
        hd.ac[i] = ht[1][ta[i]];
    }
    size_t e = len - 2;
    while (e >= hd.scan_start && !(d[e] == 0xFF && d[e + 1] == 0xD9)) {
        if (e == 0) break;
        --e;
    }
    if (e < hd.scan_start || !(d[e] == 0xFF && d[e + 1] == 0xD9)) return fail(kBadArg, "jpeg: no EOI after the scan (truncated stream)");
    hd.scan_end = e;
    hd.H = H;
    hd.W = W;
    hd.nc = nc;
    return kOk;
}

static void fill_desc(const Header& hd, Desc& D) {
    memset(&D, 0, sizeof(D));
    D.H = hd.H;
    D.W = hd.W;
    D.nc = hd.nc;
    D.hs = hd.hs;
    D.vs = hd.vs;
    D.restart = hd.restart;
    D.mcux = (hd.W + 8 * hd.hs - 1) / (8 * hd.hs);
    D.mcuy = (hd.H + 8 * hd.vs - 1) / (8 * hd.vs);
    const int total = D.mcux * D.mcuy;
    const int R = hd.restart ? hd.restart : total;
    D.n_int = (total + R - 1) / R;
    for (int c = 0; c < hd.nc; ++c) {
        D.bw[c] = D.mcux * (c == 0 ? hd.hs : 1);
        D.bh[c] = D.mcuy * (c == 0 ? hd.vs : 1);
        memcpy(D.q[c], hd.q[c], sizeof(D.q[c]));
        D.dc[c] = hd.dc[c];
        D.ac[c] = hd.ac[c];
    }
    D.raw_len = (long long)(hd.scan_end - hd.scan_start);
}

static long long blocks_of(const Desc& D) {
    long long b = 0;
    for (int c = 0; c < D.nc; ++c) b += (long long)D.bw[c] * D.bh[c];
    return b;
}

struct Layout {
    size_t desc, raw, vals, cub, cub_bytes, seg, data, coef, planes, total;   // device offsets
    size_t host_raw, host_total;                                     // host staging: descs, then raw bytes
    long long n_raw, n_seg, n_blk, n_pix, max_blk, max_pix;
};

// Headers of all n streams -> descriptors and the workspace layout (descs / raw are filled only when `descs` is given)
static int plan(const uint8_t* const* data, const size_t* lengths, int n, std::vector<Desc>* descs, std::vector<Header>* hds, Layout& L) {
    if (!data || !lengths || n <= 0) return fail(kBadArg, "irn_jpeg_exact: bad argument");
    L = Layout{};
    Header hd;
    Desc D;
    for (int i = 0; i < n; ++i) {
        int rc = parse(data[i], lengths[i], hd);
        if (rc) {
            char why[512];
            snprintf(why, sizeof(why), "%s", irn_last_error());
            return fail(rc, "image %d: %s", i, why);
        }
        fill_desc(hd, D);
        D.raw0 = L.n_raw;
        D.seg0 = L.n_seg;
        D.blk0 = L.n_blk;
        D.pix0 = L.n_pix;
        const long long nb = blocks_of(D);
        L.n_raw += D.raw_len;
        L.n_seg += D.n_int + 1;
        L.n_blk += nb;
        L.n_pix += nb * 64;
        L.max_blk = nb > L.max_blk ? nb : L.max_blk;
        L.max_pix = (long long)D.H * D.W > L.max_pix ? (long long)D.H * D.W : L.max_pix;
        if (descs) descs->push_back(D);
        if (hds) hds->push_back(hd);
    }
    if (L.n_raw >= (1ll << 31)) return fail(kUnsupported, "irn_jpeg_exact: more than 2 GB of entropy-coded data in one call");
    size_t o = 0;
    auto take = [&](size_t bytes) { size_t r = o; o = align_up(o + bytes, 256); return r; };
    L.desc = take(sizeof(Desc) * n);
    L.raw = take(L.n_raw + 16);
    L.vals = take(sizeof(unsigned long long) * (L.n_raw + 1));
    L.cub_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, L.cub_bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)(L.n_raw + 1));
    L.cub = take(L.cub_bytes);
    L.seg = take(sizeof(long long) * L.n_seg);
    L.data = take(L.n_raw + 16);
    L.coef = take(sizeof(int16_t) * 64 * L.n_blk);
    L.planes = take(L.n_pix);
    L.total = o;
    L.host_raw = align_up(sizeof(Desc) * n, 256);
    L.host_total = L.host_raw + L.n_raw;
    return kOk;
}

// ------------------------------------------------------------------------------------------------------------------------------
// device

// Stage 1a: per byte of image blockIdx.y's segment, kept (low 32 bits) and is-RSTn (high 32 bits); the entry past the last byte is 0.
__global__ void flag_kernel(const Desc* __restrict__ descs, const uint8_t* __restrict__ raw, unsigned long long* __restrict__ vals,
                            long long n_raw) {
    const Desc& D = descs[blockIdx.y];
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < D.raw_len; i += (long long)gridDim.x * blockDim.x) {
        const uint8_t* p = raw + D.raw0 + i;
        const uint8_t b = p[0];
        const bool after_ff = i > 0 && p[-1] == 0xFF;
        const bool rst = after_ff && b >= 0xD0 && b <= 0xD7;
        const bool drop = (after_ff && b == 0x00) || rst || (b == 0xFF && i + 1 < D.raw_len && p[1] >= 0xD0 && p[1] <= 0xD7);
        vals[D.raw0 + i] = (rst ? (1ull << 32) : 0ull) | (drop ? 0ull : 1ull);
    }
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) vals[n_raw] = 0;
}

// Stage 1b: scatter the kept bytes; record where each restart interval starts (the interval-start table of image i holds n_int + 1
// entries, the last one being the end of the image's unstuffed bytes); check the markers.
__global__ void scatter_kernel(const Desc* __restrict__ descs, const uint8_t* __restrict__ raw, const unsigned long long* __restrict__ sums,
                               uint8_t* __restrict__ out, long long* __restrict__ seg, int* __restrict__ status) {
    const int img = blockIdx.y;
    const Desc& D = descs[img];
    const unsigned long long base = sums[D.raw0];
    const unsigned rst0 = unsigned(base >> 32);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        seg[D.seg0] = (long long)(base & 0xffffffffu);
        seg[D.seg0 + D.n_int] = (long long)(sums[D.raw0 + D.raw_len] & 0xffffffffu);
    }
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < D.raw_len; i += (long long)gridDim.x * blockDim.x) {
        const uint8_t* p = raw + D.raw0 + i;
        const uint8_t b = p[0];
        const unsigned long long s = sums[D.raw0 + i], s1 = sums[D.raw0 + i + 1];
        if ((s1 ^ s) & 1ull) {              // kept
            out[s & 0xffffffffu] = b;
            // a marker other than stuffing and RSTn (fill bytes FF FF included): not a single-scan baseline segment
            if (b == 0xFF && (i + 1 >= D.raw_len || (p[1] != 0x00 && (p[1] < 0xD0 || p[1] > 0xD7)))) atomicOr(status + img, kStMarker);
        } else if ((s1 >> 32) != (s >> 32)) {     // the Dx of RSTn: interval k + 1 starts at the next kept byte
            const unsigned k = unsigned(s >> 32) - rst0;
            if ((long long)k + 1 < D.n_int && (b & 7) == (k & 7))
                seg[D.seg0 + k + 1] = (long long)(s & 0xffffffffu);
            else
                atomicOr(status + img, kStRestart);
        }
    }
}

struct SmemTable {
    uint16_t fast[512];      // 9-bit lookahead: (length << 8) | symbol, 0 = longer code
    int maxcode[18];         // per length, -1 = none; [17] sentinel
    int valoff[17];          // symbol index = valoff[l] + code
    uint8_t vals[256];
};

struct Bits {
    const uint8_t* p;
    const uint8_t* end;
    unsigned long long acc;
    int n;                   // valid bits in acc (msb-aligned)
    long long left;          // bits of the interval not yet consumed (negative: read past the end)

    __device__ void refill() {
        while (n <= 56) {
            const uint8_t b = p < end ? *p : 0;
            ++p;
            acc |= (unsigned long long)b << (56 - n);
            n += 8;
        }
    }
    __device__ unsigned peek16() const { return unsigned(acc >> 48); }
    __device__ void skip(int k) {
        acc <<= k;
        n -= k;
        left -= k;
    }
    __device__ int get(int k) {      // k <= 16, after a refill
        if (k == 0) return 0;
        const int v = int(acc >> (64 - k));
        skip(k);
        return v;
    }
};

// -1 on an invalid code
__device__ __forceinline__ int decode_symbol(Bits& br, const SmemTable& t) {
    const unsigned v = br.peek16();
    const unsigned f = t.fast[v >> 7];
    if (f) {
        br.skip(int(f >> 8));
        return int(f & 255);
    }
    int l = 10;
    while (l <= 16 && int(v >> (16 - l)) > t.maxcode[l]) ++l;
    if (l > 16) return -1;
    const int sym = t.vals[(t.valoff[l] + int(v >> (16 - l))) & 255];
    br.skip(l);
    return sym;
}

__device__ __forceinline__ int extend(int v, int s) { return (s && v < (1 << (s - 1))) ? v - (1 << s) + 1 : v; }

constexpr int kEntropyThreads = 128;

// Stage 2: one CTA per image, thread t decodes restart intervals t, t + 128, ...
__global__ void __launch_bounds__(kEntropyThreads) entropy_kernel(const Desc* __restrict__ descs, const uint8_t* __restrict__ data,
                                                                  const long long* __restrict__ seg, int16_t* __restrict__ coef,
                                                                  int* __restrict__ status) {
    __shared__ SmemTable tabs[2 * kMaxComp];
    __shared__ uint8_t zz[64];
    const int img = blockIdx.x;
    const Desc& D = descs[img];
    const int nt = 2 * D.nc;
    if (threadIdx.x < nt) {       // canonical code -> maxcode / valoff per length (T.81 C.2, F.2.2.3)
        const Huff& h = (threadIdx.x & 1) ? D.ac[threadIdx.x >> 1] : D.dc[threadIdx.x >> 1];
        SmemTable& t = tabs[threadIdx.x];
        int code = 0, k = 0;
        for (int l = 1; l <= 16; ++l) {
            const int c = h.counts[l - 1];
            t.valoff[l] = k - code;
            t.maxcode[l] = c ? code + c - 1 : -1;
            code = (code + c) << 1;
            k += c;
        }
        t.maxcode[17] = 0x7fffffff;
    }
    for (int i = threadIdx.x; i < nt * 256; i += blockDim.x) tabs[i >> 8].vals[i & 255] = ((i >> 8) & 1 ? D.ac[i >> 9] : D.dc[i >> 9]).vals[i & 255];
    if (threadIdx.x < 64) zz[threadIdx.x] = kZigzagDev[threadIdx.x];
    __syncthreads();
    for (int i = threadIdx.x; i < nt * 512; i += blockDim.x) {
        SmemTable& t = tabs[i >> 9];
        const int e = i & 511;
        uint16_t f = 0;
        for (int l = 1; l <= 9; ++l) {
            const int code = e >> (9 - l);
            if (code <= t.maxcode[l]) {
                f = uint16_t((l << 8) | t.vals[(t.valoff[l] + code) & 255]);
                break;
            }
        }
        t.fast[e] = f;
    }
    __syncthreads();

    const int total = D.mcux * D.mcuy;
    const int R = D.restart ? D.restart : total;
    const long long comp_blk0[kMaxComp] = {D.blk0, D.blk0 + (long long)D.bw[0] * D.bh[0],
                                           D.blk0 + (long long)D.bw[0] * D.bh[0] + (long long)D.bw[1] * D.bh[1]};
    for (int k = threadIdx.x; k < D.n_int; k += blockDim.x) {
        const long long a = seg[D.seg0 + k], b = seg[D.seg0 + k + 1];
        if (a < 0 || b < a) {
            atomicOr(status + img, kStRestart);
            continue;
        }
        Bits br{data + a, data + b, 0ull, 0, (b - a) * 8};
        br.refill();
        int pred[kMaxComp] = {0, 0, 0};
        int err = 0;
        const int m_end = min(total, (k + 1) * R);
        for (int m = k * R; m < m_end && !err; ++m) {
            const int my = m / D.mcux, mx = m - my * D.mcux;
#pragma unroll
            for (int c = 0; c < kMaxComp; ++c) {
                if (c >= D.nc || err) break;
                const int hc = c == 0 ? D.hs : 1, vc = c == 0 ? D.vs : 1;
                const SmemTable& tdc = tabs[2 * c];
                const SmemTable& tac = tabs[2 * c + 1];
                for (int by = 0; by < vc && !err; ++by)
                    for (int bx = 0; bx < hc && !err; ++bx) {
                        int16_t* blk = coef + 64 * (comp_blk0[c] + (long long)(my * vc + by) * D.bw[c] + mx * hc + bx);
                        int4* b4 = reinterpret_cast<int4*>(blk);
#pragma unroll
                        for (int j = 0; j < 8; ++j) b4[j] = make_int4(0, 0, 0, 0);
                        br.refill();
                        int s = decode_symbol(br, tdc);
                        if (s < 0 || s > 15) {
                            err = kStCode;
                            break;
                        }
                        pred[c] += extend(br.get(s), s);
                        blk[0] = int16_t(pred[c]);
                        for (int z = 1; z < 64;) {
                            br.refill();
                            const int rs = decode_symbol(br, tac);
                            if (rs < 0) {
                                err = kStCode;
                                break;
                            }
                            const int r = rs >> 4;
                            s = rs & 15;
                            if (s == 0) {
                                if (r != 15) break;
                                z += 16;
                                continue;
                            }
                            z += r;
                            if (z > 63) {
                                err = kStRun;
                                break;
                            }
                            blk[zz[z]] = int16_t(extend(br.get(s), s));
                            ++z;
                        }
                        if (!err && br.left < 0) err = kStOverrun;
                    }
            }
        }
        if (err) atomicOr(status + img, err);
    }
}

// Stage 3: dequantise + islow IDCT.  blockIdx.y = image; 16 blocks per CTA, 8 threads per block.
constexpr int kIdctThreads = 128;

__device__ __forceinline__ void idct_1d(const int* v, int* out, int shift) {
    constexpr int F0_298 = 2446, F0_390 = 3196, F0_541 = 4433, F0_765 = 6270, F0_899 = 7373, F1_175 = 9633, F1_501 = 12299,
                  F1_847 = 15137, F1_961 = 16069, F2_053 = 16819, F2_562 = 20995, F3_072 = 25172;   // round(c * 2^13)
    int z2 = v[2], z3 = v[6];
    int z1 = (z2 + z3) * F0_541;
    const int tmp2 = z1 - z3 * F1_847;
    const int tmp3 = z1 + z2 * F0_765;
    const int tmp0 = (v[0] + v[4]) * 8192;
    const int tmp1 = (v[0] - v[4]) * 8192;
    const int t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
    int o0 = v[7], o1 = v[5], o2 = v[3], o3 = v[1];
    z1 = o0 + o3;
    z2 = o1 + o2;
    z3 = o0 + o2;
    int z4 = o1 + o3;
    const int z5 = (z3 + z4) * F1_175;
    o0 *= F0_298;
    o1 *= F2_053;
    o2 *= F3_072;
    o3 *= F1_501;
    z1 *= -F0_899;
    z2 *= -F2_562;
    z3 = z3 * -F1_961 + z5;
    z4 = z4 * -F0_390 + z5;
    o0 += z1 + z3;
    o1 += z2 + z4;
    o2 += z2 + z3;
    o3 += z1 + z4;
    const int r = 1 << (shift - 1);
    out[0] = (t10 + o3 + r) >> shift;
    out[7] = (t10 - o3 + r) >> shift;
    out[1] = (t11 + o2 + r) >> shift;
    out[6] = (t11 - o2 + r) >> shift;
    out[2] = (t12 + o1 + r) >> shift;
    out[5] = (t12 - o1 + r) >> shift;
    out[3] = (t13 + o0 + r) >> shift;
    out[4] = (t13 - o0 + r) >> shift;
}

__global__ void __launch_bounds__(kIdctThreads) idct_kernel(const Desc* __restrict__ descs, const int16_t* __restrict__ coef,
                                                            uint8_t* __restrict__ planes) {
    __shared__ int ws[kIdctThreads / 8][8][9];
    const Desc& D = descs[blockIdx.y];
    const int lb = threadIdx.x >> 3, j = threadIdx.x & 7;
    long long b = (long long)blockIdx.x * (kIdctThreads / 8) + lb;
    int c = 0;
    long long pix = D.pix0;
    for (; c < D.nc; ++c) {
        const long long nb = (long long)D.bw[c] * D.bh[c];
        if (b < nb) break;
        b -= nb;
        pix += nb * 64;
    }
    if (c == D.nc) return;       // whole 8-thread groups leave together; the rest never sync across groups
    const int16_t* in = coef + 64 * (D.blk0 + (pix - D.pix0) / 64 + b);
    const uint16_t* q = D.q[c];
    int v[8], o[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) v[r] = int(in[r * 8 + j]) * int(q[r * 8 + j]);
    idct_1d(v, o, 13 - 2);       // pass 1: column j
#pragma unroll
    for (int r = 0; r < 8; ++r) ws[lb][r][j] = o[r];
    __syncwarp(0xFFu << (threadIdx.x & 24));       // the block's 8 lanes
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = ws[lb][j][k];
    idct_1d(v, o, 13 + 2 + 3);   // pass 2: row j
    unsigned lo = 0, hi = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int x = ((o[k] + 512) & 1023) - 512;      // the range-limit table's wrap, then the clamp
        const unsigned u = unsigned(min(max(x + 128, 0), 255));
        if (k < 4) lo |= u << (8 * k);
        else hi |= u << (8 * (k - 4));
    }
    const int stride = D.bw[c] * 8;
    const long long by = b / D.bw[c], bx = b - by * D.bw[c];
    *reinterpret_cast<uint2*>(planes + pix + (by * 8 + j) * stride + bx * 8) = make_uint2(lo, hi);
}

// Stage 4: up-sampling + YCbCr -> RGB, one thread per output pixel; blockIdx.y = image.
__device__ __forceinline__ int chroma(const uint8_t* s, int stride, int y, int x, int dw, int dh, int hs, int vs) {
    if (hs == 1) return s[y * stride + x];
    const int c = x >> 1, odd = x & 1;
    if (dw <= 2) return s[(y >> (vs - 1)) * stride + c];          // narrow plane: replication
    const int cn = odd ? min(c + 1, dw - 1) : max(c - 1, 0);
    if (vs == 1) return (3 * s[y * stride + c] + s[y * stride + cn] + 1 + odd) >> 2;
    const int r = y >> 1;
    const int r2 = (y & 1) ? min(r + 1, dh - 1) : max(r - 1, 0);
    const int t = 3 * s[r * stride + c] + s[r2 * stride + c];
    const int tn = 3 * s[r * stride + cn] + s[r2 * stride + cn];
    return (3 * t + tn + 8 - odd) >> 4;
}

__global__ void color_kernel(const Desc* __restrict__ descs, const uint8_t* __restrict__ planes, uint8_t* __restrict__ out) {
    const Desc& D = descs[blockIdx.y];
    const long long n = (long long)D.H * D.W;
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int y = int(i / D.W), x = int(i - (long long)y * D.W);
    const uint8_t* py = planes + D.pix0;
    const int Y = py[(long long)y * D.bw[0] * 8 + x];
    uint8_t* o = out + D.out0 + 3 * i;
    if (D.nc == 1) {
        o[0] = o[1] = o[2] = uint8_t(Y);
        return;
    }
    const long long n0 = (long long)D.bw[0] * D.bh[0] * 64, n1 = (long long)D.bw[1] * D.bh[1] * 64;
    const int stride = D.bw[1] * 8;
    const int dw = (D.W + D.hs - 1) / D.hs, dh = (D.H + D.vs - 1) / D.vs;
    const int cb = chroma(py + n0, stride, y, x, dw, dh, D.hs, D.vs) - 128;
    const int cr = chroma(py + n0 + n1, stride, y, x, dw, dh, D.hs, D.vs) - 128;
    constexpr int kR = 91881, kB = 116130, kGb = 22554, kGr = 46802, kHalf = 1 << 15;   // round(c * 2^16)
    const int r = Y + ((kR * cr + kHalf) >> 16);
    const int g = Y + ((-kGb * cb + kHalf - kGr * cr) >> 16);
    const int b = Y + ((kB * cb + kHalf) >> 16);
    o[0] = uint8_t(min(max(r, 0), 255));
    o[1] = uint8_t(min(max(g, 0), 255));
    o[2] = uint8_t(min(max(b, 0), 255));
}

struct Timing {
    bool on = false;
    cudaEvent_t ev[5] = {};
    bool valid = false;
};
static thread_local Timing g_timing;

}  // namespace jx
}  // namespace irn

using namespace irn;
using namespace irn::jx;

extern "C" int irn_jpeg_exact_inspect(const uint8_t* data, size_t length, int* info) {
    if (!info) return fail(kBadArg, "irn_jpeg_exact_inspect: info is null");
    Header hd;
    int rc = parse(data, length, hd);
    if (rc) return rc;
    info[0] = hd.H;
    info[1] = hd.W;
    info[2] = hd.nc;
    info[3] = hd.hs;
    info[4] = hd.vs;
    info[5] = hd.restart;
    return kOk;
}

extern "C" int irn_jpeg_exact_workspace_bytes(const uint8_t* const* data, const size_t* lengths, int n, size_t* device_bytes,
                                              size_t* host_bytes) {
    if (!device_bytes || !host_bytes) return fail(kBadArg, "irn_jpeg_exact_workspace_bytes: null output");
    Layout L;
    int rc = plan(data, lengths, n, nullptr, nullptr, L);
    if (rc) return rc;
    *device_bytes = L.total;
    *host_bytes = L.host_total;
    return kOk;
}

extern "C" int irn_jpeg_exact_decode(const uint8_t* const* data, const size_t* lengths, int n, const int64_t* out_offsets, uint8_t* out_dev,
                                     int32_t* status_dev, void* workspace, size_t workspace_bytes, void* host_staging,
                                     size_t host_bytes, irn_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    launch_counter() = 0;
    if (!out_offsets || !out_dev || !status_dev || !workspace || !host_staging)
        return fail(kBadArg, "irn_jpeg_exact_decode: null argument");
    std::vector<Desc> descs;
    std::vector<Header> hds;
    Layout L;
    int rc = plan(data, lengths, n, &descs, &hds, L);
    if (rc) return rc;
    if (workspace_bytes < L.total || host_bytes < L.host_total)
        return fail(kWorkspace, "irn_jpeg_exact_decode: workspace %zu / %zu bytes, need %zu / %zu", workspace_bytes, host_bytes, L.total,
                    L.host_total);
    if ((uintptr_t)workspace % 256) return fail(kBadArg, "irn_jpeg_exact_decode: workspace must be 256-byte aligned");
    uint8_t* hs = (uint8_t*)host_staging;
    for (int i = 0; i < n; ++i) {
        if (out_offsets[i] < 0) return fail(kBadArg, "irn_jpeg_exact_decode: negative output offset for image %d", i);
        descs[i].out0 = out_offsets[i];
        memcpy(hs + L.host_raw + descs[i].raw0, data[i] + hds[i].scan_start, descs[i].raw_len);
    }
    memcpy(hs, descs.data(), sizeof(Desc) * n);
    uint8_t* ws = (uint8_t*)workspace;
    const Desc* d_desc = (const Desc*)(ws + L.desc);
    uint8_t* d_raw = ws + L.raw;
    unsigned long long* d_vals = (unsigned long long*)(ws + L.vals);
    long long* d_seg = (long long*)(ws + L.seg);
    int16_t* d_coef = (int16_t*)(ws + L.coef);
    uint8_t* d_planes = ws + L.planes;
    IRN_CUDA(cudaMemcpyAsync(ws + L.desc, hs, sizeof(Desc) * n, cudaMemcpyHostToDevice, stream));
    if (L.n_raw) IRN_CUDA(cudaMemcpyAsync(d_raw, hs + L.host_raw, L.n_raw, cudaMemcpyHostToDevice, stream));
    IRN_CUDA(cudaMemsetAsync(status_dev, 0, sizeof(int32_t) * n, stream));
    IRN_CUDA(cudaMemsetAsync(d_seg, 0xFF, sizeof(long long) * L.n_seg, stream));     // -1: no restart marker seen

    Timing& tm = g_timing;
    if (tm.on) IRN_CUDA(cudaEventRecord(tm.ev[0], stream));
    long long max_raw = 0;
    for (const Desc& D : descs) max_raw = D.raw_len > max_raw ? D.raw_len : max_raw;
    const int gx_raw = (int)std::min<long long>(std::max<long long>((max_raw + 255) / 256, 1), 1024);
    flag_kernel<<<dim3(gx_raw, n), 256, 0, stream>>>(d_desc, d_raw, d_vals, L.n_raw);
    IRN_LAUNCH_CHECK("jpeg_exact flag_kernel");
    size_t cub_bytes = L.cub_bytes;
    IRN_CUDA(cub::DeviceScan::ExclusiveSum(ws + L.cub, cub_bytes, d_vals, d_vals, (int)(L.n_raw + 1), stream));
    IRN_LAUNCH_CHECK("jpeg_exact unstuff scan");
    uint8_t* d_data = ws + L.data;
    scatter_kernel<<<dim3(gx_raw, n), 256, 0, stream>>>(d_desc, d_raw, d_vals, d_data, d_seg, status_dev);
    IRN_LAUNCH_CHECK("jpeg_exact scatter_kernel");
    if (tm.on) IRN_CUDA(cudaEventRecord(tm.ev[1], stream));
    entropy_kernel<<<n, kEntropyThreads, 0, stream>>>(d_desc, d_data, d_seg, d_coef, status_dev);
    IRN_LAUNCH_CHECK("jpeg_exact entropy_kernel");
    if (tm.on) IRN_CUDA(cudaEventRecord(tm.ev[2], stream));
    idct_kernel<<<dim3((unsigned)((L.max_blk + 15) / 16), n), kIdctThreads, 0, stream>>>(d_desc, d_coef, d_planes);
    IRN_LAUNCH_CHECK("jpeg_exact idct_kernel");
    if (tm.on) IRN_CUDA(cudaEventRecord(tm.ev[3], stream));
    color_kernel<<<dim3((unsigned)((L.max_pix + 255) / 256), n), 256, 0, stream>>>(d_desc, d_planes, out_dev);
    IRN_LAUNCH_CHECK("jpeg_exact color_kernel");
    if (tm.on) {
        IRN_CUDA(cudaEventRecord(tm.ev[4], stream));
        tm.valid = true;
    }
    return kOk;
}

extern "C" int irn_jpeg_exact_set_timing(int enable) {
    Timing& tm = g_timing;
    if (enable && !tm.ev[0])
        for (auto& e : tm.ev) IRN_CUDA(cudaEventCreate(&e));
    tm.on = enable != 0;
    tm.valid = false;
    return kOk;
}

extern "C" int irn_jpeg_exact_last_ms(float* ms4) {
    Timing& tm = g_timing;
    if (!tm.valid) return fail(kBadArg, "irn_jpeg_exact_last_ms: no timed call");
    IRN_CUDA(cudaEventSynchronize(tm.ev[4]));
    for (int i = 0; i < 4; ++i) IRN_CUDA(cudaEventElapsedTime(ms4 + i, tm.ev[i], tm.ev[i + 1]));
    return kOk;
}
