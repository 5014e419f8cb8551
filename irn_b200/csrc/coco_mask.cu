// MS COCO mask evaluation on the device: ground-truth rasterisation, prediction bit packing, mask overlap counts.
//
// Bit plane (every mask of an H x W image): W columns of ceil(H/32) uint32 words, column-major like COCO's RLE; bit b of word j of
// column x is pixel (row 32j+b, column x); the bits past row H-1 of a column's last word are zero.  Predictions and ground truth use
// the same layout, so an overlap is a popcount of AND over the words.  Every output is an integer: the result does not depend on the
// launch configuration.
//
// Polygons follow pycocotools' rleFrPoly (restated from its published algorithm): vertices upsampled x5 and truncated, (int)(5v+.5);
// every edge walked along its major axis with a double DDA, (int)(s + slope*t + .5); the samples where the upsampled x changes map
// back to a pixel column (skipped unless integral and inside the image) and a clamped, ceil'd row; a pixel is inside when the number
// of such boundary toggles at or before it, in column-major order, is odd.  The DDA and the back-mapping are explicit _rn double
// operations: a contracted multiply-add would move boundary pixels.  An annotation of several polygons is their union, as
// pycocotools merges them.  Uncompressed RLE arrives as its toggle positions (the running sums of the counts).
#include <climits>
#include <cstring>
#include <vector>

#include "common.h"

namespace irn {

constexpr int kRasterThreads = 256;
constexpr int kOverlapThreads = 256;
constexpr int kGtTile = 8;     // ground-truth planes per overlap block: each prediction word is read once per tile

__host__ __device__ inline int col_words(int H) { return (H + 31) >> 5; }

struct RasterPart {     // one polygon or one RLE of an annotation: its own toggle plane, OR-ed into the annotation's plane
    long long tog;      // word offset of the toggle plane in the workspace
    long long out;      // word offset of the annotation's plane in the output
    int H, W;
};

struct RasterEdge {     // edge j of a polygon of k vertices starting at vertex `first`
    int part, first, k, j;
};

struct PackImg {        // image i of a pack call: M bool masks [M,H,W] at byte `src`, their planes at word `dst`
    long long src, dst;
    int H, W, M, block0;    // block0: the image's first tile block
};

struct AreaItem {       // popcount of one plane
    long long plane;
    int words, out;
};

struct OverlapItem {    // prediction m of an image against up to kGtTile of its ground-truth planes
    long long pred, gt, out;    // word offsets of the prediction plane and the first ground-truth plane; index of inter[m][g0]
    int words, ng;
};

// ---------------------------------------------------------------------------------------------------------------- rasterisation
__device__ __forceinline__ void toggle(uint32_t* plane, int H, int W, int x, int y) {
    const long long word = (long long)x * col_words(H) + (y >> 5);
    if (word < (long long)W * col_words(H)) atomicXor(plane + word, 1u << (y & 31));
}

__device__ __forceinline__ int up5(double v) { return __double2int_rz(__dadd_rn(__dmul_rn(5.0, v), 0.5)); }

// sample d of an edge from (xs0, ys0) to (xe0, ye0) (upsampled), in generation order
__device__ __forceinline__ void edge_sample(int xs, int ys, int xe, int ye, int d, int& u, int& v) {
    const int dx = abs(xe - xs), dy = abs(ys - ye);
    const bool flip = (dx >= dy && xs > xe) || (dx < dy && ys > ye);
    if (flip) {
        int t = xs; xs = xe; xe = t;
        t = ys; ys = ye; ye = t;
    }
    if (dx >= dy) {
        const int t = flip ? dx - d : d;
        u = t + xs;
        if (dx == 0) {      // a zero-length edge: the C code's 0/0 slope converts to x86's integer indefinite
            v = INT_MIN;
            return;
        }
        const double s = __ddiv_rn((double)(ye - ys), (double)dx);
        v = __double2int_rz(__dadd_rn(__dadd_rn((double)ys, __dmul_rn(s, (double)t)), 0.5));
    } else {
        const double s = __ddiv_rn((double)(xe - xs), (double)dy);
        const int t = flip ? dy - d : d;
        v = t + ys;
        u = __double2int_rz(__dadd_rn(__dadd_rn((double)xs, __dmul_rn(s, (double)t)), 0.5));
    }
}

// the toggle of the consecutive samples (u0, v0) -> (u1, v1), if any
__device__ __forceinline__ void sample_toggle(uint32_t* plane, int H, int W, int u0, int v0, int u1, int v1) {
    if (u1 == u0) return;
    double xd = (double)(u1 < u0 ? u1 : u1 - 1);
    xd = __dsub_rn(__ddiv_rn(__dadd_rn(xd, 0.5), 5.0), 0.5);
    if (floor(xd) != xd || xd < 0.0 || xd > (double)(W - 1)) return;
    double yd = (double)(v1 < v0 ? v1 : v0);
    yd = __dsub_rn(__ddiv_rn(__dadd_rn(yd, 0.5), 5.0), 0.5);
    yd = yd < 0.0 ? 0.0 : (yd > (double)H ? (double)H : yd);
    toggle(plane, H, W, (int)xd, (int)ceil(yd));
}

// one thread per polygon edge: every sample pair of the edge, and the pair that joins it to the previous edge's last sample
__global__ void poly_toggle_kernel(const RasterPart* __restrict__ parts, const RasterEdge* __restrict__ edges, int n_edges,
                                   const double* __restrict__ xy, uint32_t* __restrict__ tog) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_edges) return;
    const RasterEdge E = edges[e];
    const RasterPart P = parts[E.part];
    uint32_t* plane = tog + P.tog;
    const double* p = xy + 2 * (long long)E.first;
    const int j1 = E.j + 1 == E.k ? 0 : E.j + 1;
    const int xs = up5(p[2 * E.j]), ys = up5(p[2 * E.j + 1]), xe = up5(p[2 * j1]), ye = up5(p[2 * j1 + 1]);
    const int len = max(abs(xe - xs), abs(ys - ye));
    int u0, v0;
    if (E.j > 0) {      // the last sample of edge j-1 precedes this edge's first one
        const int jp = E.j - 1;
        const int pxs = up5(p[2 * jp]), pys = up5(p[2 * jp + 1]);
        edge_sample(pxs, pys, xs, ys, max(abs(xs - pxs), abs(pys - ys)), u0, v0);
    } else {
        edge_sample(xs, ys, xe, ye, 0, u0, v0);
    }
    for (int d = E.j > 0 ? 0 : 1; d <= len; ++d) {
        int u1, v1;
        edge_sample(xs, ys, xe, ye, d, u1, v1);
        sample_toggle(plane, P.H, P.W, u0, v0, u1, v1);
        u0 = u1;
        v0 = v1;
    }
}

// one thread per RLE toggle (part, flat column-major position)
__global__ void rle_toggle_kernel(const RasterPart* __restrict__ parts, const int2* __restrict__ toggles, int n_toggles,
                                  uint32_t* __restrict__ tog) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_toggles) return;
    const int2 t = toggles[i];
    const RasterPart P = parts[t.x];
    const int x = t.y / P.H;
    toggle(tog + P.tog, P.H, P.W, x, t.y - x * P.H);
}

__device__ __forceinline__ uint32_t prefix_xor(uint32_t w) {     // bit b = XOR of bits 0..b
    w ^= w << 1;
    w ^= w << 2;
    w ^= w << 4;
    w ^= w << 8;
    w ^= w << 16;
    return w;
}

// one block per part: prefix-XOR of its toggle plane in flat order (each thread a contiguous run of words, a block scan of the runs'
// parities), padding bits cleared, OR-ed into the annotation's plane
__global__ void __launch_bounds__(kRasterThreads) fill_kernel(const RasterPart* __restrict__ parts, const uint32_t* __restrict__ tog,
                                                              uint32_t* __restrict__ out) {
    __shared__ uint32_t s_par[kRasterThreads];
    const RasterPart P = parts[blockIdx.x];
    const int cw = col_words(P.H);
    const long long words = (long long)P.W * cw;
    const long long per = (words + kRasterThreads - 1) / kRasterThreads;
    const long long w0 = min(words, per * threadIdx.x), w1 = min(words, w0 + per);
    const uint32_t* src = tog + P.tog;
    uint32_t par = 0;
    for (long long w = w0; w < w1; ++w) par ^= __popc(src[w]) & 1;
    s_par[threadIdx.x] = par;
    __syncthreads();
    if (threadIdx.x == 0) {     // exclusive XOR scan of 256 bits
        uint32_t acc = 0;
        for (int i = 0; i < kRasterThreads; ++i) {
            const uint32_t v = s_par[i];
            s_par[i] = acc;
            acc ^= v;
        }
    }
    __syncthreads();
    uint32_t carry = s_par[threadIdx.x] ? 0xffffffffu : 0u;
    const uint32_t tail = (P.H & 31) ? (1u << (P.H & 31)) - 1u : 0xffffffffu;
    uint32_t* dst = out + P.out;
    for (long long w = w0; w < w1; ++w) {
        const uint32_t v = prefix_xor(src[w]) ^ carry;
        carry = (v >> 31) ? 0xffffffffu : 0u;
        const uint32_t m = (w % cw == cw - 1) ? (v & tail) : v;
        if (m) atomicOr(dst + w, m);
    }
}

// ---------------------------------------------------------------------------------------------------------------- prediction packing
// one block per 32 x 32 tile of one mask: the tile's bytes through shared memory, one ballot per column word
__global__ void __launch_bounds__(256) pack_kernel(const PackImg* __restrict__ imgs, int n_img, const uint8_t* __restrict__ masks,
                                                   uint32_t* __restrict__ planes) {
    __shared__ uint8_t s[32][33];
    int lo = 0, hi = n_img - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (imgs[mid].block0 <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
    }
    const PackImg I = imgs[lo];
    const int tx_n = (I.W + 31) >> 5, ty_n = col_words(I.H);
    int b = blockIdx.x - I.block0;
    const int m = b / (tx_n * ty_n);
    b -= m * tx_n * ty_n;
    const int ty = b / tx_n, tx = b - ty * tx_n;
    const int y0 = ty * 32, x0 = tx * 32;
    const uint8_t* src = masks + I.src + (long long)m * I.H * I.W;
    for (int i = threadIdx.x; i < 1024; i += 256) {
        const int r = i >> 5, c = i & 31;
        s[r][c] = (y0 + r < I.H && x0 + c < I.W) ? (src[(long long)(y0 + r) * I.W + x0 + c] != 0) : 0;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t* dst = planes + I.dst + (long long)m * I.W * ty_n;
    for (int c = warp; c < 32; c += 8) {
        const uint32_t word = __ballot_sync(0xffffffffu, s[lane][c]);
        if (lane == 0 && x0 + c < I.W) dst[(long long)(x0 + c) * ty_n + ty] = word;
    }
}

// ---------------------------------------------------------------------------------------------------------------- overlaps
__device__ __forceinline__ int block_sum(int v, int* s_red) {      // every thread gets the sum; s_red: 32 ints
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    v = (int)threadIdx.x < (int)(blockDim.x >> 5) ? s_red[threadIdx.x] : 0;
    if (threadIdx.x < 32)
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__global__ void __launch_bounds__(kOverlapThreads) area_kernel(const AreaItem* __restrict__ items, const uint32_t* __restrict__ pred,
                                                               const uint32_t* __restrict__ gt, int n_pred_items, int32_t* __restrict__ area_pred,
                                                               int32_t* __restrict__ area_gt) {
    __shared__ int s_red[32];
    const AreaItem it = items[blockIdx.x];
    const bool is_pred = (int)blockIdx.x < n_pred_items;
    const uint32_t* p = (is_pred ? pred : gt) + it.plane;
    int acc = 0;
    for (int w = threadIdx.x; w < it.words; w += blockDim.x) acc += __popc(__ldg(p + w));
    acc = block_sum(acc, s_red);
    if (threadIdx.x == 0) (is_pred ? area_pred : area_gt)[it.out] = acc;
}

__global__ void __launch_bounds__(kOverlapThreads) overlap_kernel(const OverlapItem* __restrict__ items, const uint32_t* __restrict__ pred,
                                                                  const uint32_t* __restrict__ gt, int32_t* __restrict__ inter) {
    __shared__ int s_red[32];
    const OverlapItem it = items[blockIdx.x];
    const uint32_t* p = pred + it.pred;
    const uint32_t* g = gt + it.gt;
    int acc[kGtTile];
#pragma unroll
    for (int k = 0; k < kGtTile; ++k) acc[k] = 0;
    for (int w = threadIdx.x; w < it.words; w += blockDim.x) {
        const uint32_t pv = __ldg(p + w);
#pragma unroll
        for (int k = 0; k < kGtTile; ++k)
            if (k < it.ng) acc[k] += __popc(pv & __ldg(g + (long long)k * it.words + w));
    }
#pragma unroll
    for (int k = 0; k < kGtTile; ++k) {
        if (k >= it.ng) break;
        const int v = block_sum(acc[k], s_red);
        if (threadIdx.x == 0) inter[it.out + k] = v;
    }
}

template <typename T>
static size_t put(std::vector<char>& blob, const std::vector<T>& v) {      // append, 16-byte aligned; returns the byte offset
    const size_t o = align_up(blob.size(), 16);
    blob.resize(o + sizeof(T) * v.size());
    if (!v.empty()) std::memcpy(blob.data() + o, v.data(), sizeof(T) * v.size());
    return o;
}

static bool bad_size(int H, int W) { return H <= 0 || W <= 0 || (long long)H * W > (1ll << 30); }

}  // namespace irn

using namespace irn;

extern "C" long long irn_coco_plane_words(int H, int W) {
    if (bad_size(H, W)) return -1;
    return (long long)W * col_words(H);
}

// the rasteriser's layout: [descriptor blob | toggle planes]
static size_t raster_blob_bytes(int n_parts, int n_edges, int n_vertices, int n_toggles) {
    size_t b = align_up(sizeof(RasterPart) * n_parts, 16);
    b += align_up(sizeof(RasterEdge) * n_edges, 16);
    b += align_up(16 * (size_t)n_vertices, 16);
    b += align_up(8 * (size_t)n_toggles, 16);
    return align_up(b, 256);
}

extern "C" size_t irn_coco_raster_workspace_bytes(int n_parts, const int32_t* part_hw, int n_edges, int n_vertices, int n_toggles) {
    if (n_parts < 0 || n_edges < 0 || n_vertices < 0 || n_toggles < 0 || (n_parts > 0 && !part_hw)) return 0;
    size_t words = 0;
    for (int i = 0; i < n_parts; ++i) {
        if (bad_size(part_hw[2 * i], part_hw[2 * i + 1])) return 0;
        words += (size_t)part_hw[2 * i + 1] * col_words(part_hw[2 * i]);
    }
    return raster_blob_bytes(n_parts, n_edges, n_vertices, n_toggles) + 4 * words + 256;
}

extern "C" int irn_coco_rasterize(int n_ann, const int32_t* ann_hw, int n_parts, const int32_t* part_ann, int n_edges,
                                  const int32_t* edges, int n_vertices, const double* vertices, int n_toggles, const int32_t* toggles,
                                  uint32_t* planes, size_t plane_words, void* workspace, size_t workspace_bytes, irn_stream_t stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    launch_counter() = 0;
    if (n_ann < 0 || n_parts < 0 || n_edges < 0 || n_vertices < 0 || n_toggles < 0)
        return fail(kBadArg, "irn_coco_rasterize: negative count");
    if (n_ann == 0) return kOk;
    if (!ann_hw || (n_parts && !part_ann) || (n_edges && (!edges || !vertices)) || (n_toggles && !toggles))
        return fail(kBadArg, "irn_coco_rasterize: null pointer");
    std::vector<long long> ann_off(n_ann + 1, 0);
    for (int a = 0; a < n_ann; ++a) {
        if (bad_size(ann_hw[2 * a], ann_hw[2 * a + 1]))
            return fail(kBadArg, "irn_coco_rasterize: annotation %d has size %dx%d", a, ann_hw[2 * a], ann_hw[2 * a + 1]);
        ann_off[a + 1] = ann_off[a] + (long long)ann_hw[2 * a + 1] * col_words(ann_hw[2 * a]);
    }
    if ((size_t)ann_off[n_ann] != plane_words)
        return fail(kBadArg, "irn_coco_rasterize: %zu plane words, the sizes add up to %lld", plane_words, ann_off[n_ann]);
    if (!is_device_ptr(planes) || !is_device_ptr(workspace)) return fail(kBadArg, "irn_coco_rasterize: planes and workspace must be device memory");
    std::vector<RasterPart> parts(n_parts);
    std::vector<int32_t> part_hw(2 * (size_t)n_parts);
    long long tog_words = 0;
    for (int i = 0; i < n_parts; ++i) {
        const int a = part_ann[i];
        if (a < 0 || a >= n_ann) return fail(kBadArg, "irn_coco_rasterize: part %d names annotation %d of %d", i, a, n_ann);
        parts[i] = {tog_words, ann_off[a], ann_hw[2 * a], ann_hw[2 * a + 1]};
        part_hw[2 * i] = ann_hw[2 * a];
        part_hw[2 * i + 1] = ann_hw[2 * a + 1];
        tog_words += ann_off[a + 1] - ann_off[a];
    }
    std::vector<RasterEdge> ev(n_edges);
    for (int e = 0; e < n_edges; ++e) {
        const RasterEdge E = {edges[4 * e], edges[4 * e + 1], edges[4 * e + 2], edges[4 * e + 3]};
        if (E.part < 0 || E.part >= n_parts || E.k < 1 || E.j < 0 || E.j >= E.k || E.first < 0 || (long long)E.first + E.k > n_vertices)
            return fail(kBadArg, "irn_coco_rasterize: edge %d (part %d, vertices %d + %d, edge %d) out of range", e, E.part, E.first, E.k, E.j);
        ev[e] = E;
    }
    std::vector<int32_t> tv(toggles, toggles + 2 * (size_t)n_toggles);
    for (int i = 0; i < n_toggles; ++i) {
        const int p = tv[2 * i], pos = tv[2 * i + 1];
        if (p < 0 || p >= n_parts || pos < 0 || (long long)pos > (long long)parts[p].H * parts[p].W)
            return fail(kBadArg, "irn_coco_rasterize: toggle %d (part %d, position %d) out of range", i, p, pos);
    }
    const size_t need = irn_coco_raster_workspace_bytes(n_parts, part_hw.data(), n_edges, n_vertices, n_toggles);
    if (workspace_bytes < need) return fail(kWorkspace, "irn_coco_rasterize: workspace %zu < %zu bytes", workspace_bytes, need);
    std::vector<char> blob;
    const size_t o_parts = put(blob, parts), o_edges = put(blob, ev);
    const size_t o_xy = put(blob, std::vector<double>(vertices, vertices + 2 * (size_t)n_vertices));
    const size_t o_tog = put(blob, tv);
    char* ws = (char*)workspace;
    const size_t o_planes = raster_blob_bytes(n_parts, n_edges, n_vertices, n_toggles);
    uint32_t* tog = (uint32_t*)(ws + o_planes);
    IRN_CUDA(cudaMemcpyAsync(ws, blob.data(), blob.size(), cudaMemcpyHostToDevice, st));
    IRN_CUDA(cudaMemsetAsync(planes, 0, 4 * plane_words, st));
    if (n_parts == 0) return kOk;
    IRN_CUDA(cudaMemsetAsync(tog, 0, 4 * (size_t)tog_words, st));
    const RasterPart* d_parts = (const RasterPart*)(ws + o_parts);
    if (n_edges) {
        poly_toggle_kernel<<<(n_edges + 127) / 128, 128, 0, st>>>(d_parts, (const RasterEdge*)(ws + o_edges), n_edges,
                                                                 (const double*)(ws + o_xy), tog);
        IRN_LAUNCH_CHECK("poly_toggle_kernel");
    }
    if (n_toggles) {
        rle_toggle_kernel<<<(n_toggles + 255) / 256, 256, 0, st>>>(d_parts, (const int2*)(ws + o_tog), n_toggles, tog);
        IRN_LAUNCH_CHECK("rle_toggle_kernel");
    }
    fill_kernel<<<n_parts, kRasterThreads, 0, st>>>(d_parts, tog, planes);
    IRN_LAUNCH_CHECK("fill_kernel");
    return kOk;
}

extern "C" size_t irn_coco_pack_workspace_bytes(int n_img) {
    return n_img < 0 ? 0 : align_up(sizeof(PackImg) * (size_t)n_img, 256) + 256;
}

extern "C" int irn_coco_pack_masks(const uint8_t* masks, size_t mask_bytes, int n_img, const int32_t* hwm, uint32_t* planes,
                                   size_t plane_words, void* workspace, size_t workspace_bytes, irn_stream_t stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    launch_counter() = 0;
    if (n_img < 0) return fail(kBadArg, "irn_coco_pack_masks: n_img=%d", n_img);
    if (n_img == 0) return kOk;
    if (!hwm) return fail(kBadArg, "irn_coco_pack_masks: null sizes");
    std::vector<PackImg> imgs(n_img);
    long long src = 0, dst = 0, blocks = 0;
    for (int i = 0; i < n_img; ++i) {
        const int H = hwm[3 * i], W = hwm[3 * i + 1], M = hwm[3 * i + 2];
        if (bad_size(H, W) || M < 0) return fail(kBadArg, "irn_coco_pack_masks: image %d has %d masks of %dx%d", i, M, H, W);
        imgs[i] = {src, dst, H, W, M, (int)blocks};
        src += (long long)M * H * W;
        dst += (long long)M * W * col_words(H);
        blocks += (long long)M * col_words(H) * ((W + 31) >> 5);
        if (blocks > 0x7fffffffll) return fail(kUnsupported, "irn_coco_pack_masks: batch too large: split it");
    }
    if ((size_t)src != mask_bytes) return fail(kBadArg, "irn_coco_pack_masks: %zu mask bytes, the sizes add up to %lld", mask_bytes, src);
    if ((size_t)dst != plane_words) return fail(kBadArg, "irn_coco_pack_masks: %zu plane words, the sizes add up to %lld", plane_words, dst);
    if (workspace_bytes < irn_coco_pack_workspace_bytes(n_img))
        return fail(kWorkspace, "irn_coco_pack_masks: workspace %zu < %zu bytes", workspace_bytes, irn_coco_pack_workspace_bytes(n_img));
    if (blocks == 0) return kOk;
    if (!is_device_ptr(masks) || !is_device_ptr(planes) || !is_device_ptr(workspace))
        return fail(kBadArg, "irn_coco_pack_masks: masks, planes and workspace must be device memory");
    IRN_CUDA(cudaMemcpyAsync(workspace, imgs.data(), sizeof(PackImg) * n_img, cudaMemcpyHostToDevice, st));
    pack_kernel<<<(unsigned)blocks, 256, 0, st>>>((const PackImg*)workspace, n_img, masks, planes);
    IRN_LAUNCH_CHECK("pack_kernel");
    return kOk;
}

// items of an overlap call: [area items of the predictions | of the ground truth], then the overlap items
static void overlap_items(int n_img, const int32_t* hwmg, std::vector<AreaItem>& areas, std::vector<OverlapItem>& ov, int& n_pred_items) {
    long long po = 0, go = 0;
    int pa = 0, ga = 0;
    long long io = 0;
    std::vector<AreaItem> gt_areas;
    for (int i = 0; i < n_img; ++i) {
        const int H = hwmg[4 * i], W = hwmg[4 * i + 1], M = hwmg[4 * i + 2], G = hwmg[4 * i + 3];
        const int words = W * col_words(H);
        for (int m = 0; m < M; ++m) {
            areas.push_back({po + (long long)m * words, words, pa + m});
            for (int g0 = 0; g0 < G; g0 += kGtTile)
                ov.push_back({po + (long long)m * words, go + (long long)g0 * words, io + (long long)m * G + g0, words, min(kGtTile, G - g0)});
        }
        for (int g = 0; g < G; ++g) gt_areas.push_back({go + (long long)g * words, words, ga + g});
        po += (long long)M * words;
        go += (long long)G * words;
        pa += M;
        ga += G;
        io += (long long)M * G;
    }
    n_pred_items = (int)areas.size();
    areas.insert(areas.end(), gt_areas.begin(), gt_areas.end());
}

static int overlap_checks(int n_img, const int32_t* hwmg, long long* pw, long long* gw, long long* n_inter, long long* n_pred, long long* n_gt) {
    *pw = *gw = *n_inter = *n_pred = *n_gt = 0;
    for (int i = 0; i < n_img; ++i) {
        const int H = hwmg[4 * i], W = hwmg[4 * i + 1], M = hwmg[4 * i + 2], G = hwmg[4 * i + 3];
        if (bad_size(H, W) || M < 0 || G < 0) return i + 1;
        const long long words = (long long)W * col_words(H);
        *pw += M * words;
        *gw += G * words;
        *n_inter += (long long)M * G;
        *n_pred += M;
        *n_gt += G;
    }
    return 0;
}

extern "C" size_t irn_coco_overlap_workspace_bytes(int n_img, const int32_t* hwmg) {
    if (n_img < 0 || (n_img > 0 && !hwmg)) return 0;
    long long pw, gw, ni, np, ng;
    if (overlap_checks(n_img, hwmg, &pw, &gw, &ni, &np, &ng)) return 0;
    long long ov = 0;
    for (int i = 0; i < n_img; ++i) ov += (long long)hwmg[4 * i + 2] * ((hwmg[4 * i + 3] + kGtTile - 1) / kGtTile);
    return align_up(sizeof(AreaItem) * (size_t)(np + ng), 16) + align_up(sizeof(OverlapItem) * (size_t)ov, 16) + 256;
}

extern "C" int irn_coco_overlaps(const uint32_t* pred_planes, size_t pred_words, const uint32_t* gt_planes, size_t gt_words, int n_img,
                                 const int32_t* hwmg, int32_t* inter, int32_t* area_pred, int32_t* area_gt, void* workspace,
                                 size_t workspace_bytes, irn_stream_t stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    launch_counter() = 0;
    if (n_img < 0) return fail(kBadArg, "irn_coco_overlaps: n_img=%d", n_img);
    if (n_img == 0) return kOk;
    if (!hwmg) return fail(kBadArg, "irn_coco_overlaps: null sizes");
    long long pw, gw, ni, np, ng;
    if (int bad = overlap_checks(n_img, hwmg, &pw, &gw, &ni, &np, &ng))
        return fail(kBadArg, "irn_coco_overlaps: image %d has size %dx%d, %d predictions, %d ground truths", bad - 1, hwmg[4 * (bad - 1)],
                    hwmg[4 * (bad - 1) + 1], hwmg[4 * (bad - 1) + 2], hwmg[4 * (bad - 1) + 3]);
    if ((size_t)pw != pred_words || (size_t)gw != gt_words)
        return fail(kBadArg, "irn_coco_overlaps: %zu / %zu plane words, the sizes add up to %lld / %lld", pred_words, gt_words, pw, gw);
    if (ni > 0x7fffffffll || np + ng > 0x7fffffffll) return fail(kUnsupported, "irn_coco_overlaps: batch too large: split it");
    const size_t need = irn_coco_overlap_workspace_bytes(n_img, hwmg);
    if (workspace_bytes < need) return fail(kWorkspace, "irn_coco_overlaps: workspace %zu < %zu bytes", workspace_bytes, need);
    if (np + ng == 0) return kOk;
    if (!is_device_ptr(workspace) || (np && (!is_device_ptr(pred_planes) || !is_device_ptr(area_pred))) ||
        (ng && (!is_device_ptr(gt_planes) || !is_device_ptr(area_gt))) || (ni && !is_device_ptr(inter)))
        return fail(kBadArg, "irn_coco_overlaps: planes, outputs and workspace must be device memory");
    std::vector<AreaItem> areas;
    std::vector<OverlapItem> ov;
    int n_pred_items = 0;
    overlap_items(n_img, hwmg, areas, ov, n_pred_items);
    std::vector<char> blob;
    const size_t o_areas = put(blob, areas), o_ov = put(blob, ov);
    char* ws = (char*)workspace;
    IRN_CUDA(cudaMemcpyAsync(ws, blob.data(), blob.size(), cudaMemcpyHostToDevice, st));
    area_kernel<<<(unsigned)areas.size(), kOverlapThreads, 0, st>>>((const AreaItem*)(ws + o_areas), pred_planes, gt_planes, n_pred_items,
                                                                    area_pred, area_gt);
    IRN_LAUNCH_CHECK("area_kernel");
    if (!ov.empty()) {
        overlap_kernel<<<(unsigned)ov.size(), kOverlapThreads, 0, st>>>((const OverlapItem*)(ws + o_ov), pred_planes, gt_planes, inter);
        IRN_LAUNCH_CHECK("overlap_kernel");
    }
    return kOk;
}
