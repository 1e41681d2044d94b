// faiss_b200 -- IDSelector membership (faiss/impl/IDSelector.cpp) and its evaluation into slot masks.
//
// A selector tree is compiled on the host into a postfix program; one kernel evaluates it for every slot
// (one thread per slot, the 32 slots of a warp give one mask word through a ballot).  Array / Batch leaves
// become one sorted, de-duplicated device array searched by bisection; Bitmap leaves are uploaded as they
// are; a callback leaf is evaluated on the host over the stored ids and uploaded as its own slot mask.
#include <algorithm>
#include <cub/cub.cuh>

#include "idselector.h"
#include "select.cuh"

namespace fb200 {

// ------------------------------------------------------------------------------------------
// host: construction and is_member
// ------------------------------------------------------------------------------------------
IDSelector* IDSelector::range(idx_t imin, idx_t imax) {
    auto* s = new IDSelector(RANGE);
    s->imin = imin;
    s->imax = imax;
    return s;
}

static IDSelector* setOf(IDSelector* s, size_t n, const idx_t* ids) {
    FB_THROW_IF_NOT_MSG(n == 0 || ids != nullptr, "null id array passed to an IDSelector");
    s->ids.assign(ids, ids + n);
    std::sort(s->ids.begin(), s->ids.end());
    s->ids.erase(std::unique(s->ids.begin(), s->ids.end()), s->ids.end());
    return s;
}
IDSelector* IDSelector::array(size_t n, const idx_t* ids) {
    return setOf(new IDSelector(ARRAY), n, ids);
}
IDSelector* IDSelector::batch(size_t n, const idx_t* ids) {
    return setOf(new IDSelector(BATCH), n, ids);
}
IDSelector* IDSelector::bitmapOf(size_t n, const uint8_t* bitmap) {
    FB_THROW_IF_NOT_MSG(n == 0 || bitmap != nullptr, "null bitmap passed to IDSelectorBitmap");
    auto* s = new IDSelector(BITMAP);
    s->bitmap.assign(bitmap, bitmap + n);
    return s;
}
IDSelector* IDSelector::negation(const IDSelector* sel) {
    FB_THROW_IF_NOT_MSG(sel != nullptr, "null IDSelector operand");
    auto* s = new IDSelector(NOT);
    s->lhs = sel;
    return s;
}
IDSelector* IDSelector::binary(Kind kind, const IDSelector* lhs, const IDSelector* rhs) {
    FB_THROW_IF_NOT_MSG(lhs != nullptr && rhs != nullptr, "null IDSelector operand");
    FB_THROW_IF_NOT(kind == AND || kind == OR || kind == XOR);
    auto* s = new IDSelector(kind);
    s->lhs = lhs;
    s->rhs = rhs;
    return s;
}
IDSelector* IDSelector::callback(Fn fn, void* ctx) {
    FB_THROW_IF_NOT_MSG(fn != nullptr, "null IDSelector callback");
    auto* s = new IDSelector(CALLBACK);
    s->fn = fn;
    s->ctx = ctx;
    return s;
}

bool IDSelector::is_member(idx_t id) const {
    switch (kind) {
        case RANGE:
            return id >= imin && id < imax;
        case ARRAY:
        case BATCH:
            return std::binary_search(ids.begin(), ids.end(), id);
        case BITMAP: {
            const uint64_t u = (uint64_t)id;
            return (u >> 3) < bitmap.size() && ((bitmap[u >> 3] >> (u & 7)) & 1);
        }
        case NOT:
            return !lhs->is_member(id);
        case AND:
            return lhs->is_member(id) && rhs->is_member(id);
        case OR:
            return lhs->is_member(id) || rhs->is_member(id);
        case XOR:
            return lhs->is_member(id) != rhs->is_member(id);
        case CALLBACK:
            return fn(ctx, id) != 0;
    }
    return false;
}

bool IDSelector::usesCallback() const {
    return kind == CALLBACK || (lhs && lhs->usesCallback()) || (rhs && rhs->usesCallback());
}

// ------------------------------------------------------------------------------------------
// device: the postfix program
// ------------------------------------------------------------------------------------------
namespace {

enum SelOpKind : int { OP_RANGE, OP_SET, OP_BITMAP, OP_SLOTBITS, OP_NOT, OP_AND, OP_OR, OP_XOR };

struct SelOp {
    int kind;
    int64_t a, b; // RANGE: [a, b); SET: ids[a, a + b); BITMAP: bytes[a, a + b); SLOTBITS: slot words from a
};

constexpr int kMaxSelDepth = 64; // evaluation stack: one bit per level

struct SelProgram {
    std::vector<SelOp> ops;
    std::vector<idx_t> ids;
    std::vector<uint8_t> bytes;
    std::vector<uint32_t> slotBits;
    int depth = 0, maxDepth = 0;
};

void push(SelProgram& p, const SelOp& op, int delta) {
    p.ops.push_back(op);
    p.depth += delta;
    p.maxDepth = std::max(p.maxDepth, p.depth);
}

void compile(const IDSelector& s, SelProgram& p, int64_t n, const std::vector<idx_t>& hostIds, const uint8_t* valid) {
    switch (s.kind) {
        case IDSelector::RANGE:
            push(p, {OP_RANGE, s.imin, s.imax}, 1);
            return;
        case IDSelector::ARRAY:
        case IDSelector::BATCH:
            push(p, {OP_SET, (int64_t)p.ids.size(), (int64_t)s.ids.size()}, 1);
            p.ids.insert(p.ids.end(), s.ids.begin(), s.ids.end());
            return;
        case IDSelector::BITMAP:
            push(p, {OP_BITMAP, (int64_t)p.bytes.size(), (int64_t)s.bitmap.size()}, 1);
            p.bytes.insert(p.bytes.end(), s.bitmap.begin(), s.bitmap.end());
            return;
        case IDSelector::CALLBACK: {
            const int64_t words = slotMaskWords(n), base = (int64_t)p.slotBits.size();
            p.slotBits.resize(base + words, 0u);
            for (int64_t i = 0; i < n; i++) {
                if (valid && !valid[i])
                    continue;
                const idx_t id = hostIds.empty() ? i : hostIds[i];
                if (s.fn(s.ctx, id) != 0)
                    p.slotBits[base + (i >> 5)] |= 1u << (i & 31);
            }
            push(p, {OP_SLOTBITS, base, 0}, 1);
            return;
        }
        case IDSelector::NOT:
            compile(*s.lhs, p, n, hostIds, valid);
            push(p, {OP_NOT, 0, 0}, 0);
            return;
        case IDSelector::AND:
        case IDSelector::OR:
        case IDSelector::XOR:
            compile(*s.lhs, p, n, hostIds, valid);
            compile(*s.rhs, p, n, hostIds, valid);
            push(p, {s.kind == IDSelector::AND ? OP_AND : s.kind == IDSelector::OR ? OP_OR : OP_XOR, 0, 0}, -1);
            return;
    }
}

__global__ void slot_mask_kernel(
        const SelOp* __restrict__ prog,
        int nops,
        const idx_t* __restrict__ slotIds,
        int64_t n,
        const idx_t* __restrict__ setIds,
        const uint8_t* __restrict__ bytes,
        const uint32_t* __restrict__ slotBits,
        uint32_t* __restrict__ mask) {
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long stack = 0;
    if (s < n) {
        const idx_t id = slotIds ? slotIds[s] : (idx_t)s;
        for (int i = 0; i < nops; i++) {
            const SelOp op = prog[i];
            unsigned long long v;
            switch (op.kind) {
                case OP_RANGE:
                    v = id >= op.a && id < op.b;
                    break;
                case OP_SET: { // first position >= id in the sorted ids
                    int64_t lo = op.a, hi = op.a + op.b;
                    while (lo < hi) {
                        const int64_t mid = (lo + hi) >> 1;
                        if (setIds[mid] < id)
                            lo = mid + 1;
                        else
                            hi = mid;
                    }
                    v = lo < op.a + op.b && setIds[lo] == id;
                    break;
                }
                case OP_BITMAP: {
                    const uint64_t u = (uint64_t)id;
                    v = (u >> 3) < (uint64_t)op.b && ((bytes[op.a + (int64_t)(u >> 3)] >> (u & 7)) & 1);
                    break;
                }
                case OP_SLOTBITS:
                    v = (slotBits[op.a + (s >> 5)] >> (s & 31)) & 1u;
                    break;
                case OP_NOT:
                    stack ^= 1ull;
                    continue;
                default: { // binary operators: the two top entries -> one
                    const unsigned long long r = stack & 1ull, l = (stack >> 1) & 1ull;
                    stack >>= 2;
                    v = op.kind == OP_AND ? (l & r) : op.kind == OP_OR ? (l | r) : (l ^ r);
                    break;
                }
            }
            stack = (stack << 1) | v;
        }
    }
    const unsigned word = __ballot_sync(kFullMask, s < n && (stack & 1ull));
    if ((threadIdx.x & 31) == 0 && s < n)
        mask[s >> 5] = word;
}

template <typename T>
GpuMemoryReservation upload(GpuResources* res, int device, const std::vector<T>& v, cudaStream_t stream) {
    auto r = res->temp(device, sizeof(T) * std::max<size_t>(1, v.size()));
    if (!v.empty())
        CUDA_VERIFY(cudaMemcpyAsync(r.data, v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice, stream));
    return r;
}

// set bits of word w, the bits at or past n excluded
struct MaskPopc {
    const uint32_t* m;
    int64_t n;
    __device__ int operator()(int64_t w) const {
        const int64_t rest = n - w * 32;
        const uint32_t keep = rest >= 32 ? 0xffffffffu : ((1u << rest) - 1u);
        return __popc(m[w] & keep);
    }
};

struct MaskBit {
    const uint32_t* m;
    __device__ bool operator()(idx_t r) const {
        return (m[r >> 5] >> (r & 31)) & 1u;
    }
};

__global__ void remap_labels_kernel(idx_t* labels, int64_t count, const idx_t* __restrict__ ids) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count && labels[i] >= 0)
        labels[i] = ids[labels[i]];
}

} // namespace

void buildSlotMask(
        GpuResources* res,
        int device,
        const IDSelector& sel,
        int64_t n,
        const idx_t* idsDev,
        const uint8_t* valid,
        uint32_t* maskDev,
        cudaStream_t stream) {
    if (n == 0)
        return;
    std::vector<idx_t> hostIds; // a callback leaf is called with the stored ids
    if (idsDev && sel.usesCallback()) {
        hostIds.resize((size_t)n);
        CUDA_VERIFY(cudaMemcpyAsync(hostIds.data(), idsDev, sizeof(idx_t) * n, cudaMemcpyDeviceToHost, stream));
        CUDA_VERIFY(cudaStreamSynchronize(stream));
    }
    SelProgram p;
    compile(sel, p, n, hostIds, valid);
    FB_THROW_IF_NOT_FMT(p.maxDepth <= kMaxSelDepth, "IDSelector nested too deeply (%d levels, at most %d)", p.maxDepth, kMaxSelDepth);
    auto ops = upload(res, device, p.ops, stream);
    auto ids = upload(res, device, p.ids, stream);
    auto bytes = upload(res, device, p.bytes, stream);
    auto bits = upload(res, device, p.slotBits, stream);
    KernelTiming::begin("sel_mask", stream);
    slot_mask_kernel<<<(unsigned)ceil_div(n, (int64_t)256), 256, 0, stream>>>(
            ops.as<SelOp>(), (int)p.ops.size(), idsDev, n, ids.as<idx_t>(), bytes.as<uint8_t>(), bits.as<uint32_t>(),
            maskDev);
    KernelTiming::end("sel_mask", stream);
    CUDA_CHECK_LAST();
    // the host vectors above are the sources of pending copies
    CUDA_VERIFY(cudaStreamSynchronize(stream));
}

int64_t runCountMask(GpuResources* res, int device, const uint32_t* maskDev, int64_t n, cudaStream_t stream) {
    if (n == 0)
        return 0;
    const int64_t words = slotMaskWords(n);
    FB_THROW_IF_NOT(words < (int64_t(1) << 31));
    auto sum = res->temp(device, sizeof(int64_t));
    cub::TransformInputIterator<int64_t, MaskPopc, cub::CountingInputIterator<int64_t>> bits(
            cub::CountingInputIterator<int64_t>(0), MaskPopc{maskDev, n});
    size_t tmpBytes = 0;
    CUDA_VERIFY(cub::DeviceReduce::Sum(nullptr, tmpBytes, bits, sum.as<int64_t>(), (int)words, stream));
    auto tmp = res->temp(device, tmpBytes);
    CUDA_VERIFY(cub::DeviceReduce::Sum(tmp.data, tmpBytes, bits, sum.as<int64_t>(), (int)words, stream));
    int64_t h = 0;
    CUDA_VERIFY(cudaMemcpyAsync(&h, sum.data, sizeof(int64_t), cudaMemcpyDeviceToHost, stream));
    CUDA_VERIFY(cudaStreamSynchronize(stream));
    return h;
}

// DeviceSelect counts items in int: rows are compacted a page of at most 2^30 at a time, each page's selected
// rows written after the previous page's
int64_t runCompactMask(GpuResources* res, int device, const uint32_t* maskDev, int64_t n, idx_t* rowsOut, cudaStream_t stream) {
    constexpr int64_t kPage = int64_t(1) << 30;
    auto count = res->temp(device, sizeof(int));
    size_t tmpBytes = 0;
    CUDA_VERIFY(cub::DeviceSelect::If(
            nullptr, tmpBytes, cub::CountingInputIterator<idx_t>(0), rowsOut, count.as<int>(), (int)std::min(n, kPage),
            MaskBit{maskDev}, stream));
    auto tmp = res->temp(device, tmpBytes);
    int64_t total = 0;
    for (int64_t r0 = 0; r0 < n; r0 += kPage) {
        const int np = (int)std::min(kPage, n - r0);
        CUDA_VERIFY(cub::DeviceSelect::If(
                tmp.data, tmpBytes, cub::CountingInputIterator<idx_t>(r0), rowsOut + total, count.as<int>(), np,
                MaskBit{maskDev}, stream));
        int h = 0;
        CUDA_VERIFY(cudaMemcpyAsync(&h, count.data, sizeof(int), cudaMemcpyDeviceToHost, stream));
        CUDA_VERIFY(cudaStreamSynchronize(stream));
        total += h;
    }
    return total;
}

void runRemapLabels(idx_t* labels, int64_t count, const idx_t* ids, cudaStream_t stream) {
    if (count == 0)
        return;
    remap_labels_kernel<<<(unsigned)ceil_div(count, (int64_t)256), 256, 0, stream>>>(labels, count, ids);
    CUDA_CHECK_LAST();
}

} // namespace fb200
