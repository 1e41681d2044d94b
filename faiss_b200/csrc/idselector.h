// faiss_b200 -- IDSelector (faiss/impl/IDSelector.h): the filter of SearchParameters::sel, and its evaluation
// into a per-slot bit mask on the device.
//
// Membership is the CPU's is_member (faiss/impl/IDSelector.{h,cpp}):
//   Range   imin <= id < imax
//   Array, Batch   id is one of the given ids
//   Bitmap  (uint64)id >> 3 < n && bit (id & 7) of byte id >> 3
//   Not / And / Or / XOr   the logical operators on their children
//   Callback   fn(ctx, id) != 0: a selector the library cannot see into (evaluated on the host)
// Leaves copy their inputs at construction.  Combinators hold their children by pointer, as the reference's do:
// the children must outlive them.
#pragma once

#include <cstdint>
#include <vector>

#include "common.h"
#include "resources.h"

namespace fb200 {

struct IDSelector {
    enum Kind { RANGE, ARRAY, BATCH, BITMAP, NOT, AND, OR, XOR, CALLBACK };
    typedef int (*Fn)(void* ctx, idx_t id);

    Kind kind;
    idx_t imin = 0, imax = 0;           // RANGE
    std::vector<idx_t> ids;             // ARRAY, BATCH: sorted, without duplicates
    std::vector<uint8_t> bitmap;        // BITMAP: n bytes
    const IDSelector* lhs = nullptr;    // NOT (its operand), AND, OR, XOR
    const IDSelector* rhs = nullptr;    // AND, OR, XOR
    Fn fn = nullptr;                    // CALLBACK
    void* ctx = nullptr;

    static IDSelector* range(idx_t imin, idx_t imax);
    static IDSelector* array(size_t n, const idx_t* ids);
    static IDSelector* batch(size_t n, const idx_t* ids);
    static IDSelector* bitmapOf(size_t n, const uint8_t* bitmap);
    static IDSelector* negation(const IDSelector* sel);
    static IDSelector* binary(Kind kind, const IDSelector* lhs, const IDSelector* rhs);
    static IDSelector* callback(Fn fn, void* ctx);

    bool is_member(idx_t id) const;
    bool usesCallback() const; // is a callback leaf part of the tree?

   private:
    explicit IDSelector(Kind k) : kind(k) {}
};

// 32-bit words of a mask over n slots: bit (s & 31) of word s >> 5 is slot s
inline int64_t slotMaskWords(int64_t n) {
    return (n + 31) / 32;
}

// Evaluates `sel` over n slots into maskDev [slotMaskWords(n)] (device).  The id of slot s is idsDev[s]
// (device), or s itself when idsDev is null.  Slots with valid[s] == 0 (host, may be null) are storage that
// holds no entry: a callback leaf is not called for them and their bit is unspecified.  Enqueued on `stream`;
// the callback leaves and the upload of the selector's tables synchronise with the host.
void buildSlotMask(
        GpuResources* res,
        int device,
        const IDSelector& sel,
        int64_t n,
        const idx_t* idsDev,
        const uint8_t* valid,
        uint32_t* maskDev,
        cudaStream_t stream);

// number of set bits among the first n of a mask (synchronises with the host)
int64_t runCountMask(GpuResources* res, int device, const uint32_t* maskDev, int64_t n, cudaStream_t stream);

// row mask -> ascending list of the selected rows (device), returns their count.  rowsOut (device) holds at
// least as many entries as the mask has set bits among its first n.
int64_t runCompactMask(GpuResources* res, int device, const uint32_t* maskDev, int64_t n, idx_t* rowsOut, cudaStream_t stream);

// labels of a search over the compacted rows -> row ids (ids[label], -1 stays -1), in place
void runRemapLabels(idx_t* labels, int64_t count, const idx_t* ids, cudaStream_t stream);

} // namespace fb200
