// faiss_b200 -- GPU runtime resources (L0).
//
// Mirrors the reference's GpuResources / StandardGpuResources contract
// (faiss/gpu/GpuResources.h:200-312, faiss/gpu/StandardGpuResources.cpp:337-625):
// per device, lazily initialised: one default (ordering) stream, 2 alternate streams, one
// async-copy stream, a pinned host staging buffer, a stack ("temp") arena with 256-byte
// aligned allocations that overflows to the driver allocator, and allocation bookkeeping
// (getMemoryInfo).  No cuBLAS handle is created: nothing on the hot path calls a library.
#pragma once

#include <algorithm>
#include <map>
#include <memory>
#include <mutex>
#include <unordered_map>
#include <vector>

#include "common.h"

namespace fb200 {

// faiss/gpu/GpuResources.h:31-65
enum class AllocType : int {
    Other = 0,
    FlatData = 1,
    IVFLists = 2,
    Quantizer = 3,
    QuantizerPrecomputedCodes = 4,
    TemporaryMemoryBuffer = 10,
    TemporaryMemoryOverflow = 11,
};
// faiss/gpu/GpuResources.h:71-79
enum class MemorySpace : int { Temporary = 0, Device = 1, Unified = 2 };

struct AllocRequest { // faiss/gpu/GpuResources.h:107-139
    AllocType type = AllocType::Other;
    int device = 0;
    MemorySpace space = MemorySpace::Device;
    cudaStream_t stream = nullptr;
    size_t size = 0;
};

class GpuResources;
class Communicator; // comm.h: one NCCL rank bound to a device

// RAII reservation (faiss/gpu/GpuResources.h:172-195)
struct GpuMemoryReservation {
    GpuMemoryReservation() = default;
    GpuMemoryReservation(GpuResources* r, int dev, cudaStream_t s, void* p, size_t sz)
            : res(r), device(dev), stream(s), data(p), size(sz) {}
    GpuMemoryReservation(GpuMemoryReservation&& m) noexcept {
        *this = std::move(m);
    }
    GpuMemoryReservation& operator=(GpuMemoryReservation&& m) noexcept;
    GpuMemoryReservation(const GpuMemoryReservation&) = delete;
    GpuMemoryReservation& operator=(const GpuMemoryReservation&) = delete;
    ~GpuMemoryReservation() {
        release();
    }
    void release();
    template <typename T>
    T* as() const {
        return reinterpret_cast<T*>(data);
    }
    GpuResources* res = nullptr;
    int device = 0;
    cudaStream_t stream = nullptr;
    void* data = nullptr;
    size_t size = 0;
};

class GpuResources { // faiss/gpu/GpuResources.h:200-281
   public:
    virtual ~GpuResources() = default;
    virtual void initializeForDevice(int device) = 0;
    virtual cudaStream_t getDefaultStream(int device) = 0;
    virtual void setDefaultStream(int device, cudaStream_t stream) = 0;
    virtual std::vector<cudaStream_t> getAlternateStreams(int device) = 0;
    virtual cudaStream_t getAsyncCopyStream(int device) = 0;
    virtual void* allocMemory(const AllocRequest& req) = 0;
    virtual void deallocMemory(int device, void* in) = 0;
    virtual size_t getTempMemoryAvailable(int device) const = 0;
    virtual std::pair<void*, size_t> getPinnedMemory() = 0;
    virtual int numSMs(int device) = 0;
    // the NCCL rank this resources object holds for `device` (null: the device is not part of a
    // communicator) -- SURVEY 7 step 1: NCCL communicator ownership lives with the resources
    virtual std::shared_ptr<Communicator> getCommunicator(int /*device*/) {
        return nullptr;
    }

    GpuMemoryReservation allocMemoryHandle(const AllocRequest& req) {
        return GpuMemoryReservation(this, req.device, req.stream, allocMemory(req), req.size);
    }
    // convenience: temp allocation on the default stream of `device`
    GpuMemoryReservation temp(int device, size_t bytes) {
        AllocRequest r;
        r.type = AllocType::TemporaryMemoryBuffer;
        r.device = device;
        r.space = MemorySpace::Temporary;
        r.stream = getDefaultStream(device);
        r.size = bytes;
        return allocMemoryHandle(r);
    }
    GpuMemoryReservation device_alloc(int device, size_t bytes, AllocType t) {
        AllocRequest r;
        r.type = t;
        r.device = device;
        r.space = MemorySpace::Device;
        r.stream = getDefaultStream(device);
        r.size = bytes;
        return allocMemoryHandle(r);
    }
    void syncDefaultStream(int device) {
        CUDA_VERIFY(cudaStreamSynchronize(getDefaultStream(device)));
    }
};

// faiss/gpu/utils/StackDeviceMemory.h:22-110 -- a bump allocator over one device region.
class StackDeviceMemory {
   public:
    StackDeviceMemory(int device, size_t size);
    ~StackDeviceMemory();
    void* alloc(size_t size); // returns nullptr when it does not fit
    bool owns(void* p) const {
        return p >= start_ && p < start_ + size_;
    }
    void dealloc(void* p);
    size_t available() const {
        return size_ - (head_ - start_);
    }
    size_t highWater() const {
        return high_;
    }

   private:
    int device_;
    char* start_ = nullptr;
    char* head_ = nullptr;
    size_t size_ = 0;
    size_t high_ = 0;
    // live allocations in address order: (ptr, size, freed?)
    struct Range {
        char* p;
        size_t sz;
        bool freed;
    };
    std::vector<Range> live_;
};

class StandardGpuResources : public GpuResources { // faiss/gpu/StandardGpuResources.h:199-266
   public:
    StandardGpuResources();
    ~StandardGpuResources() override;

    void noTempMemory() {
        setTempMemory(0);
    }
    void setTempMemory(size_t size);
    void setPinnedMemory(size_t size);
    void setDefaultStream(int device, cudaStream_t stream) override;
    void revertDefaultStream(int device);
    void setDefaultNullStreamAllDevices();
    void setLogMemoryAllocations(bool enable) {
        logAlloc_ = enable;
    }
    // {device: {allocType: (count, bytes)}}  (faiss/gpu/StandardGpuResources.cpp getMemoryInfo)
    std::map<int, std::map<std::string, std::pair<int, size_t>>> getMemoryInfo() const;

    void initializeForDevice(int device) override;
    cudaStream_t getDefaultStream(int device) override;
    std::vector<cudaStream_t> getAlternateStreams(int device) override;
    cudaStream_t getAsyncCopyStream(int device) override;
    void* allocMemory(const AllocRequest& req) override;
    void deallocMemory(int device, void* in) override;
    size_t getTempMemoryAvailable(int device) const override;
    std::pair<void*, size_t> getPinnedMemory() override;
    int numSMs(int device) override;

    // NCCL: one communicator per device.  ncclInitAll = every listed device of THIS process in one clique
    // (rank i = devices[i]); ncclInitRank = this process is rank `rank` of `nranks` (one process per GPU).
    void ncclInitAll(const std::vector<int>& devices);
    void ncclInitRank(int device, int nranks, int rank, const char* uniqueId128);
    void setCommunicator(int device, std::shared_ptr<Communicator> comm);
    std::shared_ptr<Communicator> getCommunicator(int device) override;

    // GpuResourcesProvider::getResources() equivalent: the object is its own provider.
    GpuResources* getResources() {
        return this;
    }

   private:
    struct PerDevice {
        cudaStream_t defaultStream = nullptr;
        cudaStream_t userDefaultStream = nullptr;
        bool hasUserStream = false;
        std::vector<cudaStream_t> altStreams;
        cudaStream_t asyncCopyStream = nullptr;
        std::unique_ptr<StackDeviceMemory> temp;
        int numSMs = 0;
    };
    struct AllocInfo {
        AllocRequest req;
        bool fromStack;
    };
    mutable std::recursive_mutex mu_;
    std::unordered_map<int, PerDevice> dev_;
    std::unordered_map<int, std::unordered_map<void*, AllocInfo>> allocs_;
    size_t tempMemSize_;
    bool tempMemSet_ = false;
    size_t pinnedSize_;
    void* pinned_ = nullptr;
    size_t pinnedAlloc_ = 0;
    bool allNull_ = false;
    bool logAlloc_ = false;
    std::unordered_map<int, std::shared_ptr<Communicator>> comms_;
};

// RAII device switch (faiss/gpu/utils/DeviceUtils.h DeviceScope)
struct DeviceScope {
    explicit DeviceScope(int device) {
        CUDA_VERIFY(cudaGetDevice(&prev_));
        if (prev_ != device) {
            CUDA_VERIFY(cudaSetDevice(device));
        } else {
            prev_ = -1;
        }
    }
    ~DeviceScope() {
        if (prev_ != -1)
            cudaSetDevice(prev_);
    }
    int prev_ = -1;
};

// -1 if host pointer, else device ordinal (faiss/gpu/utils/DeviceUtils.h:64)
int getDeviceForAddress(const void* p);

// RAII: a pointer that is guaranteed device-resident on `device` (copies host data in)
template <typename T>
struct DeviceView {
    DeviceView(GpuResources* res, int device, const T* p, size_t count, cudaStream_t stream) {
        if (!p || count == 0) {
            ptr = nullptr;
            return;
        }
        int dev = getDeviceForAddress(p);
        if (dev == device) {
            ptr = p;
        } else {
            hold = res->temp(device, count * sizeof(T));
            CUDA_VERIFY(cudaMemcpyAsync(hold.data, p, count * sizeof(T), cudaMemcpyDefault, stream));
            ptr = hold.as<T>();
        }
    }
    const T* ptr;
    GpuMemoryReservation hold;
};

// output staging: device buffer that is copied back to a host pointer on `finish`
template <typename T>
struct DeviceOut {
    DeviceOut(GpuResources* res, int device, T* p, size_t count) : user(p), n(count) {
        int dev = getDeviceForAddress(p);
        if (dev == device) {
            ptr = p;
        } else {
            hold = res->temp(device, count * sizeof(T));
            ptr = hold.as<T>();
            staged = true;
        }
    }
    void finish(cudaStream_t stream) {
        if (staged)
            CUDA_VERIFY(cudaMemcpyAsync(user, ptr, n * sizeof(T), cudaMemcpyDefault, stream));
    }
    T* user;
    T* ptr;
    size_t n;
    bool staged = false;
    GpuMemoryReservation hold;
};

// ------------------------------------------------------------------------------------------
// growable device array backed by GpuResources (role of DeviceVector, faiss/gpu/utils/DeviceVector.cuh)
// ------------------------------------------------------------------------------------------
template <typename T>
class DeviceVector {
   public:
    DeviceVector(GpuResources* res, int device, AllocType type) : res_(res), device_(device), type_(type) {}
    ~DeviceVector() {
        clear();
    }
    DeviceVector(const DeviceVector&) = delete;
    DeviceVector& operator=(const DeviceVector&) = delete;

    T* data() const {
        return data_;
    }
    size_t size() const {
        return size_;
    }
    size_t capacity() const {
        return cap_;
    }
    void clear() {
        if (data_)
            res_->deallocMemory(device_, data_);
        data_ = nullptr;
        size_ = cap_ = 0;
    }
    // ensure capacity >= n (exact if `exact`, else geometric growth), preserving contents
    void reserve(size_t n, cudaStream_t stream, bool exact = false) {
        if (n <= cap_)
            return;
        size_t ncap = exact ? n : std::max(n, cap_ + cap_ / 2);
        AllocRequest r;
        r.type = type_;
        r.device = device_;
        r.space = MemorySpace::Device;
        r.stream = stream;
        r.size = ncap * sizeof(T);
        T* nd = (T*)res_->allocMemory(r);
        if (size_ > 0) {
            CUDA_VERIFY(cudaMemcpyAsync(nd, data_, size_ * sizeof(T), cudaMemcpyDeviceToDevice, stream));
            CUDA_VERIFY(cudaStreamSynchronize(stream));
        }
        if (data_)
            res_->deallocMemory(device_, data_);
        data_ = nd;
        cap_ = ncap;
    }
    void resize(size_t n, cudaStream_t stream) {
        reserve(n, stream);
        size_ = n;
    }
    // append n elements from a host or device pointer
    void append(const T* src, size_t n, cudaStream_t stream) {
        if (n == 0)
            return;
        reserve(size_ + n, stream);
        CUDA_VERIFY(cudaMemcpyAsync(data_ + size_, src, n * sizeof(T), cudaMemcpyDefault, stream));
        size_ += n;
    }

   private:
    GpuResources* res_;
    int device_;
    AllocType type_;
    T* data_ = nullptr;
    size_t size_ = 0, cap_ = 0;
};

} // namespace fb200
