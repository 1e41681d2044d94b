// faiss_b200 -- StandardGpuResources implementation.  See resources.h for the reference map.
#include "resources.h"

#include "comm.h"

#include <algorithm>

namespace fb200 {

static const char* allocTypeName(AllocType t) {
    switch (t) {
        case AllocType::Other:
            return "Other";
        case AllocType::FlatData:
            return "FlatData";
        case AllocType::IVFLists:
            return "IVFLists";
        case AllocType::Quantizer:
            return "Quantizer";
        case AllocType::QuantizerPrecomputedCodes:
            return "QuantizerPrecomputedCodes";
        case AllocType::TemporaryMemoryBuffer:
            return "TemporaryMemoryBuffer";
        case AllocType::TemporaryMemoryOverflow:
            return "TemporaryMemoryOverflow";
    }
    return "Unknown";
}

GpuMemoryReservation& GpuMemoryReservation::operator=(GpuMemoryReservation&& m) noexcept {
    if (this != &m) {
        release();
        res = m.res;
        device = m.device;
        stream = m.stream;
        data = m.data;
        size = m.size;
        m.res = nullptr;
        m.data = nullptr;
        m.size = 0;
    }
    return *this;
}

void GpuMemoryReservation::release() {
    if (res && data) {
        res->deallocMemory(device, data);
    }
    res = nullptr;
    data = nullptr;
    size = 0;
}

int getDeviceForAddress(const void* p) {
    if (!p)
        return -1;
    cudaPointerAttributes att;
    cudaError_t err = cudaPointerGetAttributes(&att, p);
    if (err != cudaSuccess) {
        cudaGetLastError(); // clear
        return -1;
    }
    if (att.type == cudaMemoryTypeDevice || att.type == cudaMemoryTypeManaged) {
        return att.device;
    }
    return -1;
}

// ---------------------------------------------------------------- StackDeviceMemory
static constexpr size_t kAlign = 256; // faiss/gpu/StandardGpuResources.cpp:518-521

StackDeviceMemory::StackDeviceMemory(int device, size_t size) : device_(device), size_(size) {
    DeviceScope s(device);
    if (size_ > 0) {
        CUDA_VERIFY(cudaMalloc(&start_, size_));
    }
    head_ = start_;
}

StackDeviceMemory::~StackDeviceMemory() {
    if (start_) {
        DeviceScope s(device_);
        cudaFree(start_);
    }
}

void* StackDeviceMemory::alloc(size_t size) {
    size = round_up(std::max<size_t>(size, 1), kAlign);
    if (!start_ || size > available())
        return nullptr;
    char* p = head_;
    head_ += size;
    high_ = std::max<size_t>(high_, head_ - start_);
    live_.push_back({p, size, false});
    return p;
}

void StackDeviceMemory::dealloc(void* p) {
    for (auto it = live_.rbegin(); it != live_.rend(); ++it) {
        if (it->p == p) {
            it->freed = true;
            break;
        }
    }
    // pop every freed range at the top of the stack
    while (!live_.empty() && live_.back().freed) {
        head_ = live_.back().p;
        live_.pop_back();
    }
}

// ---------------------------------------------------------------- StandardGpuResources
// default pinned size 256 MiB (faiss/gpu/StandardGpuResources.cpp:49); default temp memory: the
// reference caps at 1.5 GiB for >8 GiB devices (:58,180-208).  An H100 carries 80 GB, and the
// fused Flat path wants candidate arenas resident, so the default here is 4 GiB.
StandardGpuResources::StandardGpuResources()
        : tempMemSize_(size_t(4) << 30), pinnedSize_(size_t(256) << 20) {}

StandardGpuResources::~StandardGpuResources() {
    for (auto& kv : dev_) {
        int device = kv.first;
        cudaSetDevice(device);
        // leaked user allocations are freed defensively
        for (auto& a : allocs_[device]) {
            if (!a.second.fromStack)
                cudaFree(a.first);
        }
        kv.second.temp.reset();
        if (kv.second.defaultStream)
            cudaStreamDestroy(kv.second.defaultStream);
        for (auto s : kv.second.altStreams)
            cudaStreamDestroy(s);
        if (kv.second.asyncCopyStream)
            cudaStreamDestroy(kv.second.asyncCopyStream);
    }
    if (pinned_)
        cudaFreeHost(pinned_);
}

void StandardGpuResources::setTempMemory(size_t size) {
    std::lock_guard<std::recursive_mutex> g(mu_);
    tempMemSize_ = size;
    tempMemSet_ = true;
    for (auto& kv : dev_) {
        // re-create the arena with the new size (only legal when nothing is live)
        kv.second.temp.reset();
        kv.second.temp.reset(new StackDeviceMemory(kv.first, tempMemSize_));
    }
}

void StandardGpuResources::setPinnedMemory(size_t size) {
    std::lock_guard<std::recursive_mutex> g(mu_);
    FB_THROW_IF_NOT_MSG(!pinned_, "pinned memory already allocated");
    pinnedSize_ = size;
}

void StandardGpuResources::setDefaultStream(int device, cudaStream_t stream) {
    std::lock_guard<std::recursive_mutex> g(mu_);
    initializeForDevice(device);
    auto& d = dev_[device];
    if (d.hasUserStream && d.userDefaultStream != stream) {
        // order the new stream after the previous one
        DeviceScope s(device);
        CUDA_VERIFY(cudaStreamSynchronize(d.userDefaultStream));
    }
    d.userDefaultStream = stream;
    d.hasUserStream = true;
}

void StandardGpuResources::revertDefaultStream(int device) {
    std::lock_guard<std::recursive_mutex> g(mu_);
    auto it = dev_.find(device);
    if (it != dev_.end() && it->second.hasUserStream) {
        DeviceScope s(device);
        CUDA_VERIFY(cudaStreamSynchronize(it->second.userDefaultStream));
        it->second.hasUserStream = false;
        it->second.userDefaultStream = nullptr;
    }
}

void StandardGpuResources::setDefaultNullStreamAllDevices() {
    std::lock_guard<std::recursive_mutex> g(mu_);
    allNull_ = true;
    for (auto& kv : dev_) {
        kv.second.userDefaultStream = nullptr;
        kv.second.hasUserStream = true;
    }
}

void StandardGpuResources::initializeForDevice(int device) {
    std::lock_guard<std::recursive_mutex> g(mu_);
    if (dev_.count(device))
        return;
    int ndev = 0;
    CUDA_VERIFY(cudaGetDeviceCount(&ndev));
    FB_THROW_IF_NOT_FMT(device >= 0 && device < ndev, "invalid device %d (have %d)", device, ndev);
    DeviceScope s(device);
    cudaDeviceProp prop;
    CUDA_VERIFY(cudaGetDeviceProperties(&prop, device));
    // this library carries sm_90a SASS only; fail loudly elsewhere
    FB_THROW_IF_NOT_FMT(
            prop.major == 9 && prop.minor == 0,
            "device %d is sm_%d%d; faiss_b200 kernels are built for sm_90a (H100) only",
            device,
            prop.major,
            prop.minor);
    FB_THROW_IF_NOT(prop.warpSize == 32); // faiss/gpu/StandardGpuResources.cpp:396-401

    // stream-ordered scratch (cudaMallocAsync in the k-means update / debug seams): keep up to 2 GiB in the
    // device's default pool instead of returning it to the driver at every synchronisation
    {
        cudaMemPool_t pool = nullptr;
        if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess && pool) {
            uint64_t keep = uint64_t(2) << 30;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
        }
        cudaGetLastError();
    }
    PerDevice d;
    d.numSMs = prop.multiProcessorCount;
    CUDA_VERIFY(cudaStreamCreateWithFlags(&d.defaultStream, cudaStreamNonBlocking));
    for (int i = 0; i < 2; i++) { // kNumStreams = 2 (faiss/gpu/StandardGpuResources.cpp:46)
        cudaStream_t st;
        CUDA_VERIFY(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
        d.altStreams.push_back(st);
    }
    CUDA_VERIFY(cudaStreamCreateWithFlags(&d.asyncCopyStream, cudaStreamNonBlocking));
    if (allNull_) {
        d.hasUserStream = true;
        d.userDefaultStream = nullptr;
    }
    size_t freeB = 0, totalB = 0;
    CUDA_VERIFY(cudaMemGetInfo(&freeB, &totalB));
    size_t want = tempMemSize_;
    if (!tempMemSet_) {
        want = std::min(want, freeB / 8);
    }
    d.temp.reset(new StackDeviceMemory(device, want));
    dev_.emplace(device, std::move(d));
    allocs_[device];
}

cudaStream_t StandardGpuResources::getDefaultStream(int device) {
    std::lock_guard<std::recursive_mutex> g(mu_);
    initializeForDevice(device);
    auto& d = dev_[device];
    return d.hasUserStream ? d.userDefaultStream : d.defaultStream;
}

std::vector<cudaStream_t> StandardGpuResources::getAlternateStreams(int device) {
    std::lock_guard<std::recursive_mutex> g(mu_);
    initializeForDevice(device);
    return dev_[device].altStreams;
}

cudaStream_t StandardGpuResources::getAsyncCopyStream(int device) {
    std::lock_guard<std::recursive_mutex> g(mu_);
    initializeForDevice(device);
    return dev_[device].asyncCopyStream;
}

int StandardGpuResources::numSMs(int device) {
    std::lock_guard<std::recursive_mutex> g(mu_);
    initializeForDevice(device);
    return dev_[device].numSMs;
}

std::pair<void*, size_t> StandardGpuResources::getPinnedMemory() {
    std::lock_guard<std::recursive_mutex> g(mu_);
    if (!pinned_ && pinnedSize_ > 0) {
        CUDA_VERIFY(cudaHostAlloc(&pinned_, pinnedSize_, cudaHostAllocDefault));
        pinnedAlloc_ = pinnedSize_;
    }
    return {pinned_, pinnedAlloc_};
}

size_t StandardGpuResources::getTempMemoryAvailable(int device) const {
    std::lock_guard<std::recursive_mutex> g(mu_);
    auto it = dev_.find(device);
    if (it == dev_.end() || !it->second.temp)
        return 0;
    return it->second.temp->available();
}

void* StandardGpuResources::allocMemory(const AllocRequest& reqIn) {
    std::lock_guard<std::recursive_mutex> g(mu_);
    initializeForDevice(reqIn.device);
    AllocRequest req = reqIn;
    if (req.size == 0)
        return nullptr;
    req.size = round_up(req.size, kAlign);
    DeviceScope s(req.device);
    void* p = nullptr;
    bool fromStack = false;
    auto& d = dev_[req.device];
    if (req.space == MemorySpace::Temporary) {
        p = d.temp->alloc(req.size);
        if (p) {
            fromStack = true;
        } else {
            // overflow to the driver allocator (faiss/gpu/StandardGpuResources.cpp:525-541)
            req.type = AllocType::TemporaryMemoryOverflow;
            req.space = MemorySpace::Device;
        }
    }
    if (!p) {
        cudaError_t err;
        if (req.space == MemorySpace::Unified) {
            err = cudaMallocManaged(&p, req.size);
        } else {
            err = cudaMalloc(&p, req.size);
        }
        if (err != cudaSuccess) {
            cudaGetLastError();
            // OOM -> exception with the allocation table (faiss/gpu/StandardGpuResources.cpp:557-577)
            std::string table;
            for (auto& dv : getMemoryInfo()) {
                for (auto& kv : dv.second) {
                    char line[160];
                    snprintf(
                            line,
                            sizeof(line),
                            " dev%d %s: %d allocs, %zu bytes;",
                            dv.first,
                            kv.first.c_str(),
                            kv.second.first,
                            kv.second.second);
                    table += line;
                }
            }
            FB_THROW_FMT(
                    "cudaMalloc error %s: failed to allocate %zu bytes of %s on device %d. Outstanding:%s",
                    cudaGetErrorString(err),
                    req.size,
                    allocTypeName(req.type),
                    req.device,
                    table.c_str());
        }
    }
    if (logAlloc_) {
        fprintf(stderr, "faiss_b200 alloc dev%d %s %zu B -> %p\n", req.device, allocTypeName(req.type), req.size, p);
    }
    allocs_[req.device][p] = AllocInfo{req, fromStack};
    return p;
}

void StandardGpuResources::deallocMemory(int device, void* p) {
    if (!p)
        return;
    std::lock_guard<std::recursive_mutex> g(mu_);
    auto& m = allocs_[device];
    auto it = m.find(p);
    if (it == m.end()) {
        fprintf(stderr, "faiss_b200: deallocMemory of unknown pointer %p on device %d\n", p, device);
        return;
    }
    DeviceScope s(device);
    if (it->second.fromStack) {
        // stack memory is reused by later work on the same ordering stream, which is
        // stream-ordered after every kernel that used it; alternate-stream users must have
        // joined the default stream before releasing (they do: see streamWait helpers).
        dev_[device].temp->dealloc(p);
    } else {
        // cudaFree synchronises with all outstanding work touching the allocation
        cudaError_t err = cudaFree(p);
        if (err != cudaSuccess) {
            fprintf(stderr, "faiss_b200: cudaFree failed: %s\n", cudaGetErrorString(err));
            cudaGetLastError();
        }
    }
    if (logAlloc_) {
        fprintf(stderr, "faiss_b200 free dev%d %p\n", device, p);
    }
    m.erase(it);
}

std::map<int, std::map<std::string, std::pair<int, size_t>>> StandardGpuResources::getMemoryInfo() const {
    std::lock_guard<std::recursive_mutex> g(mu_);
    std::map<int, std::map<std::string, std::pair<int, size_t>>> out;
    for (auto& dv : allocs_) {
        auto& o = out[dv.first];
        for (auto& a : dv.second) {
            auto& e = o[allocTypeName(a.second.req.type)];
            e.first += 1;
            e.second += a.second.req.size;
        }
    }
    return out;
}

} // namespace fb200

// ---------------------------------------------------------------- launch counter / kernel timing
#include <atomic>
#include <cstring>

namespace fb200 {

long long& kernelLaunchCounter() {
    static long long c = 0;
    return c;
}

namespace {
struct TimedLaunch {
    std::string name;
    cudaEvent_t a, b;
};
std::mutex g_tmu;
bool g_timing = false;
std::vector<TimedLaunch> g_timed;
thread_local cudaEvent_t g_pendingStart = nullptr; // begin/end pair up per launching thread
} // namespace

void StandardGpuResources::ncclInitAll(const std::vector<int>& devices) {
    for (int d : devices)
        initializeForDevice(d);
    auto comms = Communicator::initAll(devices);
    std::lock_guard<std::recursive_mutex> g(mu_);
    for (size_t i = 0; i < devices.size(); i++)
        comms_[devices[i]] = comms[i];
}

void StandardGpuResources::ncclInitRank(int device, int nranks, int rank, const char* uniqueId128) {
    initializeForDevice(device);
    auto c = Communicator::initRank(device, nranks, rank, uniqueId128);
    std::lock_guard<std::recursive_mutex> g(mu_);
    comms_[device] = c;
}

void StandardGpuResources::setCommunicator(int device, std::shared_ptr<Communicator> comm) {
    std::lock_guard<std::recursive_mutex> g(mu_);
    if (comm)
        comms_[device] = std::move(comm);
    else
        comms_.erase(device);
}

std::shared_ptr<Communicator> StandardGpuResources::getCommunicator(int device) {
    std::lock_guard<std::recursive_mutex> g(mu_);
    auto it = comms_.find(device);
    return it == comms_.end() ? nullptr : it->second;
}

void KernelTiming::enable(bool on) {
    std::lock_guard<std::mutex> g(g_tmu);
    g_timing = on;
}
bool KernelTiming::enabled() {
    return g_timing;
}
void KernelTiming::begin(const char*, cudaStream_t stream) {
    if (!g_timing)
        return;
    std::lock_guard<std::mutex> g(g_tmu);
    cudaEventCreate(&g_pendingStart);
    cudaEventRecord(g_pendingStart, stream);
}
void KernelTiming::end(const char* name, cudaStream_t stream) {
    if (!g_timing || !g_pendingStart)
        return;
    std::lock_guard<std::mutex> g(g_tmu);
    TimedLaunch t;
    t.name = name;
    t.a = g_pendingStart;
    cudaEventCreate(&t.b);
    cudaEventRecord(t.b, stream);
    g_pendingStart = nullptr;
    g_timed.push_back(t);
}
void KernelTiming::collect(const char* name, double* ms, int* launches) {
    std::lock_guard<std::mutex> g(g_tmu);
    double tot = 0;
    int n = 0;
    std::vector<TimedLaunch> keep;
    for (auto& t : g_timed) {
        if (t.name == name) {
            cudaEventSynchronize(t.b);
            float e = 0;
            cudaEventElapsedTime(&e, t.a, t.b);
            tot += e;
            n++;
            cudaEventDestroy(t.a);
            cudaEventDestroy(t.b);
        } else {
            keep.push_back(t);
        }
    }
    g_timed.swap(keep);
    if (ms)
        *ms = tot;
    if (launches)
        *launches = n;
}

} // namespace fb200
