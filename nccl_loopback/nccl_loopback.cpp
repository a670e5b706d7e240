// Loopback NCCL: a stand-in for libnccl.so.2 that runs the G ranks of a communicator inside ONE process, any number
// of them on the same device.  TEST INFRASTRUCTURE ONLY: it lets the library's own NCCL paths (wva_comm_*, wva_group_*)
// run on a single GPU, which real NCCL refuses (two ranks on one device).
//
// It exports the entry points libwva_b200.so resolves with dlsym, plus loopback_counters for the tests.  The all-gather
// moves bytes with copies and events only, so no device work ever waits for work another rank has not yet enqueued:
//   1. every rank records a "ready" event on its stream and posts {send, count, sequence number};
//   2. host barrier;
//   3. every rank waits on the other ranks' "ready" events on its own stream, enqueues the G copies into its recv
//      (rank-order concatenation) and records a "done" event;
//   4. host barrier;
//   5. every rank waits on the other ranks' "done" events, so no send buffer is reused while a peer still reads it.
// Every host barrier has a timeout (NCCL_LOOPBACK_TIMEOUT_S seconds, default 60) and returns ncclSystemError when it
// expires, so a caller bug shows as a failing call, never as a wait that does not end.
#include <cuda_runtime.h>

#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

namespace {

enum {
    kSuccess = 0, kUnhandledCudaError = 1, kSystemError = 2, kInternalError = 3, kInvalidArgument = 4, kInvalidUsage = 5
};
constexpr int kInt8 = 0;
constexpr size_t kIdBytes = 128;
constexpr char kMagic[] = "nccl-loopback";

struct Comm;

struct Post {
    const void* send = nullptr;
    size_t count = 0;
    uint64_t seq = 0;
};

// the ranks of one communicator
struct Clique {
    int n = 0;
    std::mutex m;
    std::condition_variable cv;
    int arrived = 0;
    uint64_t generation = 0;
    bool broken = false;        // a barrier timed out: every later barrier fails at once
    std::vector<Comm*> ranks;
    std::vector<Post> posts;
};

struct Comm {
    Clique* clique = nullptr;
    int rank = 0, device = 0;
    uint64_t seq = 0;           // collectives issued
    uint64_t gathers = 0, last_bytes = 0;
    bool destroyed = false;
    cudaEvent_t ready = nullptr, done = nullptr;
};

std::mutex g_mu;                                    // guards everything below
std::map<std::string, Clique*> g_cliques;          // by unique id (ncclCommInitRank)
Clique* g_last = nullptr;                           // the most recently created communicator
uint64_t g_ids = 0, g_created = 0, g_destroyed = 0, g_group_start = 0, g_group_end = 0;

double timeout_s() {
    const char* e = std::getenv("NCCL_LOOPBACK_TIMEOUT_S");
    const double t = e ? std::atof(e) : 0.0;
    return t > 0 ? t : 60.0;
}

int barrier(Clique* c) {
    std::unique_lock<std::mutex> lk(c->m);
    if (c->broken) return kSystemError;
    const uint64_t gen = c->generation;
    if (++c->arrived == c->n) {
        c->arrived = 0;
        ++c->generation;
        c->cv.notify_all();
        return kSuccess;
    }
    const auto until = std::chrono::steady_clock::now() + std::chrono::duration<double>(timeout_s());
    const bool passed = c->cv.wait_until(lk, until, [&] { return c->generation != gen || c->broken; });
    if (passed && c->generation != gen) return kSuccess;
    c->broken = true;
    c->cv.notify_all();
    return kSystemError;
}

int make_events(Comm* k) {
    int prev = 0;
    if (cudaGetDevice(&prev) != cudaSuccess || cudaSetDevice(k->device) != cudaSuccess) return kUnhandledCudaError;
    const bool ok = cudaEventCreateWithFlags(&k->ready, cudaEventDisableTiming) == cudaSuccess &&
                    cudaEventCreateWithFlags(&k->done, cudaEventDisableTiming) == cudaSuccess;
    cudaSetDevice(prev);
    return ok ? kSuccess : kUnhandledCudaError;
}

Clique* new_clique(int n) {
    Clique* c = new Clique;
    c->n = n;
    c->ranks.assign((size_t)n, nullptr);
    c->posts.assign((size_t)n, Post{});
    g_last = c;
    return c;
}

}  // namespace

extern "C" {

typedef Comm* ncclComm_t;
struct ncclUniqueId { char internal[kIdBytes]; };

const char* ncclGetErrorString(int r) {
    switch (r) {
        case kSuccess: return "no error";
        case kUnhandledCudaError: return "unhandled cuda error (loopback)";
        case kSystemError: return "system error (loopback: a rank did not arrive in time)";
        case kInternalError: return "internal error (loopback)";
        case kInvalidArgument: return "invalid argument (loopback)";
        case kInvalidUsage: return "invalid usage (loopback: ranks disagree on the collective)";
        default: return "unknown result (loopback)";
    }
}

int ncclGetUniqueId(ncclUniqueId* id) {
    if (!id) return kInvalidArgument;
    std::memset(id->internal, 0, kIdBytes);
    std::lock_guard<std::mutex> lk(g_mu);
    std::snprintf(id->internal, kIdBytes, "%s:%llu", kMagic, (unsigned long long)++g_ids);
    return kSuccess;
}

int ncclCommInitRank(ncclComm_t* comm, int nranks, ncclUniqueId id, int rank) {
    if (!comm || nranks < 1 || rank < 0 || rank >= nranks) return kInvalidArgument;
    *comm = nullptr;
    Comm* k = new Comm;
    k->rank = rank;
    if (cudaGetDevice(&k->device) != cudaSuccess || make_events(k) != kSuccess) { delete k; return kUnhandledCudaError; }
    Clique* c;
    {
        std::lock_guard<std::mutex> lk(g_mu);
        const std::string key(id.internal, kIdBytes);
        auto it = g_cliques.find(key);
        c = it != g_cliques.end() ? it->second : (g_cliques[key] = new_clique(nranks));
        if (c->n != nranks || c->ranks[(size_t)rank]) { cudaEventDestroy(k->ready); cudaEventDestroy(k->done); delete k; return kInvalidUsage; }
        c->ranks[(size_t)rank] = k;
        k->clique = c;
        ++g_created;
    }
    const int rc = barrier(c);                      // the rendezvous: every rank has registered
    if (rc != kSuccess) {
        std::lock_guard<std::mutex> lk(g_mu);
        c->ranks[(size_t)rank] = nullptr;
        ++g_destroyed;
        cudaEventDestroy(k->ready); cudaEventDestroy(k->done);
        delete k;
        return rc;
    }
    *comm = k;
    return kSuccess;
}

int ncclCommInitAll(ncclComm_t* comms, int ndev, const int* devlist) {
    if (!comms || ndev < 1) return kInvalidArgument;
    std::lock_guard<std::mutex> lk(g_mu);
    Clique* c = new_clique(ndev);
    for (int i = 0; i < ndev; ++i) {
        Comm* k = new Comm;
        k->clique = c; k->rank = i; k->device = devlist ? devlist[i] : i;     // duplicate devices are allowed
        if (make_events(k) != kSuccess) return kUnhandledCudaError;
        c->ranks[(size_t)i] = k;
        comms[i] = k;
        ++g_created;
    }
    return kSuccess;
}

// not collective; the record stays so that loopback_counters can report on it afterwards
int ncclCommDestroy(ncclComm_t comm) {
    if (!comm) return kInvalidArgument;
    std::lock_guard<std::mutex> lk(g_mu);
    if (comm->destroyed) return kInvalidUsage;
    comm->destroyed = true;
    cudaEventDestroy(comm->ready); cudaEventDestroy(comm->done);
    comm->ready = comm->done = nullptr;
    ++g_destroyed;
    return kSuccess;
}

int ncclAllGather(const void* send, void* recv, size_t count, int datatype, ncclComm_t comm, cudaStream_t stream) {
    if (!comm || comm->destroyed) return kInvalidArgument;
    if (datatype != kInt8) return kInvalidArgument;
    Clique* c = comm->clique;
    const int me = comm->rank, G = c->n;
    int prev = 0;
    if (cudaGetDevice(&prev) != cudaSuccess || cudaSetDevice(comm->device) != cudaSuccess) return kUnhandledCudaError;
    int rc = kSuccess;
    if (cudaEventRecord(comm->ready, stream) != cudaSuccess) rc = kUnhandledCudaError;
    c->posts[(size_t)me] = Post{send, count, ++comm->seq};
    // every rank goes through both barriers whatever it finds, so no rank posts the next collective while a peer
    // still reads this one's posts
    int brc = barrier(c);
    bool agree = true;
    if (brc == kSuccess)
        for (int r = 0; r < G; ++r)
            agree = agree && c->posts[(size_t)r].count == count && c->posts[(size_t)r].seq == comm->seq;
    if (brc == kSuccess && agree && rc == kSuccess) {
        bool ok = true;
        for (int r = 0; r < G; ++r)
            if (r != me) ok = ok && cudaStreamWaitEvent(stream, c->ranks[(size_t)r]->ready, 0) == cudaSuccess;
        for (int r = 0; r < G && count > 0; ++r) {
            char* dst = (char*)recv + (size_t)r * count;
            const void* src = c->posts[(size_t)r].send;
            if (dst != src)
                ok = ok && cudaMemcpyPeerAsync(dst, comm->device, src, c->ranks[(size_t)r]->device, count, stream) == cudaSuccess;
        }
        ok = ok && cudaEventRecord(comm->done, stream) == cudaSuccess;
        if (!ok) rc = kUnhandledCudaError;
    }
    if (brc == kSuccess) brc = barrier(c);
    if (brc == kSuccess && agree && rc == kSuccess) {
        for (int r = 0; r < G; ++r)
            if (r != me && cudaStreamWaitEvent(stream, c->ranks[(size_t)r]->done, 0) != cudaSuccess) rc = kUnhandledCudaError;
    }
    cudaSetDevice(prev);
    if (brc != kSuccess) return brc;
    if (!agree) return kInvalidUsage;
    if (rc == kSuccess) { comm->gathers += 1; comm->last_bytes = count; }
    return rc;
}

// the library never groups its collectives: counted so that the tests can assert it
int ncclGroupStart(void) { std::lock_guard<std::mutex> lk(g_mu); ++g_group_start; return kSuccess; }
int ncclGroupEnd(void) { std::lock_guard<std::mutex> lk(g_mu); ++g_group_end; return kSuccess; }

// out[0..1]: all-gathers `comm` issued and the byte count of its last one (comm NULL: the rank-`rank` communicator of
// the most recently created clique); out[2]: 1 once that communicator is destroyed; out[3..6]: communicators
// created and destroyed, ncclGroupStart and ncclGroupEnd calls, over the whole process.
int loopback_counters(ncclComm_t comm, int rank, uint64_t out[7]) {
    if (!out) return kInvalidArgument;
    std::lock_guard<std::mutex> lk(g_mu);
    if (!comm && g_last && rank >= 0 && rank < g_last->n) comm = g_last->ranks[(size_t)rank];
    if (!comm) return kInvalidArgument;
    out[0] = comm->gathers; out[1] = comm->last_bytes; out[2] = comm->destroyed ? 1 : 0;
    out[3] = g_created; out[4] = g_destroyed; out[5] = g_group_start; out[6] = g_group_end;
    return kSuccess;
}

}  // extern "C"
