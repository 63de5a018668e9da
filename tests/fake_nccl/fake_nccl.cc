// fake_nccl.cc -- a test-only stand-in for the five NCCL calls the range-sharded scheduler makes
// (yadcc_b200/csrc/shard_host.inc), so that W ranks can run as W threads of one process on ONE GPU.
//
// Built as tests/fake_nccl/libnccl.so.2 (SONAME libnccl.so.2).  A process that loads it with RTLD_GLOBAL
// before the scheduler's dlopen("libnccl.so.2") gets this copy.  Every collective is a host rendezvous:
// sync the caller's stream, barrier, read every rank's send buffer, barrier (AllReduce runs in place),
// write the result with a copy ordered on the caller's stream.  Device memory is reached through the
// CUDA driver API, loaded at the first collective, so that the stand-in shares no runtime state with the
// scheduler's statically linked cudart and loads on a machine without a GPU.
//
// Every rank must make the same call in the same position (kind, count, type, op); anything else, or a
// barrier that waits longer than kTimeoutS, prints what each rank called and ends the process with
// kExitMismatch / kExitTimeout, so that a broken sharded protocol fails instead of hanging.
#include <dlfcn.h>
#include <unistd.h>

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

extern "C" {
// The NCCL ABI subset the scheduler uses (nccl.h, NCCL 2.x).
typedef enum { ncclSuccess = 0, ncclSystemError = 2, ncclInternalError = 3, ncclInvalidArgument = 4,
               ncclInvalidUsage = 5 } ncclResult_t;
typedef enum { ncclUint32 = 3 } ncclDataType_t;
typedef enum { ncclSum = 0 } ncclRedOp_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef struct FakeRank* ncclComm_t;
}

namespace {

constexpr int kExitMismatch = 86;
constexpr int kExitTimeout = 87;
constexpr int kTimeoutS = 120;
constexpr int kMaxRanks = 64;
constexpr char kMagic[8] = {'y', 'd', 'f', 'a', 'k', 'e', 'n', 'c'};

// ---- the driver API, resolved at the first collective --------------------------------------------------------
typedef int (*StreamSync)(void*);
typedef int (*DtoHAsync)(void*, unsigned long long, size_t, void*);
typedef int (*HtoDAsync)(unsigned long long, const void*, size_t, void*);
struct Driver {
  StreamSync sync = nullptr;
  DtoHAsync dtoh = nullptr;
  HtoDAsync htod = nullptr;
};

const Driver& driver() {
  static const Driver d = [] {
    Driver r;
    void* lib = dlopen("libcuda.so.1", RTLD_NOW | RTLD_LOCAL);
    if (!lib) { fprintf(stderr, "fake_nccl: cannot load libcuda.so.1: %s\n", dlerror()); _exit(kExitMismatch); }
    r.sync = reinterpret_cast<StreamSync>(dlsym(lib, "cuStreamSynchronize"));
    r.dtoh = reinterpret_cast<DtoHAsync>(dlsym(lib, "cuMemcpyDtoHAsync_v2"));
    r.htod = reinterpret_cast<HtoDAsync>(dlsym(lib, "cuMemcpyHtoDAsync_v2"));
    if (!r.sync || !r.dtoh || !r.htod) { fprintf(stderr, "fake_nccl: libcuda.so.1 lacks a symbol\n"); _exit(kExitMismatch); }
    return r;
  }();
  return d;
}

// Host-buffer mode (tests only): buffers are host memory, streams are ignored.
bool g_host_buffers = false;

void check_cu(int rc, const char* what) {
  if (rc != 0) { fprintf(stderr, "fake_nccl: %s failed with CUresult %d\n", what, rc); _exit(kExitMismatch); }
}
void stream_sync(void* st) {
  if (!g_host_buffers) check_cu(driver().sync(st), "cuStreamSynchronize");
}
void read_buf(void* dst, const void* src, size_t bytes, void* st) {
  if (!bytes) return;
  if (g_host_buffers) { memcpy(dst, src, bytes); return; }
  check_cu(driver().dtoh(dst, reinterpret_cast<unsigned long long>(src), bytes, st), "cuMemcpyDtoHAsync");
  check_cu(driver().sync(st), "cuStreamSynchronize");
}
// (a pageable source is staged before the call returns: `src` may change afterwards)
void write_buf(void* dst, const void* src, size_t bytes, void* st) {
  if (!bytes) return;
  if (g_host_buffers) { memcpy(dst, src, bytes); return; }
  check_cu(driver().htod(reinterpret_cast<unsigned long long>(dst), src, bytes, st), "cuMemcpyHtoDAsync");
}

// ---- communicators ------------------------------------------------------------------------------------------------
enum Kind : int { kAllGather = 1, kAllReduce = 2 };
const char* kind_name(int k) { return k == kAllGather ? "AllGather" : k == kAllReduce ? "AllReduce" : "-"; }

struct Call {
  uint64_t seq = 0;
  int kind = 0, type = -1, op = -1;
  size_t count = 0;
  const void* send = nullptr;
};

struct Comm {
  explicit Comm(int w) : world(w), calls(w) {}
  const int world;
  std::mutex mu;
  std::condition_variable cv;
  int joined = 0, arrived = 0, refs = 0;
  uint64_t generation = 0;
  std::vector<Call> calls;
  std::vector<uint8_t> seen;  // ranks that reached the current barrier (for the timeout report)

  void report(const char* why) {  // (mu held)
    fprintf(stderr, "fake_nccl: %s; calls by rank:\n", why);
    for (int r = 0; r < world; ++r) {
      const Call& c = calls[r];
      fprintf(stderr, "  rank %d: call #%llu %s count %zu type %d op %d%s\n", r, (unsigned long long)c.seq,
              kind_name(c.kind), c.count, c.type, c.op,
              seen.size() == size_t(world) && !seen[r] ? "  (not at the barrier)" : "");
    }
    fflush(stderr);
  }

  void barrier(int rank) {
    std::unique_lock<std::mutex> lk(mu);
    if (seen.size() != size_t(world)) seen.assign(world, 0);
    seen[rank] = 1;
    const uint64_t gen = generation;
    if (++arrived == world) {
      arrived = 0;
      seen.assign(world, 0);
      ++generation;
      cv.notify_all();
      return;
    }
    if (!cv.wait_for(lk, std::chrono::seconds(kTimeoutS), [&] { return generation != gen; })) {
      report("a barrier waited longer than 120 s");
      _exit(kExitTimeout);
    }
  }
};

std::mutex g_registry_mu;
std::map<std::string, Comm*> g_registry;  // communicators still waiting for ranks to join
uint64_t g_id_counter = 0;

struct Stats {
  unsigned long long collectives = 0, all_gathers = 0, all_reduces = 0, bytes = 0;
};
Stats g_stats[kMaxRanks];
std::mutex g_stats_mu;

}  // namespace

struct FakeRank {
  Comm* comm;
  int rank;
  uint64_t seq = 0;
  std::vector<uint8_t> out;  // staging of this rank's result
};

namespace {

ncclResult_t collective(FakeRank* h, int kind, const void* send, void* recv, size_t count, int type, int op,
                        void* stream) {
  if (!h) return ncclInvalidArgument;
  Comm& c = *h->comm;
  const int R = h->rank, W = c.world;
  stream_sync(stream);                                                        // 1. the send buffer is written
  {
    std::lock_guard<std::mutex> lk(c.mu);
    c.calls[R] = Call{++h->seq, kind, type, op, count, send};
  }
  c.barrier(R);                                                               // 2. everybody is here
  {
    std::lock_guard<std::mutex> lk(c.mu);
    for (int g = 0; g < W; ++g) {
      const Call& a = c.calls[g];
      if (a.seq != h->seq || a.kind != kind || a.count != count || a.type != type || a.op != op) {
        c.report("ranks disagree on a collective");
        _exit(kExitMismatch);
      }
    }
    if (type != ncclUint32 || (kind == kAllReduce && op != ncclSum)) {
      c.report("unsupported data type or reduction");
      _exit(kExitMismatch);
    }
  }
  const size_t bytes = count * 4;
  std::vector<uint32_t> part(count);
  if (kind == kAllGather) {
    h->out.resize(bytes * W);
    for (int g = 0; g < W; ++g) read_buf(h->out.data() + bytes * g, c.calls[g].send, bytes, stream);  // 3. rank-major
  } else {
    h->out.assign(bytes, 0);
    uint32_t* acc = reinterpret_cast<uint32_t*>(h->out.data());
    for (int g = 0; g < W; ++g) {
      read_buf(part.data(), c.calls[g].send, bytes, stream);
      for (size_t i = 0; i < count; ++i) acc[i] += part[i];  // the sum mod 2^32
    }
  }
  c.barrier(R);                                                               // 4. all reads done (in place)
  write_buf(recv, h->out.data(), h->out.size(), stream);                      // 5. ordered on the caller's stream
  if (R < kMaxRanks) {
    std::lock_guard<std::mutex> lk(g_stats_mu);
    Stats& s = g_stats[R];
    ++s.collectives;
    ++(kind == kAllGather ? s.all_gathers : s.all_reduces);
    s.bytes += h->out.size();
  }
  return ncclSuccess;
}

}  // namespace

extern "C" {

__attribute__((visibility("default"))) ncclResult_t ncclGetUniqueId(ncclUniqueId* id) {
  if (!id) return ncclInvalidArgument;
  memset(id, 0, sizeof *id);
  memcpy(id->internal, kMagic, sizeof kMagic);
  std::lock_guard<std::mutex> lk(g_registry_mu);
  const uint64_t k = ++g_id_counter, pid = (uint64_t)getpid();
  memcpy(id->internal + 8, &k, 8);
  memcpy(id->internal + 16, &pid, 8);
  return ncclSuccess;
}

__attribute__((visibility("default"))) ncclResult_t ncclCommInitRank(ncclComm_t* comm, int nranks, ncclUniqueId id,
                                                                      int rank) {
  if (!comm || nranks < 1 || rank < 0 || rank >= nranks || memcmp(id.internal, kMagic, sizeof kMagic) != 0)
    return ncclInvalidArgument;
  const std::string key(id.internal, sizeof id.internal);
  Comm* c;
  {
    std::lock_guard<std::mutex> lk(g_registry_mu);
    auto it = g_registry.find(key);
    if (it == g_registry.end()) it = g_registry.emplace(key, new Comm(nranks)).first;
    c = it->second;
    std::lock_guard<std::mutex> lc(c->mu);
    if (c->world != nranks || c->calls[rank].seq == ~0ull) return ncclInvalidUsage;
    c->calls[rank].seq = ~0ull;  // (taken; reset below)
    ++c->refs;
    if (++c->joined == nranks) g_registry.erase(it);  // an id names one communicator
  }
  auto* h = new FakeRank{c, rank};
  c->barrier(rank);  // blocks until all ranks have joined
  {
    std::lock_guard<std::mutex> lk(c->mu);
    c->calls[rank] = Call{};
  }
  c->barrier(rank);
  *comm = h;
  return ncclSuccess;
}

__attribute__((visibility("default"))) ncclResult_t ncclCommDestroy(ncclComm_t h) {
  if (!h) return ncclInvalidArgument;
  Comm* c = h->comm;
  delete h;
  bool last;
  {
    std::lock_guard<std::mutex> lk(c->mu);
    last = --c->refs == 0;
  }
  if (last) delete c;
  return ncclSuccess;
}

__attribute__((visibility("default"))) ncclResult_t ncclAllGather(const void* send, void* recv, size_t count,
                                                                   ncclDataType_t type, ncclComm_t h, void* stream) {
  return collective(h, kAllGather, send, recv, count, type, ncclSum, stream);
}

__attribute__((visibility("default"))) ncclResult_t ncclAllReduce(const void* send, void* recv, size_t count,
                                                                   ncclDataType_t type, ncclRedOp_t op, ncclComm_t h,
                                                                   void* stream) {
  return collective(h, kAllReduce, send, recv, count, type, op, stream);
}

__attribute__((visibility("default"))) const char* ncclGetErrorString(ncclResult_t r) {
  return r == ncclSuccess ? "success (fake_nccl)" : "error (fake_nccl)";
}

// Collectives rank `rank` made in this process, over all communicators: {calls, all-gathers, all-reduces, bytes
// written to its receive buffers}.  Also proves to a harness that this library is the libnccl.so.2 in use.
__attribute__((visibility("default"))) void yd_fake_nccl_stats(int rank, unsigned long long out[4]) {
  std::lock_guard<std::mutex> lk(g_stats_mu);
  const Stats s = rank >= 0 && rank < kMaxRanks ? g_stats[rank] : Stats{};
  out[0] = s.collectives;
  out[1] = s.all_gathers;
  out[2] = s.all_reduces;
  out[3] = s.bytes;
}

// Tests only: buffers are host memory and streams are ignored, so that the rendezvous runs without a GPU.
__attribute__((visibility("default"))) void yd_fake_nccl_host_buffers(int on) { g_host_buffers = on != 0; }

}  // extern "C"
