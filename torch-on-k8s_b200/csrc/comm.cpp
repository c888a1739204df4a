// comm.cpp — replica communicator: binds one worker replica to one GPU, owns its symmetric heap
// (CUDA VMM, exported as POSIX fds), exchanges handles with the job's other replicas over a unix
// socket, optionally binds an NVSwitch multicast object, re-forms the group in place on elastic
// add/drop, and launches the kernels of allreduce.cu as plan.cpp decides.
//
// Reference side: this is what stands behind the env contract of
// TorchJobReconciler.SetClusterSpec (controllers/train/torchjob_controller.go:394-446):
// RANK / WORLD_SIZE keep their meaning, MASTER_ADDR:MASTER_PORT is replaced by a unix-socket path
// (single box, no DNS/Services).  The elastic path replaces restartStalePod /
// restartPodInKruiseProtocol (controllers/train/elastic_scale.go:303-397): survivors are not
// restarted, only the membership changes.
#include <cuda.h>
#include <cuda_runtime.h>
#include <errno.h>
#include <fcntl.h>
#include <poll.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/socket.h>
#include <sys/stat.h>
#include <sys/time.h>
#include <sys/types.h>
#include <sys/un.h>
#include <time.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <mutex>
#include <random>
#include <string>
#include <vector>

#include "plan.h"

namespace tok {

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_err;

static void vset_error(const char* fmt, va_list ap) {
  char buf[1024];
  vsnprintf(buf, sizeof(buf), fmt, ap);
  g_err = buf;
}

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vset_error(fmt, ap);
  va_end(ap);
}

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vset_error(fmt, ap);
  va_end(ap);
  return code;
}

const char* last_error_cstr() { return g_err.c_str(); }

// ------------------------------------------------------------------------------------------------
// driver API, resolved through the runtime so that libtok8s.so has no link-time dependency on
// libcuda.so (it must load — and its control plane must work — on a box without a driver).
// ------------------------------------------------------------------------------------------------
#define TOK_DRV_FNS(X)             \
  X(cuGetErrorString)              \
  X(cuDeviceGet)                   \
  X(cuDeviceGetAttribute)          \
  X(cuMemGetAllocationGranularity) \
  X(cuMemCreate)                   \
  X(cuMemRelease)                  \
  X(cuMemAddressReserve)           \
  X(cuMemAddressFree)              \
  X(cuMemMap)                      \
  X(cuMemUnmap)                    \
  X(cuMemSetAccess)                \
  X(cuMemExportToShareableHandle)  \
  X(cuMemImportFromShareableHandle) \
  X(cuMulticastCreate)             \
  X(cuMulticastAddDevice)          \
  X(cuMulticastBindMem)            \
  X(cuMulticastUnbind)             \
  X(cuMulticastGetGranularity)

struct Drv {
#define X(n) decltype(&n) n##_ = nullptr;
  TOK_DRV_FNS(X)
#undef X
  bool ok = false;
  std::string why;
};

static Drv& drv() {
  static Drv d;
  static std::once_flag once;
  std::call_once(once, [] {
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
      d.why = std::string("no CUDA device: ") + cudaGetErrorString(e);
      cudaGetLastError();
      return;
    }
#define X(n)                                                                          \
  {                                                                                   \
    void* fp = nullptr;                                                               \
    cudaDriverEntryPointQueryResult qr;                                               \
    e = cudaGetDriverEntryPoint(#n, &fp, cudaEnableDefault, &qr);                     \
    if (e != cudaSuccess || fp == nullptr || qr != cudaDriverEntryPointSuccess) {     \
      d.why = std::string("driver entry point missing: ") + #n;                       \
      cudaGetLastError();                                                             \
      return;                                                                         \
    }                                                                                 \
    d.n##_ = reinterpret_cast<decltype(&n)>(fp);                                      \
  }
    TOK_DRV_FNS(X)
#undef X
    d.ok = true;
  });
  return d;
}

static const char* cu_err(CUresult r) {
  const char* s = nullptr;
  if (drv().cuGetErrorString_ && drv().cuGetErrorString_(r, &s) == CUDA_SUCCESS && s) return s;
  return "unknown CUresult";
}

#define CU_CHECK(call)                                                                 \
  do {                                                                                 \
    CUresult _r = (call);                                                              \
    if (_r != CUDA_SUCCESS)                                                            \
      return fail(TOK_ERR_CUDA, "%s failed: %s (%d)", #call, cu_err(_r), (int)_r);     \
  } while (0)
#define RT_CHECK(call)                                                                 \
  do {                                                                                 \
    cudaError_t _e = (call);                                                           \
    if (_e != cudaSuccess)                                                             \
      return fail(TOK_ERR_CUDA, "%s failed: %s", #call, cudaGetErrorString(_e));       \
  } while (0)

static size_t env_size(const char* name, size_t dflt) {
  const char* v = getenv(name);
  if (!v || !*v) return dflt;
  char* end = nullptr;
  unsigned long long x = strtoull(v, &end, 10);
  if (end == v) return dflt;
  return static_cast<size_t>(x);
}

static size_t round_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

static double now_s() {
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return ts.tv_sec + ts.tv_nsec * 1e-9;
}

// ------------------------------------------------------------------------------------------------
// unix-socket plumbing (star topology around the group's rank 0)
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kMagic = 0x746f6b38u;  // "tok8"

struct Hello {
  uint32_t magic;
  uint32_t abi;
  uint64_t epoch;
  int32_t rank;
  int32_t world;
  int32_t device;
  int32_t pid;
  uint64_t uid;
  uint64_t heap_bytes;
  uint64_t cap_bytes;
  int32_t mc_supported;
  int32_t reserved;
  char bus_id[32];
  char job[64];
};

// Owns one descriptor of a heap or multicast handle (exported by the driver or received from a
// peer) and closes it when it goes out of scope, on every exit path.
struct Fd {
  int fd = -1;
  Fd() = default;
  Fd(Fd&& o) noexcept : fd(o.fd) { o.fd = -1; }
  Fd& operator=(Fd&& o) noexcept {
    std::swap(fd, o.fd);
    return *this;
  }
  ~Fd() {
    if (fd >= 0) close(fd);
  }
};

static int wait_fd(int fd, short events, double deadline) {
  for (;;) {
    double left = deadline - now_s();
    if (left <= 0) return 0;
    struct pollfd p = {fd, events, 0};
    int r = poll(&p, 1, static_cast<int>(std::min(left, 1.0) * 1000) + 1);
    if (r > 0) return 1;
    if (r < 0 && errno != EINTR) return -1;
  }
}

// Sends buf (len bytes) with nfds descriptors attached to the first byte.
static int send_msg(int sock, const void* buf, size_t len, const int* fds, int nfds,
                    double deadline) {
  const char* p = static_cast<const char*>(buf);
  size_t sent = 0;
  bool first = true;
  while (sent < len) {
    if (wait_fd(sock, POLLOUT, deadline) <= 0) return -1;
    struct msghdr msg;
    memset(&msg, 0, sizeof(msg));
    struct iovec iov = {const_cast<char*>(p + sent), len - sent};
    msg.msg_iov = &iov;
    msg.msg_iovlen = 1;
    std::vector<char> ctrl;
    if (first && nfds > 0) {
      ctrl.resize(CMSG_SPACE(sizeof(int) * nfds));
      msg.msg_control = ctrl.data();
      msg.msg_controllen = ctrl.size();
      struct cmsghdr* c = CMSG_FIRSTHDR(&msg);
      c->cmsg_level = SOL_SOCKET;
      c->cmsg_type = SCM_RIGHTS;
      c->cmsg_len = CMSG_LEN(sizeof(int) * nfds);
      memcpy(CMSG_DATA(c), fds, sizeof(int) * nfds);
    }
    ssize_t n = sendmsg(sock, &msg, MSG_NOSIGNAL);
    if (n < 0) {
      if (errno == EINTR || errno == EAGAIN) continue;
      return -1;
    }
    sent += static_cast<size_t>(n);
    first = false;
  }
  return 0;
}

// Receives exactly len bytes; descriptors that arrive with them are appended to fds_out (closed
// when fds_out is null).
static int recv_msg(int sock, void* buf, size_t len, std::vector<Fd>* fds_out, double deadline) {
  char* p = static_cast<char*>(buf);
  size_t got = 0;
  while (got < len) {
    if (wait_fd(sock, POLLIN, deadline) <= 0) return -1;
    struct msghdr msg;
    memset(&msg, 0, sizeof(msg));
    struct iovec iov = {p + got, len - got};
    msg.msg_iov = &iov;
    msg.msg_iovlen = 1;
    char ctrl[CMSG_SPACE(sizeof(int) * 16)];
    msg.msg_control = ctrl;
    msg.msg_controllen = sizeof(ctrl);
    ssize_t n = recvmsg(sock, &msg, 0);
    if (n < 0) {
      if (errno == EINTR || errno == EAGAIN) continue;
      return -1;
    }
    if (n == 0) return -1;  // peer closed
    for (struct cmsghdr* c = CMSG_FIRSTHDR(&msg); c; c = CMSG_NXTHDR(&msg, c)) {
      if (c->cmsg_level == SOL_SOCKET && c->cmsg_type == SCM_RIGHTS) {
        int cnt = static_cast<int>((c->cmsg_len - CMSG_LEN(0)) / sizeof(int));
        for (int i = 0; i < cnt; ++i) {
          Fd fd;
          memcpy(&fd.fd, CMSG_DATA(c) + i * sizeof(int), sizeof(int));
          if (fds_out) fds_out->push_back(std::move(fd));
        }
      }
    }
    got += static_cast<size_t>(n);
  }
  return 0;
}

struct Star {
  bool root = false;
  int world = 0;
  int listen_fd = -1;
  std::vector<int> conn;  // root: conn[rank] for rank != 0 ; member: conn[0] = link to root
  std::string path;
  bool abstract_sock = false;  // the socket lives in the abstract namespace: no file to unlink
  double deadline = 0;

  ~Star() { close_all(); }
  void close_all() {
    for (int& c : conn)
      if (c >= 0) {
        close(c);
        c = -1;
      }
    if (listen_fd >= 0) {
      close(listen_fd);
      listen_fd = -1;
      if (!abstract_sock) unlink(path.c_str());
    }
  }
  // Collective AND of a per-member status, returned to everyone.
  int all_ok(int my_ok, int* out) {
    if (root) {
      int acc = my_ok ? 1 : 0;
      for (int r = 1; r < world; ++r) {
        int v = 0;
        if (recv_msg(conn[r], &v, sizeof(v), nullptr, deadline) != 0)
          return fail(TOK_ERR_RENDEZVOUS, "rendezvous: lost rank %d during barrier", r);
        acc &= (v ? 1 : 0);
      }
      for (int r = 1; r < world; ++r)
        if (send_msg(conn[r], &acc, sizeof(acc), nullptr, 0, deadline) != 0)
          return fail(TOK_ERR_RENDEZVOUS, "rendezvous: cannot release rank %d", r);
      *out = acc;
    } else {
      int v = my_ok ? 1 : 0;
      if (send_msg(conn[0], &v, sizeof(v), nullptr, 0, deadline) != 0 ||
          recv_msg(conn[0], &v, sizeof(v), nullptr, deadline) != 0)
        return fail(TOK_ERR_RENDEZVOUS, "rendezvous: lost the group root during barrier");
      *out = v;
    }
    return TOK_OK;
  }
};

}  // namespace tok

// ------------------------------------------------------------------------------------------------
// the communicator
// ------------------------------------------------------------------------------------------------
using namespace tok;

struct PeerMap {
  uint64_t uid = 0;
  CUmemGenericAllocationHandle handle = 0;
  CUdeviceptr va = 0;
};

struct tok_comm {
  std::string job_id;
  std::string rdzv_path;
  int rank = 0, world = 1, max_world = 1, device = 0;
  uint64_t uid = 0;
  uint64_t epoch = 0;
  CUdevice cu_dev = 0;
  char bus_id[32] = {0};
  int sm_count = 132;
  int mc_supported = 0;

  size_t gran = 0;
  size_t cap_bytes = 0;
  size_t pool_bytes = 0;   // symmetric pool for zero-copy buckets
  size_t pool_used = 0;    // bump pointer (identical allocation sequence on every replica)
  std::vector<std::pair<size_t, size_t>> pool_free;  // (offset, bytes) of released segments, by offset
  std::mutex pool_mu;      // tok_pool_malloc may be entered from any allocator-calling thread
  size_t heap_bytes = 0;
  CUmemGenericAllocationHandle local_handle = 0;
  CUdeviceptr local_va = 0;

  std::vector<PeerMap> cache;      // every peer heap currently imported and mapped (not our own)
  char* peer[kMaxWorld] = {0};     // by current rank

  bool mc_bound = false;
  CUmemGenericAllocationHandle mc_handle = 0;
  CUdeviceptr mc_va = 0;

  unsigned long long* dbg = nullptr;    // device, only with TOK_DEBUG_PHASES=1
  uint32_t* ctr = nullptr;              // device
  volatile uint32_t* hostctl = nullptr; // pinned host page
  uint32_t* hostctl_dev = nullptr;

  Tunables tun;

  std::atomic<uint64_t> launches{0};    // exchange / broadcast / local kernels
  std::atomic<uint64_t> arrivals{0};    // arrive kernels
  std::atomic<uint64_t> elided{0};      // world-1 identity buckets that needed no launch
  std::atomic<uint64_t> broadcasts{0};
  std::atomic<int> last_algo{0};
  std::atomic<int> last_ctas{0};
  bool membership_dirty = false;  // exchange() got far enough to touch the peer mappings
};

static std::atomic<tok_comm*> g_pool_comm{nullptr};  // communicator behind tok_pool_malloc()

namespace {

struct DeviceGuard {
  int prev = -1;
  bool changed = false;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) == cudaSuccess && prev != dev) {
      cudaSetDevice(dev);
      changed = true;
    }
  }
  ~DeviceGuard() {
    if (changed) cudaSetDevice(prev);
  }
};

// Gives back a heap-sized VA range reserved by map_heap() and clears *va.  `mapped` is false only
// for a reservation whose cuMemMap failed.
void unmap(tok_comm* c, CUdeviceptr* va, bool mapped = true) {
  if (!*va) return;
  if (mapped) drv().cuMemUnmap_(*va, c->heap_bytes);
  drv().cuMemAddressFree_(*va, c->heap_bytes);
  *va = 0;
}

// Maps a heap-sized handle (our own heap, a peer's heap, or the multicast object) read-write for
// this replica's GPU.  On failure *va is 0 and nothing is left reserved.
int map_heap(tok_comm* c, CUmemGenericAllocationHandle h, CUdeviceptr* va) {
  Drv& d = drv();
  CU_CHECK(d.cuMemAddressReserve_(va, c->heap_bytes, c->gran, 0, 0));
  CUresult r = d.cuMemMap_(*va, c->heap_bytes, 0, h, 0);
  if (r != CUDA_SUCCESS) {
    unmap(c, va, false);
    return fail(TOK_ERR_CUDA, "cuMemMap failed: %s", cu_err(r));
  }
  CUmemAccessDesc acc;
  memset(&acc, 0, sizeof(acc));
  acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  acc.location.id = c->cu_dev;
  acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  r = d.cuMemSetAccess_(*va, c->heap_bytes, &acc, 1);
  if (r != CUDA_SUCCESS) {
    unmap(c, va);
    return fail(TOK_ERR_CUDA,
                "cuMemSetAccess on a peer heap failed: %s (no P2P path between the replicas' GPUs?)",
                cu_err(r));
  }
  return TOK_OK;
}

void release_peer(tok_comm* c, PeerMap& m) {
  unmap(c, &m.va);
  if (m.handle) drv().cuMemRelease_(m.handle);
  m = PeerMap();
}

void teardown_multicast(tok_comm* c) {
  Drv& d = drv();
  unmap(c, &c->mc_va);
  if (c->mc_handle) {
    if (c->mc_bound) d.cuMulticastUnbind_(c->mc_handle, c->cu_dev, 0, c->heap_bytes);
    d.cuMemRelease_(c->mc_handle);
    c->mc_handle = 0;
  }
  c->mc_bound = false;
}

int alloc_local(tok_comm* c) {
  Drv& d = drv();
  CUmemAllocationProp prop;
  memset(&prop, 0, sizeof(prop));
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = c->cu_dev;
  prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  size_t gran = 0;
  CU_CHECK(d.cuMemGetAllocationGranularity_(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
  c->gran = std::max<size_t>(gran, 2u << 20);

  int mc = 0;
  d.cuDeviceGetAttribute_(&mc, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, c->cu_dev);
  c->mc_supported = (mc && !c->tun.disable_nvls) ? 1 : 0;
  size_t total = kFlagBytes + 2 * c->cap_bytes + c->pool_bytes;
  if (c->mc_supported && c->max_world > 1) {
    CUmulticastObjectProp mp;
    memset(&mp, 0, sizeof(mp));
    mp.numDevices = static_cast<unsigned>(c->max_world);
    mp.size = round_up(total, c->gran);
    mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    size_t mg = 0;
    if (d.cuMulticastGetGranularity_(&mg, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED) ==
            CUDA_SUCCESS &&
        mg > 0 && mg <= (1ull << 30))
      c->gran = std::max(c->gran, mg);
    else if (d.cuMulticastGetGranularity_(&mg, &mp, CU_MULTICAST_GRANULARITY_MINIMUM) ==
                 CUDA_SUCCESS &&
             mg > 0)
      c->gran = std::max(c->gran, mg);
  }
  c->heap_bytes = round_up(total, c->gran);
  c->pool_bytes = c->heap_bytes - kFlagBytes - 2 * c->cap_bytes;  // rounding slack joins the pool
  CU_CHECK(d.cuMemCreate_(&c->local_handle, c->heap_bytes, &prop, 0));
  int rc = map_heap(c, c->local_handle, &c->local_va);
  if (rc != TOK_OK) return rc;
  RT_CHECK(cudaMemset(reinterpret_cast<void*>(c->local_va), 0, kFlagBytes));
  RT_CHECK(cudaMalloc(reinterpret_cast<void**>(&c->ctr), kCtrWords * sizeof(uint32_t)));
  RT_CHECK(cudaMemset(c->ctr, 0, kCtrWords * sizeof(uint32_t)));
  if (env_size("TOK_DEBUG_PHASES", 0)) {
    RT_CHECK(cudaMalloc(reinterpret_cast<void**>(&c->dbg), kMaxCtas * 8 * sizeof(unsigned long long)));
    RT_CHECK(cudaMemset(c->dbg, 0, kMaxCtas * 8 * sizeof(unsigned long long)));
  }
  void* hp = nullptr;
  RT_CHECK(cudaHostAlloc(&hp, 4096, cudaHostAllocMapped | cudaHostAllocPortable));
  memset(hp, 0, 4096);
  c->hostctl = static_cast<volatile uint32_t*>(hp);
  void* dp = nullptr;
  RT_CHECK(cudaHostGetDevicePointer(&dp, hp, 0));
  c->hostctl_dev = static_cast<uint32_t*>(dp);
  return TOK_OK;
}

// Step 1 of an exchange: gathers every member's Hello + heap fd at the group's rank 0 and scatters
// the full table, with every member's fd, back.  `star` keeps the group's sockets for later steps.
int rendezvous(tok_comm* c, Star& star, std::vector<Hello>& table, std::vector<Fd>& fds) {
  star.root = (c->rank == 0);
  star.world = c->world;
  star.deadline = now_s() + c->tun.rdzv_timeout_s;
  char suffix[32];
  snprintf(suffix, sizeof(suffix), ".e%llu", static_cast<unsigned long long>(c->epoch));
  star.path = c->rdzv_path + suffix;
  struct sockaddr_un addr;
  memset(&addr, 0, sizeof(addr));
  addr.sun_family = AF_UNIX;
  // A socket path must fit sun_path (108 bytes); a rendezvous file under a long directory (a
  // deep TMPDIR, say) gets a socket in the abstract namespace instead, named by a hash of its path
  // so that every replica of the group derives the same name.  An abstract name has no filesystem
  // permissions: any process in the same network namespace could bind it first.  The group still
  // checks every Hello (magic, ABI, job, epoch, rank) and maps only heaps whose identity token
  // matches, so a squatter makes the rendezvous fail rather than join; a short rendezvous path in a
  // private directory avoids the abstract namespace altogether.
  star.abstract_sock = star.path.size() >= sizeof(addr.sun_path);
  const bool abstract_sock = star.abstract_sock;
  if (abstract_sock) {
    uint64_t h = 1469598103934665603ull;  // FNV-1a
    for (unsigned char ch : star.path) h = (h ^ ch) * 1099511628211ull;
    snprintf(addr.sun_path + 1, sizeof(addr.sun_path) - 1, "tok8s-%016llx",
             static_cast<unsigned long long>(h));
  } else {
    strcpy(addr.sun_path, star.path.c_str());
  }

  Hello me;
  memset(&me, 0, sizeof(me));
  me.magic = kMagic;
  me.abi = TOK_ABI_VERSION;
  me.epoch = c->epoch;
  me.rank = c->rank;
  me.world = c->world;
  me.device = c->device;
  me.pid = static_cast<int32_t>(getpid());
  me.uid = c->uid;
  me.heap_bytes = c->heap_bytes;
  me.cap_bytes = c->cap_bytes;
  me.mc_supported = c->mc_supported;
  memcpy(me.bus_id, c->bus_id, sizeof(me.bus_id));
  snprintf(me.job, sizeof(me.job), "%s", c->job_id.c_str());

  Fd my_fd;
  if (c->world > 1)
    CU_CHECK(drv().cuMemExportToShareableHandle_(&my_fd.fd, c->local_handle,
                                                 CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));

  if (c->world == 1) {
    table[0] = me;
  } else if (star.root) {
    star.listen_fd = socket(AF_UNIX, SOCK_STREAM | SOCK_CLOEXEC, 0);
    if (star.listen_fd < 0) return fail(TOK_ERR_RENDEZVOUS, "socket(): %s", strerror(errno));
    if (!abstract_sock) unlink(star.path.c_str());
    if (bind(star.listen_fd, reinterpret_cast<struct sockaddr*>(&addr), sizeof(addr)) != 0 ||
        listen(star.listen_fd, kMaxWorld) != 0)
      return fail(TOK_ERR_RENDEZVOUS, "bind/listen(%s): %s", star.path.c_str(), strerror(errno));
    star.conn.assign(c->world, -1);
    table[0] = me;
    fds.resize(c->world);
    fds[0] = std::move(my_fd);
    for (int joined = 1; joined < c->world; ++joined) {
      if (wait_fd(star.listen_fd, POLLIN, star.deadline) <= 0)
        return fail(TOK_ERR_RENDEZVOUS,
                    "rendezvous %s: only %d of %d replicas joined within %.0f s", star.path.c_str(),
                    joined, c->world, c->tun.rdzv_timeout_s);
      int s = accept4(star.listen_fd, nullptr, nullptr, SOCK_CLOEXEC);
      if (s < 0) {
        --joined;
        continue;
      }
      Hello h;
      std::vector<Fd> got;
      if (recv_msg(s, &h, sizeof(h), &got, star.deadline) != 0 || h.magic != kMagic ||
          got.size() != 1) {
        close(s);
        return fail(TOK_ERR_RENDEZVOUS, "rendezvous %s: malformed hello", star.path.c_str());
      }
      const bool bad = h.abi != TOK_ABI_VERSION || h.epoch != c->epoch || h.world != c->world ||
                       h.rank <= 0 || h.rank >= c->world || star.conn[h.rank] >= 0 ||
                       h.heap_bytes != c->heap_bytes || h.cap_bytes != c->cap_bytes ||
                       strncmp(h.job, me.job, sizeof(h.job)) != 0;
      if (bad) {
        close(s);
        return fail(TOK_ERR_RENDEZVOUS,
                    "rendezvous %s: replica rank=%d world=%d epoch=%llu heap=%llu job=%.63s does not "
                    "match this group (world=%d epoch=%llu heap=%llu job=%s)",
                    star.path.c_str(), h.rank, h.world, (unsigned long long)h.epoch,
                    (unsigned long long)h.heap_bytes, h.job, c->world,
                    (unsigned long long)c->epoch, (unsigned long long)c->heap_bytes, me.job);
      }
      star.conn[h.rank] = s;
      table[h.rank] = h;
      fds[h.rank] = std::move(got[0]);
    }
    std::vector<int> raw;
    for (const Fd& f : fds) raw.push_back(f.fd);
    for (int r = 1; r < c->world; ++r)
      if (send_msg(star.conn[r], table.data(), sizeof(Hello) * c->world, raw.data(), c->world,
                   star.deadline) != 0)
        return fail(TOK_ERR_RENDEZVOUS, "rendezvous: cannot send the table to rank %d", r);
  } else {
    int s = -1;
    for (;;) {
      s = socket(AF_UNIX, SOCK_STREAM | SOCK_CLOEXEC, 0);
      if (s < 0) return fail(TOK_ERR_RENDEZVOUS, "socket(): %s", strerror(errno));
      if (connect(s, reinterpret_cast<struct sockaddr*>(&addr), sizeof(addr)) == 0) break;
      close(s);
      if (now_s() > star.deadline)
        return fail(TOK_ERR_RENDEZVOUS, "rendezvous %s: the group root never appeared (%.0f s)",
                    star.path.c_str(), c->tun.rdzv_timeout_s);
      usleep(20000);
    }
    star.conn.assign(1, s);
    if (send_msg(s, &me, sizeof(me), &my_fd.fd, 1, star.deadline) != 0)
      return fail(TOK_ERR_RENDEZVOUS, "rendezvous: cannot send hello");
    if (recv_msg(s, table.data(), sizeof(Hello) * c->world, &fds, star.deadline) != 0 ||
        static_cast<int>(fds.size()) != c->world)
      return fail(TOK_ERR_RENDEZVOUS,
                  "rendezvous %s: no membership table from the root (it rejected this replica or "
                  "timed out)",
                  star.path.c_str());
  }
  return TOK_OK;
}

// Step 2: the peer table of the new membership.  Mappings of surviving peers are reused (in-place
// re-form), new peers' heaps are imported from their fds, dropped peers' heaps are released.
int rebuild_peers(tok_comm* c, Star& star, const std::vector<Hello>& table, std::vector<Fd> fds) {
  Drv& d = drv();
  c->membership_dirty = true;
  std::vector<PeerMap> next;
  int rc = TOK_OK;
  for (int r = 0; r < c->world && rc == TOK_OK; ++r) {
    if (table[r].uid == c->uid) continue;
    auto it = std::find_if(c->cache.begin(), c->cache.end(),
                           [&](const PeerMap& m) { return m.uid == table[r].uid && m.va != 0; });
    if (it != c->cache.end()) {
      next.push_back(*it);
      *it = PeerMap();  // moved
      continue;
    }
    PeerMap m;
    m.uid = table[r].uid;
    CUresult cr = d.cuMemImportFromShareableHandle_(
        &m.handle, reinterpret_cast<void*>(static_cast<uintptr_t>(fds[r].fd)),
        CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
    if (cr != CUDA_SUCCESS) {
      rc = fail(TOK_ERR_CUDA, "cuMemImportFromShareableHandle(rank %d) failed: %s", r, cu_err(cr));
      break;
    }
    rc = map_heap(c, m.handle, &m.va);
    if (rc != TOK_OK) {
      d.cuMemRelease_(m.handle);
      break;
    }
    next.push_back(m);
  }
  // whatever is left in the old cache belongs to replicas that were dropped
  for (PeerMap& m : c->cache) release_peer(c, m);
  c->cache.swap(next);
  int all = 0;
  int brc = c->world > 1 ? star.all_ok(rc == TOK_OK, &all) : (all = (rc == TOK_OK), TOK_OK);
  if (rc != TOK_OK) return rc;
  if (brc != TOK_OK) return brc;
  if (!all) return fail(TOK_ERR_RENDEZVOUS, "a peer failed to map the group's heaps");
  for (int r = 0; r < kMaxWorld; ++r) c->peer[r] = reinterpret_cast<char*>(c->local_va);
  for (const PeerMap& m : c->cache)
    for (int r = 0; r < c->world; ++r)
      if (table[r].uid == m.uid) c->peer[r] = reinterpret_cast<char*>(m.va);
  return TOK_OK;
}

// Step 3: binds every member's heap to one NVSwitch multicast object (NVLS) in three agreement
// rounds: every GPU added, every heap bound, every member mapped.  NVLS is optional: unless a
// socket is lost, a failure leaves the group on the P2P algorithms.
int bind_multicast(tok_comm* c, Star& star, const std::vector<Hello>& table) {
  Drv& d = drv();
  teardown_multicast(c);
  bool mc_possible = c->world > 1;
  for (int r = 0; r < c->world; ++r) {
    if (!table[r].mc_supported) mc_possible = false;
    for (int q = 0; q < r; ++q)
      if (strncmp(table[r].bus_id, table[q].bus_id, sizeof(table[r].bus_id)) == 0)
        mc_possible = false;  // two replicas share a GPU (single-GPU test mode)
  }
  if (!mc_possible) return TOK_OK;
  int ok = 1;
  if (star.root) {
    Fd mc_fd;
    CUmulticastObjectProp mp;
    memset(&mp, 0, sizeof(mp));
    mp.numDevices = static_cast<unsigned>(c->world);
    mp.size = c->heap_bytes;
    mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    CUresult cr = d.cuMulticastCreate_(&c->mc_handle, &mp);
    if (cr == CUDA_SUCCESS)
      cr = d.cuMemExportToShareableHandle_(&mc_fd.fd, c->mc_handle,
                                           CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0);
    if (cr != CUDA_SUCCESS) {
      set_error("multicast create/export failed: %s", cu_err(cr));
      ok = 0;
    }
    for (int r = 1; r < c->world; ++r) {
      int32_t hdr = ok;
      if (send_msg(star.conn[r], &hdr, sizeof(hdr), ok ? &mc_fd.fd : nullptr, ok ? 1 : 0,
                   star.deadline) != 0)
        return fail(TOK_ERR_RENDEZVOUS, "rendezvous: cannot send the multicast handle");
    }
  } else {
    int32_t hdr = 0;
    std::vector<Fd> got;
    if (recv_msg(star.conn[0], &hdr, sizeof(hdr), &got, star.deadline) != 0)
      return fail(TOK_ERR_RENDEZVOUS, "rendezvous: no multicast handle from the root");
    ok = hdr && got.size() == 1;
    if (ok) {
      CUresult cr = d.cuMemImportFromShareableHandle_(
          &c->mc_handle, reinterpret_cast<void*>(static_cast<uintptr_t>(got[0].fd)),
          CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
      if (cr != CUDA_SUCCESS) {
        set_error("multicast import failed: %s", cu_err(cr));
        c->mc_handle = 0;
        ok = 0;
      }
    }
  }
  if (ok && d.cuMulticastAddDevice_(c->mc_handle, c->cu_dev) != CUDA_SUCCESS) ok = 0;
  int all_added = 0;
  int rc = star.all_ok(ok, &all_added);
  if (rc != TOK_OK) return rc;
  int bound = 0;
  if (all_added) {
    CUresult cr = d.cuMulticastBindMem_(c->mc_handle, 0, c->local_handle, 0, c->heap_bytes, 0);
    if (cr == CUDA_SUCCESS) {
      c->mc_bound = true;
      bound = 1;
    } else {
      set_error("cuMulticastBindMem failed: %s", cu_err(cr));
    }
  }
  int all_bound = 0;
  rc = star.all_ok(bound, &all_bound);
  if (rc != TOK_OK) return rc;
  const int mapped = all_bound && map_heap(c, c->mc_handle, &c->mc_va) == TOK_OK;
  int all_mapped = 0;
  rc = star.all_ok(mapped, &all_mapped);
  if (rc != TOK_OK) return rc;
  if (!all_mapped) teardown_multicast(c);  // NVLS is optional: fall back to P2P algorithms
  return TOK_OK;
}

// Step 4: fresh barrier state for the new group, then every member checks every peer mapping.
int reset_barrier(tok_comm* c, Star& star, const std::vector<Hello>& table) {
  RT_CHECK(cudaMemset(reinterpret_cast<void*>(c->local_va), 0, kFlagBytes));
  RT_CHECK(cudaMemset(c->ctr, 0, kCtrWords * sizeof(uint32_t)));
  RT_CHECK(cudaDeviceSynchronize());
  c->hostctl[kCtlAbort] = 0;
  c->hostctl[kCtlStatus] = 0;
  c->hostctl[kCtlWhere] = 0;
  // identity token at the end of the control page: after the host barrier every replica reads every
  // peer's token THROUGH ITS PEER MAPPING and compares it with the uid the membership table lists for
  // that rank — a wrong or stale mapping fails here, loudly, instead of as a silent hang later
  RT_CHECK(cudaMemcpy(reinterpret_cast<char*>(c->local_va) + kTokenOff, &c->uid, sizeof(c->uid),
                      cudaMemcpyHostToDevice));
  RT_CHECK(cudaDeviceSynchronize());
  if (c->world == 1) return TOK_OK;
  int all_reset = 0;
  int rc = star.all_ok(1, &all_reset);
  if (rc != TOK_OK) return rc;
  int good = 1;
  for (int r = 0; r < c->world; ++r) {
    uint64_t seen = 0;
    if (cudaMemcpy(&seen, c->peer[r] + kTokenOff, sizeof(seen), cudaMemcpyDeviceToHost) != cudaSuccess ||
        seen != table[r].uid) {
      set_error("peer mapping check failed: rank %d's heap as mapped by rank %d carries token %llx, "
                "the membership table says %llx",
                r, c->rank, (unsigned long long)seen, (unsigned long long)table[r].uid);
      cudaGetLastError();
      good = 0;
    }
  }
  int all_good = 0;
  rc = star.all_ok(good, &all_good);
  if (rc != TOK_OK) return rc;
  if (!good) return TOK_ERR_STATE;
  if (!all_good) return fail(TOK_ERR_STATE, "a peer's mapping check failed");
  return TOK_OK;
}

// One membership exchange.  Every replica of the group runs the same steps in the same order, so
// the socket messages and agreement rounds of each step meet their counterparts on the peers.
// membership_dirty tells tok_comm_reform whether the old peer table survived a failure.
int exchange(tok_comm* c) {
  c->membership_dirty = false;
  Star star;
  std::vector<Hello> table(c->world);
  std::vector<Fd> fds;
  int rc = rendezvous(c, star, table, fds);
  if (rc == TOK_OK) rc = rebuild_peers(c, star, table, std::move(fds));
  if (rc == TOK_OK) rc = bind_multicast(c, star, table);
  if (rc == TOK_OK) rc = reset_barrier(c, star, table);
  return rc;
}

Tunables read_tunables() {
  Tunables t;
  t.zero_copy = env_size("TOK_DISABLE_ZERO_COPY", 0) == 0;
  t.max_ctas = static_cast<int>(std::clamp<size_t>(env_size("TOK_MAX_CTAS", 64), 1, kMaxCtas));
  t.zc_ctas = static_cast<int>(std::min<size_t>(env_size("TOK_ZC_CTAS", getenv("TOK_MAX_CTAS") ? t.max_ctas : 0), kMaxCtas));
  t.cta_bytes = std::max<size_t>(env_size("TOK_CTA_BYTES", 65536), 4096);
  if (getenv("TOK_ONE_SHOT_MAX")) t.one_shot_max = env_size("TOK_ONE_SHOT_MAX", 256 << 10);
  t.nvls_min = env_size("TOK_NVLS_MIN", 0);
  t.force_algo = static_cast<int>(env_size("TOK_ALGO", 0));
  t.disable_nvls = env_size("TOK_DISABLE_NVLS", 0) != 0;
  // NCCL's watchdog default is 600 s; replicas legitimately skew by tens of seconds (first-iteration
  // cuDNN autotune, evaluation or a checkpoint on rank 0)
  t.barrier_timeout_ns = env_size("TOK_BARRIER_TIMEOUT_MS", 600000) * 1000000ull;
  t.nvls_unroll = env_size("TOK_NVLS_UNROLL", 8) == 16 ? 16 : 8;
  t.rdzv_timeout_s = static_cast<double>(env_size("TOK_RDZV_TIMEOUT_S", 120));
  return t;
}

int create_impl(const char* job_id, int rank, int world, int max_world, int device_ordinal,
                const char* rendezvous_path, uint64_t epoch, tok_comm_t** out) {
  if (!out) return fail(TOK_ERR_INVALID, "comm out pointer is null");
  *out = nullptr;
  if (!job_id || !rendezvous_path) return fail(TOK_ERR_INVALID, "job_id / rendezvous_path is null");
  if (world < 1 || world > kMaxWorld || rank < 0 || rank >= world)
    return fail(TOK_ERR_INVALID, "invalid rank %d / world %d (1..%d)", rank, world, kMaxWorld);
  if (max_world < world) max_world = world;
  if (max_world > kMaxWorld)
    return fail(TOK_ERR_INVALID, "max_world %d exceeds %d", max_world, kMaxWorld);
  Drv& d = drv();
  if (!d.ok)
    return fail(TOK_ERR_NO_DEVICE, "libtok8s data path needs a CUDA GPU (no CPU fallback): %s",
                d.why.c_str());
  int ndev = 0;
  RT_CHECK(cudaGetDeviceCount(&ndev));
  if (device_ordinal < 0 || device_ordinal >= ndev)
    return fail(TOK_ERR_INVALID, "device ordinal %d out of range (0..%d)", device_ordinal, ndev - 1);

  DeviceGuard guard(device_ordinal);
  RT_CHECK(cudaFree(nullptr));  // make sure the primary context exists
  tok_comm* c = new tok_comm();
  c->job_id = job_id;
  c->rdzv_path = rendezvous_path;
  c->rank = rank;
  c->world = world;
  c->max_world = max_world;
  c->device = device_ordinal;
  c->epoch = epoch;
  std::random_device rd;
  c->uid = (static_cast<uint64_t>(rd()) << 32) ^ rd() ^ (static_cast<uint64_t>(getpid()) << 20) ^
           static_cast<uint64_t>(now_s() * 1e6);
  if (c->uid == 0) c->uid = 1;
  c->cap_bytes = round_up(env_size("TOK_STAGING_MB", 128) << 20, 2u << 20);
  c->pool_bytes = round_up(env_size("TOK_SYMM_POOL_MB", 1024) << 20, 2u << 20);
  c->tun = read_tunables();

  int rc = TOK_OK;
  do {
    CUresult cr = d.cuDeviceGet_(&c->cu_dev, device_ordinal);
    if (cr != CUDA_SUCCESS) {
      rc = fail(TOK_ERR_CUDA, "cuDeviceGet failed: %s", cu_err(cr));
      break;
    }
    cudaDeviceGetPCIBusId(c->bus_id, sizeof(c->bus_id), device_ordinal);
    cudaDeviceGetAttribute(&c->sm_count, cudaDevAttrMultiProcessorCount, device_ordinal);
    rc = alloc_local(c);
    if (rc != TOK_OK) break;
    rc = exchange(c);
  } while (0);
  if (rc != TOK_OK) {
    std::string keep = last_error_cstr();
    tok_comm_destroy(c);
    set_error("%s", keep.c_str());
    return rc;
  }
  *out = c;
  return TOK_OK;
}

Group group(const tok_comm* c) { return {c->world, c->mc_va != 0, c->cap_bytes, c->sm_count}; }

// Start of the symmetric pool in this replica's heap: after the control page and both staging buffers.
char* pool_base(const tok_comm* c) {
  return reinterpret_cast<char*>(c->local_va) + kFlagBytes + 2 * c->cap_bytes;
}

bool in_pool(const tok_comm* c, const void* p, size_t bytes) {
  const char* q = static_cast<const char*>(p);
  return q >= pool_base(c) && q + bytes <= pool_base(c) + c->pool_bytes;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
extern "C" {

const char* tok_last_error(void) { return tok::last_error_cstr(); }

const char* tok_version(void) { return "libtok8s 0.2 (sm_90a, abi 2)"; }

void tok_free(void* p) { free(p); }

int tok_comm_create(const char* job_id, int rank, int world, int max_world, int device_ordinal,
                    const char* rendezvous_path, tok_comm_t** comm) {
  return create_impl(job_id, rank, world, max_world, device_ordinal, rendezvous_path, 0, comm);
}

int tok_comm_join(const char* job_id, int rank, int world, int max_world, int device_ordinal,
                  const char* rendezvous_path, uint64_t epoch, tok_comm_t** comm) {
  return create_impl(job_id, rank, world, max_world, device_ordinal, rendezvous_path, epoch, comm);
}

int tok_comm_reform(tok_comm_t* c, int new_world, int new_rank, uint64_t member_mask,
                    uint64_t epoch) {
  if (!c) return fail(TOK_ERR_INVALID, "comm is null");
  if (new_world < 1 || new_world > c->max_world || new_rank < 0 || new_rank >= new_world)
    return fail(TOK_ERR_INVALID, "invalid new rank %d / world %d (max_world %d)", new_rank,
                new_world, c->max_world);
  if (epoch <= c->epoch)
    return fail(TOK_ERR_STATE, "epoch must grow: have %llu, got %llu",
                (unsigned long long)c->epoch, (unsigned long long)epoch);
  if (!(member_mask & (1ull << c->rank)))
    return fail(TOK_ERR_INVALID,
                "member_mask 0x%llx drops this replica (old rank %d): destroy it instead",
                (unsigned long long)member_mask, c->rank);
  DeviceGuard guard(c->device);
  RT_CHECK(cudaDeviceSynchronize());  // no collective of the old group may still be in flight
  const int old_rank = c->rank, old_world = c->world;
  const uint64_t old_epoch = c->epoch;
  c->rank = new_rank;
  c->world = new_world;
  c->epoch = epoch;
  const int rc = exchange(c);
  if (rc == TOK_ERR_RENDEZVOUS && !c->membership_dirty) {
    // The membership exchange never completed (peers that were announced did not show up): nothing
    // of the old group was unmapped yet, so the communicator stays usable with its previous
    // membership and a later epoch (e.g. the controller's revert) can still be applied.
    c->rank = old_rank;
    c->world = old_world;
    c->epoch = old_epoch;
  }
  return rc;
}

int tok_comm_abort(tok_comm_t* c) {
  if (!c || !c->hostctl) return fail(TOK_ERR_INVALID, "comm is null");
  c->hostctl[kCtlAbort] = 1;
  return TOK_OK;
}

int tok_comm_status(tok_comm_t* c) {
  if (!c || !c->hostctl) return fail(TOK_ERR_INVALID, "comm is null");
  const uint32_t s = c->hostctl[kCtlStatus];
  if (s == 1) {
    const uint32_t where = c->hostctl[kCtlWhere];
    return fail(TOK_ERR_TIMEOUT,
                "a peer replica never reached the in-kernel barrier within %llu ms (rank %d of %d; "
                "given up in %s, CTA %u, ranks still behind: mask 0x%x, waited for value %u)",
                c->tun.barrier_timeout_ns / 1000000ull, c->rank, c->world,
                (where & 0xff) == 1 ? "the bucket arrival" : (where & 0xff) == 2 ? "a CTA barrier" : "?",
                where >> 8, c->hostctl[kCtlBehind], c->hostctl[kCtlWant]);
  }
  if (s == 2) return fail(TOK_ERR_ABORTED, "collective aborted by tok_comm_abort()");
  if (s == 3)
    return fail(TOK_ERR_STATE,
                "zero-copy bucket is not at the same symmetric-pool offset on every replica (the "
                "replicas' pool allocation sequences differ); set TOK_DISABLE_ZERO_COPY=1");
  return TOK_OK;
}

int tok_comm_destroy(tok_comm_t* c) {
  if (!c) return TOK_OK;
  {
    tok_comm* expect = c;
    g_pool_comm.compare_exchange_strong(expect, nullptr);
  }
  if (drv().ok) {
    DeviceGuard guard(c->device);
    cudaDeviceSynchronize();
    teardown_multicast(c);
    for (PeerMap& m : c->cache) release_peer(c, m);
    c->cache.clear();
    unmap(c, &c->local_va);
    if (c->local_handle) drv().cuMemRelease_(c->local_handle);
    if (c->ctr) cudaFree(c->ctr);
    if (c->dbg) cudaFree(c->dbg);
    if (c->hostctl) cudaFreeHost(const_cast<uint32_t*>(c->hostctl));
    cudaGetLastError();
  }
  delete c;
  return TOK_OK;
}

int tok_comm_caps(tok_comm_t* c, tok_caps_t* caps) {
  if (!c || !caps) return fail(TOK_ERR_INVALID, "comm / caps is null");
  memset(caps, 0, sizeof(*caps));
  caps->abi_version = TOK_ABI_VERSION;
  caps->rank = c->rank;
  caps->world = c->world;
  caps->max_world = c->max_world;
  caps->device = c->device;
  caps->multicast = c->mc_va ? 1 : 0;
  caps->p2p = 1;
  caps->epoch = c->epoch;
  caps->staging_bytes = c->cap_bytes;
  caps->heap_bytes = c->heap_bytes;
  caps->one_shot_max = one_shot_limit(group(c), c->tun);
  caps->nvls_min = c->tun.nvls_min;
  caps->max_ctas = c->tun.max_ctas;
  caps->sm_count = c->sm_count;
  return TOK_OK;
}

int tok_allreduce_algo(tok_comm_t* c, size_t wire_bytes, int* algo) {
  if (!c || !algo) return fail(TOK_ERR_INVALID, "comm / algo is null");
  *algo = pick_algo(group(c), c->tun, wire_bytes);
  return TOK_OK;
}

// ---- symmetric pool ---------------------------------------------------------------------------
// First-fit over the released segments (lowest offset first), else bump.  Deterministic: replicas
// that perform the same allocate/release sequence get the same offsets — which is all the zero-copy
// path needs, and the arrive kernel verifies it for every bucket.
int tok_comm_symm_alloc(tok_comm_t* c, size_t bytes, void** ptr) {
  if (!c || !ptr) return fail(TOK_ERR_INVALID, "comm / ptr is null");
  const size_t need = round_up(std::max<size_t>(bytes, 1), 2u << 20);  // segment-friendly alignment
  std::lock_guard<std::mutex> lock(c->pool_mu);
  char* base = pool_base(c);
  for (size_t i = 0; i < c->pool_free.size(); ++i) {
    auto& blk = c->pool_free[i];
    if (blk.second < need) continue;
    *ptr = base + blk.first;
    if (blk.second == need) {
      c->pool_free.erase(c->pool_free.begin() + static_cast<long>(i));
    } else {
      blk.first += need;
      blk.second -= need;
    }
    return TOK_OK;
  }
  if (c->pool_used + need > c->pool_bytes)
    return fail(TOK_ERR_INVALID,
                "symmetric pool exhausted: %zu MiB used + %zu MiB requested > %zu MiB (TOK_SYMM_POOL_MB)",
                c->pool_used >> 20, need >> 20, c->pool_bytes >> 20);
  *ptr = base + c->pool_used;
  c->pool_used += need;
  return TOK_OK;
}

int tok_comm_symm_free(tok_comm_t* c, void* ptr, size_t bytes) {
  if (!c) return fail(TOK_ERR_INVALID, "comm is null");
  if (!ptr) return TOK_OK;
  const size_t size = round_up(std::max<size_t>(bytes, 1), 2u << 20);
  std::lock_guard<std::mutex> lock(c->pool_mu);
  const char* base = pool_base(c);
  const char* p = static_cast<const char*>(ptr);
  if (p < base || p + size > base + c->pool_used || ((p - base) & ((2u << 20) - 1)))
    return fail(TOK_ERR_INVALID, "pointer %p (+%zu) is not a live symmetric-pool segment", ptr, size);
  const size_t off = static_cast<size_t>(p - base);
  auto it = std::lower_bound(c->pool_free.begin(), c->pool_free.end(), std::make_pair(off, size_t{0}));
  if ((it != c->pool_free.end() && it->first < off + size) ||
      (it != c->pool_free.begin() && (it - 1)->first + (it - 1)->second > off))
    return fail(TOK_ERR_STATE, "symmetric-pool segment at offset %zu released twice", off);
  it = c->pool_free.insert(it, std::make_pair(off, size));
  if (it + 1 != c->pool_free.end() && it->first + it->second == (it + 1)->first) {  // merge right
    it->second += (it + 1)->second;
    c->pool_free.erase(it + 1);
  }
  if (it != c->pool_free.begin() && (it - 1)->first + (it - 1)->second == it->first) {  // merge left
    (it - 1)->second += it->second;
    it = c->pool_free.erase(it) - 1;
  }
  if (it->first + it->second == c->pool_used) {  // the top of the pool shrinks back
    c->pool_used = it->first;
    c->pool_free.erase(it);
  }
  return TOK_OK;
}

int tok_comm_symm_info(tok_comm_t* c, void** base, size_t* bytes, size_t* used) {
  if (!c) return fail(TOK_ERR_INVALID, "comm is null");
  if (base) *base = pool_base(c);
  if (bytes) *bytes = c->pool_bytes;
  if (used) {
    std::lock_guard<std::mutex> lock(c->pool_mu);
    size_t freed = 0;
    for (auto& b : c->pool_free) freed += b.second;
    *used = c->pool_used - freed;
  }
  return TOK_OK;
}

int tok_comm_use_as_pool(tok_comm_t* c) {
  g_pool_comm.store(c);
  return TOK_OK;
}

// torch.cuda.memory.CUDAPluggableAllocator entry points: segments of a torch.cuda.MemPool are carved
// from the symmetric pool of the communicator selected with tok_comm_use_as_pool() and go back to
// its free list when torch releases them (DDP drops its first-generation buckets after iteration 1).
void* tok_pool_malloc(ptrdiff_t size, int device, void* stream) {
  (void)stream;
  tok_comm* c = g_pool_comm.load();
  if (!c || size <= 0 || device != c->device) return nullptr;
  void* p = nullptr;
  if (tok_comm_symm_alloc(c, static_cast<size_t>(size), &p) != TOK_OK) return nullptr;
  return p;
}

void tok_pool_free(void* ptr, size_t size, int device, void* stream) {
  (void)stream;
  tok_comm* c = g_pool_comm.load();
  if (!c || device != c->device) return;  // communicator already gone: the heap went with it
  tok_comm_symm_free(c, ptr, size);
}

int tok_comm_debug_read(tok_comm_t* c, uint64_t* out, size_t words) {
  if (!c || !out) return fail(TOK_ERR_INVALID, "comm / out is null");
  if (!c->dbg) return fail(TOK_ERR_STATE, "phase timestamps are off (set TOK_DEBUG_PHASES=1 before tok_comm_create)");
  const size_t n = std::min<size_t>(words, kMaxCtas * 8);
  DeviceGuard guard(c->device);
  RT_CHECK(cudaMemcpy(out, c->dbg, n * sizeof(uint64_t), cudaMemcpyDeviceToHost));
  return TOK_OK;
}

int tok_comm_launches(tok_comm_t* c, uint64_t* launches) {
  if (!c || !launches) return fail(TOK_ERR_INVALID, "comm / launches is null");
  *launches = c->launches.load() + c->arrivals.load();
  return TOK_OK;
}

int tok_comm_stats(tok_comm_t* c, tok_stats_t* st) {
  if (!c || !st) return fail(TOK_ERR_INVALID, "comm / stats is null");
  memset(st, 0, sizeof(*st));
  st->launches = c->launches.load();
  st->arrivals = c->arrivals.load();
  st->elided = c->elided.load();
  st->broadcasts = c->broadcasts.load();
  st->last_algo = c->last_algo.load();
  st->last_ctas = c->last_ctas.load();
  return TOK_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------
// executing plan.cpp's plans
// ------------------------------------------------------------------------------------------------
namespace {

void fill_common(const tok_comm* c, KArgs* a) {
  memset(a, 0, sizeof(*a));
  a->stage_off[0] = kFlagBytes;
  a->stage_off[1] = kFlagBytes + c->cap_bytes;
  a->slot_bytes = c->cap_bytes / kMaxWorld;
  for (int r = 0; r < kMaxWorld; ++r) a->peer[r] = c->peer[r];
  a->mc = reinterpret_cast<char*>(c->mc_va);
  a->ctr = c->ctr;
  a->hostctl = c->hostctl_dev;
  a->timeout_ns = c->tun.barrier_timeout_ns;
  a->dbg = c->dbg;
  a->rank = c->rank;
  a->world = c->world;
  a->unroll = c->tun.nvls_unroll;
}

size_t heap_off(const tok_comm* c, const void* p) {
  return static_cast<size_t>(static_cast<const char*>(p) - reinterpret_cast<const char*>(c->local_va));
}

// Checks a bucket call's arguments and the group's health, then plans the bucket.
int plan_bucket(tok_comm* c, const void* in, const void* out, size_t count, int in_dtype,
                int wire_dtype, int out_dtype, float scale, unsigned flags, Bucket* b,
                AllreducePlan* pl) {
  if (!c) return fail(TOK_ERR_INVALID, "comm is null");
  auto bad_dt = [](int d) { return d != TOK_F32 && d != TOK_BF16 && d != TOK_F16; };
  if (bad_dt(in_dtype) || bad_dt(wire_dtype) || bad_dt(out_dtype))
    return fail(TOK_ERR_INVALID, "unsupported dtype (in %d wire %d out %d)", in_dtype, wire_dtype,
                out_dtype);
  if (!in || !out) return fail(TOK_ERR_INVALID, "in / out is null");
  if ((reinterpret_cast<uintptr_t>(in) & 15) || (reinterpret_cast<uintptr_t>(out) & 15))
    return fail(TOK_ERR_ALIGN, "bucket pointers must be 16-byte aligned (in %p out %p)", in, out);
  const int st = tok_comm_status(c);
  if (st != TOK_OK) return st;
  *b = {count, in_dtype, wire_dtype, out_dtype, scale, flags, in == out,
        in_pool(c, in, count * dtype_size(in_dtype))};
  return plan_allreduce(group(c), c->tun, *b, pl);
}

int launch_error(const char* what, int e) {
  return fail(TOK_ERR_CUDA, "%s launch failed: %s", what,
              cudaGetErrorString(static_cast<cudaError_t>(e)));
}

int do_arrive(tok_comm* c, size_t buf_off, void* stream) {
  KArgs a;
  fill_common(c, &a);
  a.buf_off = buf_off;
  int e = launch_arrive(a, stream);
  if (e != 0) return launch_error("arrive kernel", e);
  c->arrivals.fetch_add(1);
  return TOK_OK;
}

// Takes the result `e` of launching a `what` kernel: counts the launch, or reports its error.
int launched(tok_comm* c, int e, const char* what, int algo, int ctas) {
  if (e != 0) return launch_error(what, e);
  c->launches.fetch_add(1);
  c->last_algo.store(algo);
  c->last_ctas.store(ctas);
  return TOK_OK;
}

}  // namespace

extern "C" {

int tok_bucket_arrive(tok_comm_t* c, const void* bucket, size_t count, int dtype, float scale,
                      unsigned flags, void* cuda_stream, int* arrived) {
  if (arrived) *arrived = 0;
  if (count == 0) return TOK_OK;
  Bucket b;
  AllreducePlan pl;
  int st = plan_bucket(c, bucket, bucket, count, dtype, dtype, dtype, scale, flags, &b, &pl);
  if (st != TOK_OK) return st;
  if (!pl.inplace) return TOK_OK;  // staged kernels carry their own barriers
  DeviceGuard guard(c->device);
  st = do_arrive(c, heap_off(c, bucket), cuda_stream);
  if (st == TOK_OK && arrived) *arrived = 1;
  return st;
}

int tok_allreduce_bucket(tok_comm_t* c, const void* in, void* out, size_t count, int in_dtype,
                         int wire_dtype, int out_dtype, float scale, unsigned flags,
                         void* cuda_stream) {
  if (c && count == 0) return TOK_OK;
  Bucket b;
  AllreducePlan pl;
  int st = plan_bucket(c, in, out, count, in_dtype, wire_dtype, out_dtype, scale, flags, &b, &pl);
  if (st != TOK_OK) return st;
  if (pl.elide) {
    c->elided.fetch_add(1);
    return TOK_OK;
  }
  const size_t isz = dtype_size(in_dtype);
  const size_t osz = dtype_size(out_dtype);
  DeviceGuard guard(c->device);
  if (pl.inplace && !(flags & TOK_FLAG_ARRIVED)) {
    st = do_arrive(c, heap_off(c, in), cuda_stream);
    if (st != TOK_OK) return st;
  }
  KArgs a;
  fill_common(c, &a);
  a.scale = scale;
  a.flags = flags & TOK_FLAG_SCALE_POST;
  for (size_t off = 0; off < count; off += pl.launch_elems) {
    const size_t n = std::min(pl.launch_elems, count - off);
    const Grid grid = allreduce_grid(group(c), c->tun, b, pl, n);
    a.in = static_cast<const char*>(in) + off * isz;
    a.out = static_cast<char*>(out) + off * osz;
    a.count = n;
    a.total_packs = grid.total_packs;
    a.packs_per_cta = grid.packs_per_cta;
    if (pl.inplace) a.buf_off = heap_off(c, in) + off * isz;
    st = launched(c, launch_allreduce(pl.algo, in_dtype, wire_dtype, out_dtype, grid.ctas, a, cuda_stream),
                  "allreduce kernel", pl.algo, grid.ctas);
    if (st != TOK_OK) return st;
  }
  return TOK_OK;
}

int tok_comm_debug_peek(tok_comm_t* c, int rank, size_t byte_off, uint32_t* out, size_t words) {
  if (!c || !out) return fail(TOK_ERR_INVALID, "comm / out is null");
  if (rank < 0 || rank >= c->world || byte_off + words * 4 > kFlagBytes)
    return fail(TOK_ERR_INVALID, "rank / offset out of range");
  DeviceGuard guard(c->device);
  RT_CHECK(cudaMemcpy(out, c->peer[rank] + byte_off, words * 4, cudaMemcpyDeviceToHost));
  return TOK_OK;
}

int tok_comm_debug_barrier(tok_comm_t* c, int variant, int ctas, size_t count, void* cuda_stream) {
  if (!c) return fail(TOK_ERR_INVALID, "comm is null");
  if (variant < 0 || variant > 4 || ctas < 1 || ctas > 64)
    return fail(TOK_ERR_INVALID, "variant 0..4, ctas 1..64");
  if (c->world < 2) return fail(TOK_ERR_STATE, "a barrier needs world >= 2");
  int st = tok_comm_status(c);
  if (st != TOK_OK) return st;
  DeviceGuard guard(c->device);
  KArgs a;
  fill_common(c, &a);
  a.count = count;
  a.flags = static_cast<uint32_t>(variant);
  int e = launch_barrier_bench(ctas, a, cuda_stream);
  return e != 0 ? launch_error("barrier bench", e) : TOK_OK;
}

int tok_broadcast(tok_comm_t* c, void* buf, size_t bytes, int root, void* cuda_stream) {
  if (!c) return fail(TOK_ERR_INVALID, "comm is null");
  if (root < 0 || root >= c->world)
    return fail(TOK_ERR_INVALID, "broadcast root %d out of range (world %d)", root, c->world);
  if (bytes == 0 || c->world == 1) return TOK_OK;
  if (!buf) return fail(TOK_ERR_INVALID, "buf is null");
  if (reinterpret_cast<uintptr_t>(buf) & 15)
    return fail(TOK_ERR_ALIGN, "broadcast buffer must be 16-byte aligned (%p)", buf);
  int st = tok_comm_status(c);
  if (st != TOK_OK) return st;
  DeviceGuard guard(c->device);
  const BroadcastPlan bp = plan_broadcast(group(c), c->tun, bytes, in_pool(c, buf, bytes));
  KArgs a;
  fill_common(c, &a);
  a.root = root;
  if (bp.mode != kBcastStaged) {  // peers read the bucket where it lies: they wait for its arrival
    a.buf_off = heap_off(c, buf);
    st = do_arrive(c, a.buf_off, cuda_stream);
    if (st != TOK_OK) return st;
  }
  for (size_t off = 0; off < bytes; off += bp.launch_bytes) {
    const size_t n = std::min(bp.launch_bytes, bytes - off);
    const Grid grid = broadcast_grid(c->tun, n);
    a.in = a.out = static_cast<char*>(buf) + off;
    a.count = n;
    a.packs_per_cta = grid.packs_per_cta;
    st = launched(c, launch_broadcast(bp.mode, grid.ctas, a, cuda_stream), "broadcast kernel",
                  bp.mode, grid.ctas);
    if (st != TOK_OK) return st;
  }
  c->broadcasts.fetch_add(1);
  return TOK_OK;
}

}  // extern "C"
