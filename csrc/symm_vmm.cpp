// Symmetric memory v2: CUDA virtual-memory-management allocations shared between the ranks of a process group through
// POSIX file descriptors (passed over an abstract unix datagram socket with SCM_RIGHTS), every peer's allocation mapped
// into this process's address space, and — when the devices sit behind an NVSwitch that supports it — an NVLS *multicast
// object* bound to all of them: one `multimem.st` to the multicast address lands in every rank's buffer, one
// `multimem.ld_reduce` returns the in-switch sum of every rank's copy (fp32 accumulation).  This is what the NVLS
// variants of the fused tensor-parallel kernels (csrc/gemm_sm90.cu MODE 5 / 6) dereference.
//
// The exchange is driven from python in phases (ops/symm.py::get_vmm_workspace) because the rendezvous between the ranks
// (names, barriers, "did multicast work for everybody") travels over the process group's host control plane:
//   vmm_begin        allocate + map the local buffer, open the datagram socket            → (id, socket name, mc supported)
//   vmm_send         export the local handle (rank 0: also create + export the multicast object) to every peer
//   vmm_recv         import + map every peer's handle; import the multicast object and add this device
//   [barrier]        cuMulticastBindMem blocks until every device was added — python barriers in between
//   vmm_bind         bind the local memory, map the multicast VA                          → ok / error string
//   vmm_ptrs         unicast pointer table + multicast base (0 if unavailable)
// Driver entry points are resolved with cudaGetDriverEntryPoint so the extension does not link libcuda (the build box
// has no driver).  No reference counterpart: the reference's collectives are XLA ops (SURVEY §5.8).
#include <cuda.h>
#include <cuda_runtime.h>
#include <errno.h>
#include <poll.h>
#include <sys/socket.h>
#include <sys/un.h>
#include <unistd.h>

#include <cstring>
#include <map>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include "symm.h"

namespace nxd {
namespace {

struct Drv {
  CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long);
  CUresult (*MemRelease)(CUmemGenericAllocationHandle);
  CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long);
  CUresult (*MemAddressFree)(CUdeviceptr, size_t);
  CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long);
  CUresult (*MemUnmap)(CUdeviceptr, size_t);
  CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t);
  CUresult (*MemGetAllocationGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags);
  CUresult (*MemExportToShareableHandle)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long);
  CUresult (*MemImportFromShareableHandle)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType);
  CUresult (*MulticastCreate)(CUmemGenericAllocationHandle*, const CUmulticastObjectProp*);
  CUresult (*MulticastAddDevice)(CUmemGenericAllocationHandle, CUdevice);
  CUresult (*MulticastBindMem)(CUmemGenericAllocationHandle, size_t, CUmemGenericAllocationHandle, size_t, size_t,
                               unsigned long long);
  CUresult (*MulticastGetGranularity)(size_t*, const CUmulticastObjectProp*, CUmulticastGranularity_flags);
  CUresult (*MulticastUnbind)(CUmemGenericAllocationHandle, CUdevice, size_t, size_t);
  CUresult (*DeviceGetAttribute)(int*, CUdevice_attribute, CUdevice);
  CUresult (*DeviceGet)(CUdevice*, int);
  CUresult (*GetErrorString)(CUresult, const char**);
  bool ok = false;
};

template <typename F> void resolve(F& fn, const char* name) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q);
  if (e != cudaSuccess || p == nullptr || q != cudaDriverEntryPointSuccess)
    throw std::runtime_error(std::string("cudaGetDriverEntryPoint(") + name + ") failed");
  fn = reinterpret_cast<F>(p);
}

Drv& drv() {
  static Drv d;
  static std::once_flag once;
  std::call_once(once, [] {
    resolve(d.MemCreate, "cuMemCreate");
    resolve(d.MemRelease, "cuMemRelease");
    resolve(d.MemAddressReserve, "cuMemAddressReserve");
    resolve(d.MemAddressFree, "cuMemAddressFree");
    resolve(d.MemMap, "cuMemMap");
    resolve(d.MemUnmap, "cuMemUnmap");
    resolve(d.MemSetAccess, "cuMemSetAccess");
    resolve(d.MemGetAllocationGranularity, "cuMemGetAllocationGranularity");
    resolve(d.MemExportToShareableHandle, "cuMemExportToShareableHandle");
    resolve(d.MemImportFromShareableHandle, "cuMemImportFromShareableHandle");
    resolve(d.MulticastCreate, "cuMulticastCreate");
    resolve(d.MulticastAddDevice, "cuMulticastAddDevice");
    resolve(d.MulticastBindMem, "cuMulticastBindMem");
    resolve(d.MulticastGetGranularity, "cuMulticastGetGranularity");
    resolve(d.MulticastUnbind, "cuMulticastUnbind");
    resolve(d.DeviceGetAttribute, "cuDeviceGetAttribute");
    resolve(d.DeviceGet, "cuDeviceGet");
    resolve(d.GetErrorString, "cuGetErrorString");
    d.ok = true;
  });
  return d;
}

std::string cu_err(CUresult r) {
  const char* s = nullptr;
  if (drv().GetErrorString(r, &s) != CUDA_SUCCESS || !s) s = "unknown";
  return std::string(s) + " (" + std::to_string((int)r) + ")";
}
#define CU_CHECK(call)                                                                         \
  do {                                                                                         \
    CUresult _r = (call);                                                                      \
    if (_r != CUDA_SUCCESS) throw std::runtime_error(std::string(#call) + ": " + cu_err(_r)); \
  } while (0)

struct VmmRegion {
  int device = 0;
  int rank = 0, world = 1;
  size_t size = 0;                 // mapped size (aligned)
  CUmemGenericAllocationHandle mem = 0;
  CUdeviceptr local_va = 0;
  std::vector<CUmemGenericAllocationHandle> peer_mem;   // imported handles (0 for self)
  std::vector<CUdeviceptr> peer_va;                     // [world]
  bool want_mc = false, mc_added = false, mc_bound = false;
  CUmemGenericAllocationHandle mc = 0;
  CUdeviceptr mc_va = 0;
  int sock = -1;
  std::string sock_name;
};

std::mutex g_mu;
std::map<int64_t, VmmRegion> g_regions;
int64_t g_next = 1 << 20;          // disjoint from the cudaIpc regions of symm.cpp

VmmRegion& region(int64_t id) {
  auto it = g_regions.find(id);
  if (it == g_regions.end()) throw std::runtime_error("symm_vmm: bad handle");
  return it->second;
}

CUmemAllocationProp alloc_prop(int device) {
  CUmemAllocationProp p;
  std::memset(&p, 0, sizeof(p));
  p.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  p.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  p.location.id = device;
  p.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  return p;
}

void set_rw(CUdeviceptr va, size_t size, int device) {
  CUmemAccessDesc a;
  std::memset(&a, 0, sizeof(a));
  a.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  a.location.id = device;
  a.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  CU_CHECK(drv().MemSetAccess(va, size, &a, 1));
}

sockaddr_un abstract_addr(const std::string& name, socklen_t* len) {
  sockaddr_un a;
  std::memset(&a, 0, sizeof(a));
  a.sun_family = AF_UNIX;
  // abstract namespace: sun_path[0] == 0, no filesystem entry to clean up
  std::memcpy(a.sun_path + 1, name.data(), std::min(name.size(), sizeof(a.sun_path) - 2));
  *len = (socklen_t)(offsetof(sockaddr_un, sun_path) + 1 + std::min(name.size(), sizeof(a.sun_path) - 2));
  return a;
}

struct FdMsg { int32_t rank; int32_t kind; };   // kind 0 = memory handle, 1 = multicast object

void send_fd(int sock, const std::string& to, int fd, FdMsg m) {
  socklen_t alen;
  sockaddr_un addr = abstract_addr(to, &alen);
  msghdr msg;
  std::memset(&msg, 0, sizeof(msg));
  iovec io{&m, sizeof(m)};
  alignas(cmsghdr) char ctrl[CMSG_SPACE(sizeof(int))];
  std::memset(ctrl, 0, sizeof(ctrl));
  msg.msg_name = &addr;
  msg.msg_namelen = alen;
  msg.msg_iov = &io;
  msg.msg_iovlen = 1;
  msg.msg_control = ctrl;
  msg.msg_controllen = sizeof(ctrl);
  cmsghdr* c = CMSG_FIRSTHDR(&msg);
  c->cmsg_level = SOL_SOCKET;
  c->cmsg_type = SCM_RIGHTS;
  c->cmsg_len = CMSG_LEN(sizeof(int));
  std::memcpy(CMSG_DATA(c), &fd, sizeof(int));
  for (int attempt = 0; attempt < 2000; ++attempt) {
    if (sendmsg(sock, &msg, 0) >= 0) return;
    if (errno == ECONNREFUSED || errno == ENOENT || errno == EAGAIN || errno == ENOBUFS) { usleep(5000); continue; }
    break;
  }
  throw std::runtime_error(std::string("symm_vmm: sendmsg to ") + to + " failed: " + strerror(errno));
}

int recv_fd(int sock, FdMsg* m, int timeout_ms) {
  pollfd pf{sock, POLLIN, 0};
  int pr = poll(&pf, 1, timeout_ms);
  if (pr <= 0) throw std::runtime_error("symm_vmm: timed out waiting for a peer's memory handle");
  msghdr msg;
  std::memset(&msg, 0, sizeof(msg));
  iovec io{m, sizeof(*m)};
  alignas(cmsghdr) char ctrl[CMSG_SPACE(sizeof(int))];
  msg.msg_iov = &io;
  msg.msg_iovlen = 1;
  msg.msg_control = ctrl;
  msg.msg_controllen = sizeof(ctrl);
  if (recvmsg(sock, &msg, 0) < (ssize_t)sizeof(*m)) throw std::runtime_error(std::string("symm_vmm: recvmsg: ") + strerror(errno));
  cmsghdr* c = CMSG_FIRSTHDR(&msg);
  if (!c || c->cmsg_level != SOL_SOCKET || c->cmsg_type != SCM_RIGHTS) throw std::runtime_error("symm_vmm: message without fd");
  int fd;
  std::memcpy(&fd, CMSG_DATA(c), sizeof(int));
  return fd;
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
VmmBegin vmm_begin(size_t nbytes, int rank, int world, bool want_multicast) {
  Drv& d = drv();
  VmmRegion r;
  r.rank = rank;
  r.world = world;
  if (cudaGetDevice(&r.device) != cudaSuccess) throw std::runtime_error("cudaGetDevice failed");
  cudaFree(0);                                          // make sure the primary context exists
  CUdevice dev;
  CU_CHECK(d.DeviceGet(&dev, r.device));
  int posix_ok = 0, mc_ok = 0;
  CU_CHECK(d.DeviceGetAttribute(&posix_ok, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR_SUPPORTED, dev));
  if (!posix_ok) throw std::runtime_error("symm_vmm: device does not support POSIX-fd shareable handles");
  d.DeviceGetAttribute(&mc_ok, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev);
  const CUmemAllocationProp prop = alloc_prop(r.device);
  size_t gran = 0;
  CU_CHECK(d.MemGetAllocationGranularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
  if (want_multicast && mc_ok && world > 1) {
    CUmulticastObjectProp mp;
    std::memset(&mp, 0, sizeof(mp));
    mp.numDevices = (unsigned)world;
    mp.size = nbytes;
    mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    size_t mg = 0;
    if (d.MulticastGetGranularity(&mg, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED) == CUDA_SUCCESS && mg > gran) gran = mg;
    r.want_mc = true;
  }
  if (gran < (2u << 20)) gran = 2u << 20;
  r.size = (nbytes + gran - 1) / gran * gran;
  CU_CHECK(d.MemCreate(&r.mem, r.size, &prop, 0));
  CU_CHECK(d.MemAddressReserve(&r.local_va, r.size, gran, 0, 0));
  CU_CHECK(d.MemMap(r.local_va, r.size, 0, r.mem, 0));
  set_rw(r.local_va, r.size, r.device);
  if (cudaMemset((void*)r.local_va, 0, r.size) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess)
    throw std::runtime_error("symm_vmm: clearing the new allocation failed");
  r.peer_mem.assign(world, 0);
  r.peer_va.assign(world, 0);
  r.peer_va[rank] = r.local_va;

  r.sock = socket(AF_UNIX, SOCK_DGRAM | SOCK_CLOEXEC, 0);
  if (r.sock < 0) throw std::runtime_error(std::string("symm_vmm: socket: ") + strerror(errno));
  VmmBegin out;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    out.id = g_next++;
  }
  r.sock_name = "nxd_symm_" + std::to_string((long)getpid()) + "_" + std::to_string((long)out.id);
  socklen_t alen;
  sockaddr_un addr = abstract_addr(r.sock_name, &alen);
  if (bind(r.sock, (sockaddr*)&addr, alen) != 0) throw std::runtime_error(std::string("symm_vmm: bind: ") + strerror(errno));
  out.sock_name = r.sock_name;
  out.multicast_supported = r.want_mc;
  out.size = r.size;
  std::lock_guard<std::mutex> lk(g_mu);
  g_regions[out.id] = r;
  return out;
}

// Phase 2: ship this rank's memory handle to every peer; group rank 0 also creates the multicast object and ships it.
std::string vmm_send(int64_t id, const std::vector<std::string>& sock_names, bool use_multicast) {
  Drv& d = drv();
  std::lock_guard<std::mutex> lk(g_mu);
  VmmRegion& r = region(id);
  r.want_mc = r.want_mc && use_multicast;
  int fd = -1;
  CU_CHECK(d.MemExportToShareableHandle(&fd, r.mem, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
  for (int p = 0; p < r.world; ++p)
    if (p != r.rank) send_fd(r.sock, sock_names[p], fd, FdMsg{r.rank, 0});
  close(fd);
  std::string mc_error;
  if (r.want_mc && r.rank == 0) {
    // a failure here must still reach the peers (they are about to wait for the object): send them the memory fd
    // again tagged kind 2 = "no multicast", so every rank falls back together
    CUmulticastObjectProp mp;
    std::memset(&mp, 0, sizeof(mp));
    mp.numDevices = (unsigned)r.world;
    mp.size = r.size;
    mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    CUresult cr = d.MulticastCreate(&r.mc, &mp);
    int mfd = -1;
    if (cr == CUDA_SUCCESS) cr = d.MemExportToShareableHandle(&mfd, r.mc, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0);
    if (cr != CUDA_SUCCESS) {
      mc_error = "cuMulticastCreate/export: " + cu_err(cr);
      r.want_mc = false;
      int fd2 = -1;
      CU_CHECK(d.MemExportToShareableHandle(&fd2, r.mem, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
      for (int p = 1; p < r.world; ++p) send_fd(r.sock, sock_names[p], fd2, FdMsg{0, 2});
      close(fd2);
    } else {
      for (int p = 1; p < r.world; ++p) send_fd(r.sock, sock_names[p], mfd, FdMsg{0, 1});
      close(mfd);
    }
  }
  return mc_error;
}

// Phase 3: import + map the peers; import the multicast object (ranks > 0) and add this device to it.
std::string vmm_recv(int64_t id) {
  Drv& d = drv();
  std::lock_guard<std::mutex> lk(g_mu);
  VmmRegion& r = region(id);
  std::string mc_error;
  int expect = r.world - 1 + ((r.want_mc && r.rank != 0) ? 1 : 0);
  CUdevice dev;
  CU_CHECK(d.DeviceGet(&dev, r.device));
  for (int i = 0; i < expect; ++i) {
    FdMsg m{};
    int fd = recv_fd(r.sock, &m, 120000);
    if (m.kind == 0) {
      if (m.rank < 0 || m.rank >= r.world || m.rank == r.rank || r.peer_mem[m.rank]) { close(fd); throw std::runtime_error("symm_vmm: unexpected handle message"); }
      CUmemGenericAllocationHandle h;
      CU_CHECK(d.MemImportFromShareableHandle(&h, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
      close(fd);
      CUdeviceptr va = 0;
      CU_CHECK(d.MemAddressReserve(&va, r.size, 0, 0, 0));
      CU_CHECK(d.MemMap(va, r.size, 0, h, 0));
      set_rw(va, r.size, r.device);
      r.peer_mem[m.rank] = h;
      r.peer_va[m.rank] = va;
    } else if (m.kind == 1) {
      CUresult cr = d.MemImportFromShareableHandle(&r.mc, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
      close(fd);
      if (cr != CUDA_SUCCESS) { mc_error = "import multicast object: " + cu_err(cr); r.want_mc = false; r.mc = 0; }
    } else {
      close(fd);
      mc_error = "rank 0 could not create the multicast object";
      r.want_mc = false;
    }
  }
  if (r.want_mc && r.mc) {
    CUresult cr = d.MulticastAddDevice(r.mc, dev);
    if (cr != CUDA_SUCCESS) { mc_error = "cuMulticastAddDevice: " + cu_err(cr); r.want_mc = false; }
    else r.mc_added = true;
  }
  return mc_error;
}

// Phase 4 (after a barrier: every device has been added): bind the local memory and map the multicast address range.
std::string vmm_bind(int64_t id, bool everyone_ok) {
  Drv& d = drv();
  std::lock_guard<std::mutex> lk(g_mu);
  VmmRegion& r = region(id);
  if (!(r.want_mc && r.mc_added && everyone_ok)) { r.want_mc = false; return everyone_ok ? "multicast not set up on this rank" : ""; }
  CUresult cr = d.MulticastBindMem(r.mc, 0, r.mem, 0, r.size, 0);
  if (cr != CUDA_SUCCESS) { r.want_mc = false; return "cuMulticastBindMem: " + cu_err(cr); }
  r.mc_bound = true;
  cr = d.MemAddressReserve(&r.mc_va, r.size, 0, 0, 0);
  if (cr == CUDA_SUCCESS) cr = d.MemMap(r.mc_va, r.size, 0, r.mc, 0);
  if (cr != CUDA_SUCCESS) { r.want_mc = false; r.mc_va = 0; return "map multicast VA: " + cu_err(cr); }
  try { set_rw(r.mc_va, r.size, r.device); } catch (const std::exception& e) { r.want_mc = false; r.mc_va = 0; return e.what(); }
  return "";
}

VmmPtrs vmm_ptrs(int64_t id, bool multicast_everywhere) {
  std::lock_guard<std::mutex> lk(g_mu);
  VmmRegion& r = region(id);
  VmmPtrs out;
  for (int p = 0; p < r.world; ++p) out.peer.push_back((int64_t)r.peer_va[p]);
  out.multicast = (r.want_mc && multicast_everywhere) ? (int64_t)r.mc_va : 0;
  out.size = r.size;
  if (r.sock >= 0) { close(r.sock); r.sock = -1; }
  return out;
}

void* vmm_local(int64_t id, size_t* nbytes) {
  std::lock_guard<std::mutex> lk(g_mu);
  VmmRegion& r = region(id);
  if (nbytes) *nbytes = r.size;
  return (void*)r.local_va;
}

void vmm_free(int64_t id) {
  Drv& d = drv();
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_regions.find(id);
  if (it == g_regions.end()) return;
  VmmRegion& r = it->second;
  cudaDeviceSynchronize();
  if (r.mc_va) { d.MemUnmap(r.mc_va, r.size); d.MemAddressFree(r.mc_va, r.size); }
  if (r.mc_bound) { CUdevice dev; if (d.DeviceGet(&dev, r.device) == CUDA_SUCCESS) d.MulticastUnbind(r.mc, dev, 0, r.size); }
  if (r.mc) d.MemRelease(r.mc);
  for (int p = 0; p < r.world; ++p) {
    if (p == r.rank || !r.peer_va[p]) continue;
    d.MemUnmap(r.peer_va[p], r.size);
    d.MemAddressFree(r.peer_va[p], r.size);
    d.MemRelease(r.peer_mem[p]);
  }
  d.MemUnmap(r.local_va, r.size);
  d.MemAddressFree(r.local_va, r.size);
  d.MemRelease(r.mem);
  if (r.sock >= 0) close(r.sock);
  g_regions.erase(it);
}

bool is_vmm_id(int64_t id) { return id >= (1 << 20); }

}  // namespace nxd
