// ddstore_b200/csrc/vmm.cpp -- shard memory that peers can map at full NVLink speed.
//
// The reference exposes a shard with MPI_Win_create (include/ddstore.hpp:56-61). Here the shard is physical
// HBM created with the CUDA virtual-memory-management API (cuMemCreate, 2 MiB granularity), exported as a POSIX
// file descriptor, passed to the other ranks of the box over an abstract AF_UNIX datagram socket (SCM_RIGHTS) and
// mapped there with cuMemImportFromShareableHandle + cuMemMap. Random 4 KiB peer reads through a legacy
// cudaIpcOpenMemHandle mapping were found to be several times slower than the same reads through a same-process
// peer mapping (not re-measured on H100) -- hence VMM, with legacy IPC kept as the fallback.
//
// The driver entry points are resolved at run time with cudaGetDriverEntryPoint, so the library has no link-time
// dependency on libcuda and still loads (and fails loudly in dds_create) on a machine without a GPU.
//
// A HOST-placed shard (dds_add_placed) is pinned host memory instead: a memfd mapped MAP_SHARED and registered with
// cudaHostRegister(Mapped | Portable). It travels to the other processes of the box as a file descriptor over the same
// socket, and needs neither a driver attribute nor /dev/shm.
#include <cuda.h>
#include <cuda_runtime_api.h>
#include <poll.h>
#include <sys/mman.h>
#include <sys/socket.h>
#include <sys/un.h>
#include <unistd.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "ddstore_b200.h"
#include "internal.h"
#include "vmm.h"

namespace {

struct DriverApi {
    CUresult (*MemCreate)(CUmemGenericAllocationHandle *, size_t, const CUmemAllocationProp *, unsigned long long);
    CUresult (*MemRelease)(CUmemGenericAllocationHandle);
    CUresult (*MemAddressReserve)(CUdeviceptr *, size_t, size_t, CUdeviceptr, unsigned long long);
    CUresult (*MemAddressFree)(CUdeviceptr, size_t);
    CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long);
    CUresult (*MemUnmap)(CUdeviceptr, size_t);
    CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc *, size_t);
    CUresult (*MemExportToShareableHandle)(void *, CUmemGenericAllocationHandle, CUmemAllocationHandleType,
                                           unsigned long long);
    CUresult (*MemImportFromShareableHandle)(CUmemGenericAllocationHandle *, void *, CUmemAllocationHandleType);
    CUresult (*MemGetAllocationGranularity)(size_t *, const CUmemAllocationProp *, CUmemAllocationGranularity_flags);
    CUresult (*GetErrorString)(CUresult, const char **);
    CUresult (*DeviceGet)(CUdevice *, int);
    CUresult (*DeviceGetAttribute)(int *, CUdevice_attribute, CUdevice);
    bool ok = false;
};

DriverApi g_drv;
std::once_flag g_drv_once;

template <typename F>
bool resolve(const char *name, F *fn) {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || !p ||
        q != cudaDriverEntryPointSuccess) {
        (void)cudaGetLastError();
        return false;
    }
    *fn = (F)p;
    return true;
}

void load_driver() {
    bool ok = true;
    ok &= resolve("cuMemCreate", &g_drv.MemCreate);
    ok &= resolve("cuMemRelease", &g_drv.MemRelease);
    ok &= resolve("cuMemAddressReserve", &g_drv.MemAddressReserve);
    ok &= resolve("cuMemAddressFree", &g_drv.MemAddressFree);
    ok &= resolve("cuMemMap", &g_drv.MemMap);
    ok &= resolve("cuMemUnmap", &g_drv.MemUnmap);
    ok &= resolve("cuMemSetAccess", &g_drv.MemSetAccess);
    ok &= resolve("cuMemExportToShareableHandle", &g_drv.MemExportToShareableHandle);
    ok &= resolve("cuMemImportFromShareableHandle", &g_drv.MemImportFromShareableHandle);
    ok &= resolve("cuMemGetAllocationGranularity", &g_drv.MemGetAllocationGranularity);
    ok &= resolve("cuGetErrorString", &g_drv.GetErrorString);
    ok &= resolve("cuDeviceGet", &g_drv.DeviceGet);
    ok &= resolve("cuDeviceGetAttribute", &g_drv.DeviceGetAttribute);
    g_drv.ok = ok;
}

int drv_fail(CUresult r, const char *what) {
    const char *s = nullptr;
    if (g_drv.GetErrorString) g_drv.GetErrorString(r, &s);
    char buf[256];
    snprintf(buf, sizeof(buf), "%s: %s", what, s ? s : "unknown driver error");
    return dds_internal::fail(DDS_ERR_CUDA, buf);
}
#define DRV(expr)                                         \
    do {                                                  \
        CUresult r__ = (expr);                            \
        if (r__ != CUDA_SUCCESS) return drv_fail(r__, #expr); \
    } while (0)

CUmemAllocationProp make_prop(int device) {
    CUmemAllocationProp prop;
    memset(&prop, 0, sizeof(prop));
    prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    prop.location.id = device;
    prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    return prop;
}

int set_access(CUdeviceptr p, size_t size, int device) {
    CUmemAccessDesc acc;
    memset(&acc, 0, sizeof(acc));
    acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    acc.location.id = device;
    acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    DRV(g_drv.MemSetAccess(p, size, &acc, 1));
    return DDS_OK;
}

sockaddr_un abstract_addr(const std::string &name, socklen_t *len) {
    sockaddr_un a;
    memset(&a, 0, sizeof(a));
    a.sun_family = AF_UNIX;
    size_t n = name.size() < sizeof(a.sun_path) - 2 ? name.size() : sizeof(a.sun_path) - 2;
    memcpy(a.sun_path + 1, name.data(), n); // leading NUL: abstract namespace, nothing to unlink
    *len = (socklen_t)(offsetof(sockaddr_un, sun_path) + 1 + n);
    return a;
}

} // namespace

namespace dds_vmm {

bool available(int device) {
    if (const char *e = getenv("DDS_SHARD_ALLOC"))
        if (!strcmp(e, "legacy")) return false;
    std::call_once(g_drv_once, load_driver);
    if (!g_drv.ok) return false;
    CUdevice dev;
    int vmm = 0, fd = 0;
    if (g_drv.DeviceGet(&dev, device) != CUDA_SUCCESS) return false;
    if (g_drv.DeviceGetAttribute(&vmm, CU_DEVICE_ATTRIBUTE_VIRTUAL_MEMORY_MANAGEMENT_SUPPORTED, dev) != CUDA_SUCCESS) vmm = 0;
    if (g_drv.DeviceGetAttribute(&fd, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR_SUPPORTED, dev) != CUDA_SUCCESS)
        fd = 0;
    return vmm && fd;
}

int alloc(int device, size_t bytes, Block *out) {
    memset(out, 0, sizeof(*out));
    out->fd = -1;
    CUmemAllocationProp prop = make_prop(device);
    size_t gran = 0;
    DRV(g_drv.MemGetAllocationGranularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
    if (gran == 0) gran = 2u << 20;
    size_t size = ((bytes + gran - 1) / gran) * gran;
    if (size == 0) size = gran;
    CUmemGenericAllocationHandle h;
    DRV(g_drv.MemCreate(&h, size, &prop, 0));
    CUdeviceptr p = 0;
    CUresult r = g_drv.MemAddressReserve(&p, size, gran, 0, 0);
    if (r != CUDA_SUCCESS) {
        g_drv.MemRelease(h);
        return drv_fail(r, "cuMemAddressReserve");
    }
    r = g_drv.MemMap(p, size, 0, h, 0);
    if (r != CUDA_SUCCESS) {
        g_drv.MemAddressFree(p, size);
        g_drv.MemRelease(h);
        return drv_fail(r, "cuMemMap");
    }
    if (int rc = set_access(p, size, device)) {
        g_drv.MemUnmap(p, size);
        g_drv.MemAddressFree(p, size);
        g_drv.MemRelease(h);
        return rc;
    }
    out->ptr = (void *)p;
    out->size = size;
    out->handle = (unsigned long long)h;
    out->device = device;
    out->mapped = true;
    return DDS_OK;
}

int export_fd(Block *b) {
    if (b->fd >= 0) return DDS_OK;
    int fd = -1;
    DRV(g_drv.MemExportToShareableHandle(&fd, (CUmemGenericAllocationHandle)b->handle,
                                         CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
    b->fd = fd;
    return DDS_OK;
}

int grant(const Block *b, int device) { return set_access((CUdeviceptr)b->ptr, b->size, device); }

int import_fd(int device, int fd, size_t size, Block *out) {
    memset(out, 0, sizeof(*out));
    out->fd = -1;
    CUmemAllocationProp prop = make_prop(device);
    size_t gran = 0;
    DRV(g_drv.MemGetAllocationGranularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
    if (gran == 0) gran = 2u << 20;
    CUmemGenericAllocationHandle h;
    DRV(g_drv.MemImportFromShareableHandle(&h, (void *)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
    CUdeviceptr p = 0;
    CUresult r = g_drv.MemAddressReserve(&p, size, gran, 0, 0);
    if (r != CUDA_SUCCESS) {
        g_drv.MemRelease(h);
        return drv_fail(r, "cuMemAddressReserve (import)");
    }
    r = g_drv.MemMap(p, size, 0, h, 0);
    if (r != CUDA_SUCCESS) {
        g_drv.MemAddressFree(p, size);
        g_drv.MemRelease(h);
        return drv_fail(r, "cuMemMap (import)");
    }
    if (int rc = set_access(p, size, device)) {
        g_drv.MemUnmap(p, size);
        g_drv.MemAddressFree(p, size);
        g_drv.MemRelease(h);
        return rc;
    }
    out->ptr = (void *)p;
    out->size = size;
    out->handle = (unsigned long long)h;
    out->device = device;
    out->mapped = true;
    return DDS_OK;
}

namespace {

// map `size` bytes of memfd `fd` and register them mapped + portable (valid on every device of the process)
int host_map(int fd, size_t size, Block *out) {
    void *h = mmap(nullptr, size, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    if (h == MAP_FAILED) return dds_internal::fail(DDS_ERR_CUDA, "host shard: mmap failed");
    cudaError_t e = cudaHostRegister(h, size, cudaHostRegisterMapped | cudaHostRegisterPortable);
    void *d = nullptr;
    if (e == cudaSuccess) {
        e = cudaHostGetDevicePointer(&d, h, 0);
        if (e != cudaSuccess) cudaHostUnregister(h);
    }
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        munmap(h, size);
        return dds_internal::fail(DDS_ERR_CUDA, std::string("host shard: cudaHostRegister: ") + cudaGetErrorString(e));
    }
    out->ptr = d;
    out->host = h;
    out->size = size;
    out->mapped = true;
    return DDS_OK;
}

} // namespace

int host_alloc(size_t bytes, Block *out) {
    memset(out, 0, sizeof(*out));
    out->fd = -1;
    const size_t page = (size_t)sysconf(_SC_PAGESIZE);
    size_t size = ((bytes + page - 1) / page) * page;
    if (size == 0) size = page;
    int fd = memfd_create("dds-host-shard", MFD_CLOEXEC);
    if (fd < 0) return dds_internal::fail(DDS_ERR_CUDA, "host shard: memfd_create failed");
    if (ftruncate(fd, (off_t)size) != 0) {
        close(fd);
        return dds_internal::fail(DDS_ERR_CUDA, "host shard: ftruncate failed");
    }
    if (int rc = host_map(fd, size, out)) {
        close(fd);
        return rc;
    }
    out->fd = fd;
    return DDS_OK;
}

int host_import(int fd, size_t size, Block *out) {
    memset(out, 0, sizeof(*out));
    out->fd = -1;
    return host_map(fd, size, out);
}

void release(Block *b) {
    if (!b || !b->mapped) return;
    if (b->fd >= 0) close(b->fd);
    if (b->host) {
        cudaHostUnregister(b->host);
        munmap(b->host, b->size);
        b->host = nullptr;
        b->mapped = false;
        b->ptr = nullptr;
        b->fd = -1;
        return;
    }
    g_drv.MemUnmap((CUdeviceptr)b->ptr, b->size);
    g_drv.MemAddressFree((CUdeviceptr)b->ptr, b->size);
    g_drv.MemRelease((CUmemGenericAllocationHandle)b->handle);
    b->mapped = false;
    b->ptr = nullptr;
    b->fd = -1;
}

// Every rank hands `my_fd` to each rank r with want[r] != 0 and receives one descriptor from each such rank
// (want is symmetric: ranks of other processes on this host). COLLECTIVE over `comm` (two barriers).
// The sockets live in the abstract namespace under a name derived from a random job token; every datagram is checked
// against the kernel-supplied sender credentials (SO_PASSCRED: same uid, and the pid that rank published in the
// bootstrap all-gather), so another local process can neither inject a descriptor nor impersonate a rank; messages
// that fail the check are dropped. A rank whose export failed sends "no descriptor" (my_fd < 0) explicitly.
int exchange_fds(dds_comm_t *comm, const std::string &tag, int my_fd, const std::vector<char> &want,
                 const std::vector<int> &pids, std::vector<int> *got) {
    const int rank = dds_comm_rank(comm), size = dds_comm_size(comm);
    got->assign((size_t)size, -1);
    int expect = 0;
    for (int r = 0; r < size; r++) expect += (r != rank && want[(size_t)r]) ? 1 : 0;
    int sock = socket(AF_UNIX, SOCK_DGRAM | SOCK_CLOEXEC, 0);
    if (sock < 0) return dds_internal::fail(DDS_ERR_COMM, "fd exchange: socket() failed");
    socklen_t alen;
    sockaddr_un me = abstract_addr(tag + "-" + std::to_string(rank), &alen);
    int rc = DDS_OK;
    int one = 1;
    if (setsockopt(sock, SOL_SOCKET, SO_PASSCRED, &one, sizeof(one)) != 0)
        rc = dds_internal::fail(DDS_ERR_COMM, "fd exchange: SO_PASSCRED failed");
    if (!rc && bind(sock, (sockaddr *)&me, alen) != 0) rc = dds_internal::fail(DDS_ERR_COMM, "fd exchange: bind() failed");
    int brc = dds_comm_barrier(comm); // every socket is bound before anyone sends
    if (!rc) rc = brc;
    struct Msg {
        int32_t rank, has_fd;
    };
    if (!rc) {
        for (int r = 0; r < size && !rc; r++) {
            if (r == rank || !want[(size_t)r]) continue;
            socklen_t plen;
            sockaddr_un peer = abstract_addr(tag + "-" + std::to_string(r), &plen);
            Msg payload = {rank, my_fd >= 0 ? 1 : 0};
            iovec iov = {&payload, sizeof(payload)};
            char ctrl[CMSG_SPACE(sizeof(int))];
            memset(ctrl, 0, sizeof(ctrl));
            msghdr msg;
            memset(&msg, 0, sizeof(msg));
            msg.msg_name = &peer;
            msg.msg_namelen = plen;
            msg.msg_iov = &iov;
            msg.msg_iovlen = 1;
            if (my_fd >= 0) {
                msg.msg_control = ctrl;
                msg.msg_controllen = sizeof(ctrl);
                cmsghdr *c = CMSG_FIRSTHDR(&msg);
                c->cmsg_level = SOL_SOCKET;
                c->cmsg_type = SCM_RIGHTS;
                c->cmsg_len = CMSG_LEN(sizeof(int));
                memcpy(CMSG_DATA(c), &my_fd, sizeof(int));
            }
            if (sendmsg(sock, &msg, 0) < 0) rc = dds_internal::fail(DDS_ERR_COMM, "fd exchange: sendmsg() failed");
        }
        std::vector<char> seen((size_t)size, 0);
        for (int k = 0; k < expect && !rc;) {
            pollfd pf = {sock, POLLIN, 0};
            if (poll(&pf, 1, 120000) <= 0) {
                rc = dds_internal::fail(DDS_ERR_COMM, "fd exchange: timed out waiting for a peer's descriptor");
                break;
            }
            Msg from = {-1, 0};
            iovec iov = {&from, sizeof(from)};
            char ctrl[CMSG_SPACE(sizeof(int)) + CMSG_SPACE(sizeof(struct ucred))];
            msghdr msg;
            memset(&msg, 0, sizeof(msg));
            msg.msg_iov = &iov;
            msg.msg_iovlen = 1;
            msg.msg_control = ctrl;
            msg.msg_controllen = sizeof(ctrl);
            ssize_t n = recvmsg(sock, &msg, MSG_CMSG_CLOEXEC);
            if (n < 0) {
                rc = dds_internal::fail(DDS_ERR_COMM, "fd exchange: recvmsg() failed");
                break;
            }
            int fd = -1;
            bool have_cred = false;
            struct ucred cred;
            memset(&cred, 0, sizeof(cred));
            for (cmsghdr *c = CMSG_FIRSTHDR(&msg); c; c = CMSG_NXTHDR(&msg, c)) {
                if (c->cmsg_level != SOL_SOCKET) continue;
                if (c->cmsg_type == SCM_RIGHTS && c->cmsg_len >= CMSG_LEN(sizeof(int))) memcpy(&fd, CMSG_DATA(c), sizeof(int));
                if (c->cmsg_type == SCM_CREDENTIALS && c->cmsg_len >= CMSG_LEN(sizeof(struct ucred))) {
                    memcpy(&cred, CMSG_DATA(c), sizeof(cred));
                    have_cred = true;
                }
            }
            const bool ok = n == (ssize_t)sizeof(from) && have_cred && cred.uid == geteuid() && from.rank >= 0 &&
                            from.rank < size && from.rank != rank && want[(size_t)from.rank] && !seen[(size_t)from.rank] &&
                            (int)cred.pid == pids[(size_t)from.rank] && (from.has_fd != 0) == (fd >= 0);
            if (!ok) { // not one of ours (or a duplicate): drop it, keep waiting for the real peer
                if (fd >= 0) close(fd);
                continue;
            }
            seen[(size_t)from.rank] = 1;
            (*got)[(size_t)from.rank] = fd; // -1: the peer had nothing to export
            k++;
        }
    }
    brc = dds_comm_barrier(comm); // nobody closes its socket while a peer may still be sending to it
    close(sock);
    return rc ? rc : brc;
}

} // namespace dds_vmm
