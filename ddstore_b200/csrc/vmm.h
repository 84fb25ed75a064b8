// ddstore_b200/csrc/vmm.h -- CUDA VMM shard blocks, mapped host shard blocks + descriptor passing (see vmm.cpp)
#ifndef DDS_VMM_H
#define DDS_VMM_H
#include <stddef.h>

#include <string>
#include <vector>

#include "ddstore_b200.h"

namespace dds_vmm {

struct Block {
    void *ptr;
    size_t size;               // mapped size (multiple of the allocation granularity, or of the page size)
    unsigned long long handle; // CUmemGenericAllocationHandle
    int device;
    int fd;                    // exported POSIX fd (owner side), -1 otherwise
    bool mapped;
    void *host;                // host shard block: the mmap'd address (ptr is its device alias); nullptr for HBM
};

bool available(int device);
int alloc(int device, size_t bytes, Block *out);
int export_fd(Block *b);
int grant(const Block *b, int device); // let another device of THIS process read/write the block
int import_fd(int device, int fd, size_t size, Block *out);
// Host shard blocks: a memfd mapped MAP_SHARED and registered mapped + portable, so that kernels on any device of the
// process read it over PCIe through `ptr`. The owner keeps the memfd in `fd` for exchange_fds; every other process
// maps the descriptor it received.
int host_alloc(size_t bytes, Block *out);
int host_import(int fd, size_t size, Block *out);
void release(Block *b); // either kind
// my_fd < 0: nothing to export (sent explicitly); pids[r] = process id rank r published (sender verification)
int exchange_fds(dds_comm_t *comm, const std::string &tag, int my_fd, const std::vector<char> &want,
                 const std::vector<int> &pids, std::vector<int> *got);

} // namespace dds_vmm
#endif
