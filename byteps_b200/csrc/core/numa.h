// NUMA placement helpers (raw Linux syscalls and sysfs; no libnuma - it is not in the image, and the reference
// only reaches NUMA through `numactl` in its launcher, /root/reference/launcher/launch.py:155-204).
//
// Why they exist: in colocated CPU-server mode the GPU DMAs a partition straight out of the server's
// shared-memory store (pull by reference).  A device-timed copy profile on a 2-socket host showed those copies
// several times slower for runs of keys than for memory the copying process placed itself: the store of a key is first touched by whichever server
// thread handled its init push.  With BYTEPS_NUMA_AWARE=1 the worker announces the NUMA node of its GPU in the
// init push, the server binds the key's store to that node and prefers an engine thread on it, and the worker
// binds its own staging window the same way.  Everything here degrades to a no-op (returns false / -1) when the
// kernel, the container or a single-node host does not support it.
#pragma once
#include <stddef.h>

#include <string>
#include <vector>

namespace bps {

// number of NUMA nodes with memory (>= 1); BYTEPS_NUMA_FAKE_NODES overrides it for tests
int numa_num_nodes();
// node of a PCI device ("0000:1b:00.0", case-insensitive; what cudaDeviceGetPCIBusId returns), -1 if unknown
int numa_node_of_pci(const std::string& bus_id);
// CPUs of a node (parsed from /sys/devices/system/node/nodeN/cpulist); empty if unknown
std::vector<int> numa_cpus_of_node(int node);
// "0-3,8,10-11" -> {0,1,2,3,8,10,11}
std::vector<int> parse_cpu_list(const std::string& s);
// prefer `node` for the pages of [p, p+len) and migrate the ones that are already resident; false if refused
bool numa_bind_memory(void* p, size_t len, int node);
// node the page at `p` currently lives on (-1: not resident / unknown)
int numa_node_of_addr(const void* p);
// restrict the calling thread to the CPUs of `node` that it may already run on; false if none / refused
bool numa_pin_thread_to_node(int node);
// the whole process (calling thread's CPU mask - inherited by threads created afterwards - and its default memory
// policy) prefers `node`: what `numactl --cpunodebind=N --preferred=N` does for a server started on the GPUs' socket.
// Returns a bit mask: 1 = CPUs set, 2 = memory policy set.
int numa_prefer_node_for_process(int node);
// BYTEPS_NUMA_AWARE (default 0): the placement logic is opt-in until it has been measured on a 2-socket GPU host
bool numa_aware();

// the init push of a key carries (pushers, node of the pusher's GPU) in one int: low 16 bits pushers, next 8
// bits node + 1 (0 = no hint)
inline int numa_pack_head(int pushers, int node) { return (pushers & 0xffff) | (node >= 0 && node < 255 ? (node + 1) << 16 : 0); }
inline int numa_head_pushers(int head) { return head & 0xffff; }
inline int numa_head_node(int head) { return ((head >> 16) & 0xff) - 1; }

}  // namespace bps
