// Symmetric (peer-mapped) + multicast (NVLS) device memory built directly on the CUDA VMM
// driver API: cuMemCreate / export POSIX fd / SCM_RIGHTS fd passing / cuMemImport / cuMemMap,
// and cuMulticastCreate / AddDevice / BindMem for the switch-replicated alias.
//
// This is the GPU stand-in for what libmpi gives the reference (a shared address space for
// collectives over host buffers, /root/reference/mpi_comms.py:88,132,162): every rank's gradient
// wire arena, parameter arena and signal pad are mapped into every process, so one kernel can
// gather / reduce / broadcast with plain loads and stores over NVLink.  No NCCL, no MPI.
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>
#include <thread>
#include <vector>
#include <atomic>

namespace psb {

class SymmBlock {
 public:
  // Phase 0: allocate the local physical block, export its fd and start the fd server.
  SymmBlock(int rank, int world, int device, size_t bytes, const std::string& sock_prefix);
  ~SymmBlock();
  SymmBlock(const SymmBlock&) = delete;
  SymmBlock& operator=(const SymmBlock&) = delete;

  // Phase 1 (after a cross-process barrier): import + map every peer's block.
  void map_peers();
  // Phase 2: multicast.  Rank 0 creates the object (mc_create); after a barrier the others
  // import it (mc_import); everyone adds its device (mc_add_device); after a barrier everyone
  // binds its memory and maps the multicast VA (mc_bind_and_map).  Each returns false (and
  // records why) instead of throwing, so the caller can agree on a fallback collectively.
  bool mc_supported() const;
  bool mc_create();
  bool mc_import();
  bool mc_add_device();
  bool mc_bind_and_map();
  void stop_server();   // after the last peer has fetched what it needs

  size_t size() const { return size_; }               // rounded-up size actually mapped
  size_t requested() const { return requested_; }
  int rank() const { return rank_; }
  int world() const { return world_; }
  int device() const { return device_; }
  uint64_t ptr(int r) const { return ptrs_.at(r); }   // rank r's block as mapped here
  const std::vector<uint64_t>& ptrs() const { return ptrs_; }
  uint64_t mc_ptr() const { return mc_ptr_; }         // 0 when multicast is unavailable
  const std::string& last_error() const { return err_; }

 private:
  void serve();
  int fetch_fd(int from_rank, char what);
  int rank_, world_, device_;
  size_t requested_, size_ = 0, gran_ = 0;
  std::string prefix_, err_;
  unsigned long long handle_ = 0;                      // CUmemGenericAllocationHandle (local)
  std::vector<unsigned long long> peer_handles_;
  std::vector<uint64_t> ptrs_;
  unsigned long long mc_handle_ = 0;
  bool mc_created_ = false, mc_bound_ = false;
  uint64_t mc_ptr_ = 0;
  int local_fd_ = -1, mc_fd_ = -1, listen_fd_ = -1;
  std::thread server_;
  std::atomic<bool> stop_{false};
};

}  // namespace psb
