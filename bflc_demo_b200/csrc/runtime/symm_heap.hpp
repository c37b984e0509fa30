// Symmetric HBM heap: the same-sized allocation on every rank, each rank's pages mapped
// into every other rank's address space so kernels can ld/st peer memory directly over
// NVLink 4 / NVSwitch, plus (when the fabric allows it) an NVLS multicast mapping whose
// stores land in every replica.
//
// This replaces the reference's transport stack -- TLS "Channel" client->node, FISCO p2p
// + PBFT node<->node, JSON-in-ABI payloads (README.md:238-260, main.py:158,219) -- see
// SURVEY.md 5.8.  Handle exchange is done by the caller (torch.distributed object
// all-gather); this class only exports/imports opaque handle blobs.
//
// Two substrates:
//   VMM : cuMemCreate + POSIX-fd export, peers import the fd through pidfd_getfd(2);
//         required for multicast (cuMulticastCreate/AddDevice/BindMem).
//   IPC : cudaMalloc + cudaIpcGetMemHandle / cudaIpcOpenMemHandle (no multicast).
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

namespace bflc {

class SymmHeap {
 public:
  enum class Mode : int { LOCAL = 0, IPC = 1, VMM = 2 };

  SymmHeap(size_t bytes, int rank, int world, int device, Mode mode);
  ~SymmHeap();
  SymmHeap(const SymmHeap&) = delete;
  SymmHeap& operator=(const SymmHeap&) = delete;

  // opaque blob describing this rank's allocation (IPC handle, or {pid, fd})
  std::string export_handle() const;
  // blobs of all ranks, indexed by rank (own entry ignored)
  void import_handles(const std::vector<std::string>& blobs);

  // VMM handle exchange over abstract unix sockets (SCM_RIGHTS) -- works where pidfd_getfd is
  // denied (ptrace scope / seccomp).  Protocol: every rank calls fd_listen() and publishes the
  // returned name; after a barrier every rank calls import_via_sockets(names).
  std::string fd_listen(const std::string& unique_tag);
  void import_via_sockets(const std::vector<std::string>& names);
  // multicast over the same sockets: rank 0 must have called mc_create_and_export() first
  bool mc_import_via_sockets(const std::vector<std::string>& names);

  // multicast (VMM mode only). Rank 0 creates and exports; everyone imports/binds/maps.
  // Returns empty string when the device or driver does not support multicast.
  std::string mc_create_and_export();
  bool mc_import_and_add(const std::string& blob);  // step 1: every rank adds its device
  bool mc_bind_and_map();                            // step 2 (after a barrier): bind + map

  void* local_ptr() const { return local_; }
  void* peer_ptr(int r) const { return peers_.at(static_cast<size_t>(r)); }
  void* mc_ptr() const { return mc_va_; }
  size_t bytes() const { return bytes_; }
  int rank() const { return rank_; }
  int world() const { return world_; }
  Mode mode() const { return mode_; }
  static bool multicast_supported(int device);
  const std::string& last_error() const { return err_; }

 private:
  size_t bytes_ = 0;
  int rank_ = 0, world_ = 1, device_ = 0;
  Mode mode_ = Mode::LOCAL;
  void* local_ = nullptr;
  std::vector<void*> peers_;
  // VMM state
  unsigned long long mem_handle_ = 0;
  int export_fd_ = -1;
  std::vector<unsigned long long> peer_handles_;
  unsigned long long mc_handle_ = 0;
  int mc_fd_ = -1;
  void* mc_va_ = nullptr;
  bool mc_bound_ = false;
  int listen_fd_ = -1;
  std::vector<int> exchange_fds(const std::vector<std::string>& names, int my_fd);
  void map_peer_fd(int r, int fd);
  mutable std::string err_;
};

}  // namespace bflc
