// circl_b200/csrc/context.h -- runtime behind the C ABI.
//
// One process may drive several GPUs (cb200_init_devices) or exactly one (cb200_init, the one-process-per-GPU
// launch of bench.py).  Per GPU there is a `Dev`: tables, the three-stream host staging pipeline and a worker
// thread that owns it.  Host-pointer batch calls are cut into contiguous index ranges, one per GPU, and each range
// runs on that GPU's worker (kem.Scheme / sign.Scheme callers never see devices; the results land in the caller's
// buffers, which is the gather).  Device-pointer calls run on the calling thread, asynchronously on the stream the
// thread named with cb200_set_stream; everything such a call needs besides its arguments (work areas, internal
// lanes, events, a pinned word) lives in a `WorkSet` keyed by (device, stream), so two threads on two streams never
// share scratch, and two threads on one stream are serialised by the WorkSet's mutex in stream order.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <atomic>
#include <condition_variable>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <string>
#include <thread>
#include <vector>

#include "launch.h"

namespace cb200 {

struct ProfRec {
  int id;
  cudaEvent_t a, b;
};

// What a multi-kernel flow needs besides its arguments.
struct WorkSet {
  // grow-only work areas: level 0 for the lattice flows (mlkem.cu, mldsa.cu), level 1 for the flows of hybrid.cu
  // that call into them
  void* work[2] = {nullptr, nullptr};
  size_t work_bytes[2] = {0, 0};
  // two internal lanes: consecutive sub-batches of a pipeline alternate between them so that the tail of one
  // sub-batch's kernels overlaps the head of the next (fork/join on events around them)
  cudaStream_t lane[2] = {nullptr, nullptr};
  cudaEvent_t ev_fork = nullptr, ev_join[2] = {nullptr, nullptr};
  cudaStream_t copy = nullptr;  // result pushes (cb200_gather_push): copy-engine traffic beside the kernels
  cudaEvent_t ev_copy = nullptr;
  void* fix[2] = {nullptr, nullptr};  // per lane: streams a sampler kernel left unfinished (mlkem.cu, sample_fix_kernel)
  size_t fix_bytes[2] = {0, 0};
  void* small = nullptr;  // 256-byte device buffer (ML-DSA context string of a device-pointer call)
  void* pin = nullptr;    // 64 bytes of pinned host memory (per-round counters of the signing loop)
  std::mutex mu;          // callers sharing this set enqueue one after the other
};

struct Dev {
  int device = -1;
  int sm_count = 0;             // multiprocessors of the device (sizes the persistent grids)
  void* kyber_tw = nullptr;     // 128 x {zeta, zetaq}, then 128 x {zp, kk} (kyber.cuh, low format)
  void* dil_tw = nullptr;       // 256 x {zeta, invzeta}
  void* x25519_table = nullptr; // 32 KiB: multiples 1..8 of 256^i B for the fixed-base X25519 KeyGen (x25519.cuh)
  void* ed448_table = nullptr;  // 84 KiB: multiples 1..8 of 256^i G for Ed448's fixed base (ed448.cuh)
  void* p256_table = nullptr;   // 32 KiB: affine multiples 1..8 of 16^i G for P-256's fixed base (p256.cuh)
  void* p384_table = nullptr;   // 72 KiB: the same for P-384 (p384.cuh)
  void* p521_table = nullptr;   // 139 KiB: the same for P-521 (p521.cuh)
  // host staging pipeline (owned by the worker thread).  A chunk lives in one of kSlots slots (device images of its
  // buffers + a work set); all input copies go down one stream, all output copies down another, the kernels of a
  // slot down that slot's stream, tied by events: the input copy of chunk c + kSlots waits only for the KERNELS of
  // chunk c (not for its output copy), so both copy engines stay busy across chunk boundaries.
  static constexpr int kSlots = 4;
  cudaStream_t pipe[kSlots] = {};
  cudaStream_t h2d = nullptr, d2h = nullptr;
  cudaEvent_t ev_in[kSlots] = {}, ev_k[kSlots] = {}, ev_out[kSlots] = {};
  void* scratch[kSlots] = {};
  size_t scratch_bytes[kSlots] = {};
  WorkSet staging[kSlots];      // work sets of the pipeline slots
  void* pinned = nullptr;       // grow-only pinned host staging for small per-op outputs (status bytes)
  size_t pinned_bytes = 0;
  // device-pointer calls: one work set per caller stream
  std::mutex sets_mu;
  std::map<cudaStream_t, std::unique_ptr<WorkSet>> sets;
  // kernels whose dynamic shared-memory limit has been raised on this device
  std::mutex attr_mu;
  std::set<const void*> attr_done;
  // worker thread: runs the host-pointer shards of this GPU one after the other
  std::thread worker;
  std::mutex q_mu;
  std::condition_variable q_cv;
  std::deque<std::function<void()>> q;
  bool stop = false;
};

struct Runtime {
  std::vector<std::unique_ptr<Dev>> devs;
  std::atomic<bool> ready{false};
  std::atomic<uint64_t> launches{0};
  std::atomic<unsigned> next_dev{0};  // small host-pointer calls rotate over the GPUs
  bool profiling = false;
  std::vector<ProfRec> prof;
  std::mutex prof_mu;
  std::mutex init_mu;
};
Runtime& rt();

// Kernel classes for the optional per-kernel event timing (cb200_profile_*).
enum KernelId {
  KID_KYBER_NTT = 0, KID_KYBER_INVNTT, KID_KYBER_DOT, KID_KYBER_EW,
  KID_MLKEM_HASH_EK, KID_MLKEM_G, KID_MLKEM_SAMPLE, KID_MLKEM_ENCRYPT,
  KID_DIL_NTT, KID_DIL_INVNTT, KID_DIL_DOT, KID_DIL_EW,
  KID_MLDSA_EXPAND, KID_MLDSA_MU, KID_MLDSA_MASK, KID_MLDSA_W, KID_MLDSA_CHALLENGE, KID_MLDSA_RESPONSE,
  KID_MLDSA_COMPACT, KID_X25519, KID_HYBRID_GLUE, KID_KECCAK, KID_SAMPLER, KID_MLKEM_SAMPLE_FIX, KID_X448, KID_ED25519, KID_ED448,
  KID_HPKE, KID_FRODO, KID_FRODO_GEMM, KID_P256, KID_P384, KID_P521, KID_RSA, KID_PRIO3, KID_COUNT
};
const char* kernel_name(int id);

// The device the calling thread is working on: set by a DeviceCall (device-pointer entry points) or by the worker
// thread of that device (host-pointer shards).  Flows only ever run inside one of the two.
Dev& ctx();
// Work set of `slot`: 0..kSlots-1 = pipeline slots of ctx(), kDevSlot = the set bound by the innermost DeviceCall.
constexpr int kDevSlot = Dev::kSlots;
constexpr int kLevel1 = 8;  // ensure_work(kLevel1 + slot, ...) = the level-1 area of that work set
WorkSet& wset(int slot);
bool profiling_on();

// Brackets one kernel launch with events when profiling is on; always counts the launch.
struct KernelScope {
  cudaStream_t st;
  int id;
  cudaEvent_t a = nullptr;
  KernelScope(int id, cudaStream_t st);
  ~KernelScope();
};
int require_ready();
// true for device (or managed) memory; *device receives the ordinal that owns it
bool is_device_ptr(const void* p, int* device = nullptr);
int ensure_scratch(int slot, size_t bytes);
// slot = level-0 area of that work set, kLevel1 + slot = its level-1 area
int ensure_work(int slot, size_t bytes, void** out);
int ensure_pinned(size_t bytes, void** out);
// grow-only per-lane list area of a work set; zero-filled (on `st`) whenever it is (re)allocated
int ensure_fix(int slot, int lane, size_t bytes, cudaStream_t st, void** out);
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (device, kernel)
int ensure_smem_attr(const void* func, int bytes);
inline void count_launch(uint64_t n = 1) { rt().launches.fetch_add(n, std::memory_order_relaxed); }

// Binds the calling thread to the device that owns the buffers of a device-pointer call and to the work set of
// (device, current stream of this thread) for the lifetime of the object.
struct DeviceCall {
  int rc = 0;
  cudaStream_t st = nullptr;
  Dev* dev = nullptr;
  WorkSet* ws = nullptr;
  explicit DeviceCall(const void* any_device_buffer);
  ~DeviceCall();
  DeviceCall(const DeviceCall&) = delete;
  DeviceCall& operator=(const DeviceCall&) = delete;

 private:
  Dev* prev_dev_;
  WorkSet* prev_ws_;
  int prev_device_ = -1;
  std::unique_lock<std::mutex> lock_;
};

// One buffer of a batched host-pointer call: `unit` bytes per batch element.
struct Buf {
  const void* host_in = nullptr;  // base of the whole batch; copied host -> device before the kernels (may be null)
  void* host_out = nullptr;       // base of the whole batch; copied device -> host after the kernels (may be null)
  size_t unit = 0;
  bool shared = false;            // whole buffer is `unit` bytes, identical for every element
  size_t host_stride = 0;         // bytes between elements in host memory (0 = dense = unit)
};

// A batched call on host pointers.  run(n) cuts [0, n) into one contiguous range per GPU (ranges of at least
// `min_shard` elements; small batches go to one GPU, rotating), and on each GPU's worker thread stages the range
// through HBM in chunks, overlapping the host<->device copies of one chunk with the kernels of another on three
// streams.  body(dev, count, first, stream, slot): dev[i] is the device image of bufs[i] for the current chunk,
// `first` the index of its first element in the whole batch.
struct HostCall {
  std::vector<Buf> bufs;
  size_t chunk = 1u << 15;
  size_t min_shard = 1u << 13;
  // index in bufs of the per-op status bytes (unit 1, no host pointers); they return through pinned memory, are
  // counted (bit 0 / bit 1 / any bit set) and copied to user_status if that is not null
  int status_buf = -1;
  uint8_t* user_status = nullptr;
  std::function<int(void** dev, size_t count, size_t first, cudaStream_t st, int slot)> body;
  std::atomic<size_t> bit0{0}, bit1{0}, nonzero{0};
  int run(size_t n);
};

// Runs fn(first, count) for one contiguous range per GPU, each on that GPU's worker thread (ctx() is that GPU);
// returns the first non-zero result and carries its error text over to the caller's thread.
int for_each_shard(size_t n, size_t min_shard, const std::function<int(size_t first, size_t count)>& fn);
// Staging pipeline of ctx() over elements [first0, first0 + n) of the batch described by bufs (worker thread only).
int run_staged(std::vector<Buf>& bufs, size_t first0, size_t n, size_t chunk,
               const std::function<int(void** dev, size_t count, size_t first, cudaStream_t st, int slot)>& body);

}  // namespace cb200
