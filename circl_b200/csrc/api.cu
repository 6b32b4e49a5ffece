// circl_b200/csrc/api.cu -- C ABI of libcirclb200.so (declared in include/circl_b200.h):
// runtime (devices, worker threads, work sets), pointer classification, the host staging pipeline with its
// multi-GPU sharding, and the Kyber ring entry points.
#include <sched.h>
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "../../include/circl_b200.h"
#include "common.cuh"
#include "context.h"
#include "flow_internal.h"

#include <sys/mman.h>

namespace cb200 {

static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof g_err, fmt, ap);
  va_end(ap);
}

Runtime& rt() {
  // never destroyed: a process that exits without cb200_shutdown() must not join worker threads or release CUDA
  // objects from a static destructor (the CUDA runtime may already be gone by then)
  static Runtime* r = new Runtime;
  return *r;
}

// per-thread binding (see context.h)
static thread_local Dev* t_dev = nullptr;
static thread_local WorkSet* t_ws3 = nullptr;
static thread_local cudaStream_t t_stream = nullptr;  // cb200_set_stream

Dev& ctx() {
  if (!t_dev) {  // programming error inside the library: a flow ran outside DeviceCall / worker thread
    fprintf(stderr, "cb200: internal error: no device bound to this thread\n");
    abort();
  }
  return *t_dev;
}
WorkSet& wset(int slot) {
  if (slot >= 0 && slot < Dev::kSlots) return ctx().staging[slot];
  if (!t_ws3) {
    fprintf(stderr, "cb200: internal error: no work set bound to this thread\n");
    abort();
  }
  return *t_ws3;
}
bool profiling_on() { return rt().profiling; }

static const char* kKernelNames[KID_COUNT] = {
    "kyber_ntt", "kyber_invntt", "kyber_dot", "kyber_elementwise",
    "mlkem_hash_ek", "mlkem_g", "mlkem_sample", "mlkem_encrypt",
    "dil_ntt", "dil_invntt", "dil_dot", "dil_elementwise",
    "mldsa_expand_key", "mldsa_mu_rhoprime", "mldsa_mask", "mldsa_w", "mldsa_challenge", "mldsa_response",
    "mldsa_compact", "x25519", "hybrid_glue", "keccak_f1600", "sampler", "mlkem_sample_fix", "x448", "ed25519", "ed448",
    "hpke", "frodo", "frodo_gemm", "p256", "p384", "p521", "rsa", "prio3"};
const char* kernel_name(int id) { return (id >= 0 && id < KID_COUNT) ? kKernelNames[id] : "?"; }

KernelScope::KernelScope(int id_, cudaStream_t st_) : st(st_), id(id_) {
  Runtime& r = rt();
  r.launches.fetch_add(1, std::memory_order_relaxed);
  if (r.profiling) {
    cudaEventCreate(&a);
    cudaEventRecord(a, st);
  }
}
KernelScope::~KernelScope() {
  if (!a) return;
  Runtime& r = rt();
  cudaEvent_t b;
  cudaEventCreate(&b);
  cudaEventRecord(b, st);
  std::lock_guard<std::mutex> lock(r.prof_mu);
  r.prof.push_back(ProfRec{id, a, b});
}

int require_ready() {
  if (!rt().ready) {
    set_error("cb200: not initialised (call cb200_init or cb200_init_devices; there is no CPU fallback)");
    return CB200_ERR_NOT_INIT;
  }
  return 0;
}

bool is_device_ptr(const void* p, int* device) {
  if (!p) return false;
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  if (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) {
    if (device) *device = a.device;
    return true;
  }
  return false;
}

int ensure_scratch(int slot, size_t bytes) {
  Dev& c = ctx();
  if (c.scratch_bytes[slot] >= bytes) return 0;
  if (c.scratch[slot]) CB200_CUDA(cudaFree(c.scratch[slot]));
  c.scratch[slot] = nullptr;
  c.scratch_bytes[slot] = 0;
  CB200_CUDA(cudaMalloc(&c.scratch[slot], bytes));
  c.scratch_bytes[slot] = bytes;
  return 0;
}

int ensure_work(int slot, size_t bytes, void** out) {
  const int level = slot / kLevel1;
  WorkSet& w = wset(slot % kLevel1);
  if (w.work_bytes[level] < bytes) {
    // kernels of earlier calls on this set may still be running: the set is only ever used from one stream (and
    // the lanes joined to it), and cudaFree waits for the device
    if (w.work[level]) CB200_CUDA(cudaFree(w.work[level]));
    w.work[level] = nullptr;
    w.work_bytes[level] = 0;
    CB200_CUDA(cudaMalloc(&w.work[level], bytes));
    w.work_bytes[level] = bytes;
  }
  *out = w.work[level];
  return 0;
}

int ensure_fix(int slot, int lane, size_t bytes, cudaStream_t st, void** out) {
  WorkSet& w = wset(slot % kLevel1);
  if (w.fix_bytes[lane] < bytes) {
    if (w.fix[lane]) CB200_CUDA(cudaFree(w.fix[lane]));  // waits for the device: no kernel still uses the old area
    w.fix[lane] = nullptr;
    w.fix_bytes[lane] = 0;
    CB200_CUDA(cudaMalloc(&w.fix[lane], bytes));
    w.fix_bytes[lane] = bytes;
    CB200_CUDA(cudaMemsetAsync(w.fix[lane], 0, 64, st));  // the counters in front of the list
  }
  *out = w.fix[lane];
  return 0;
}

int ensure_pinned(size_t bytes, void** out) {
  Dev& c = ctx();
  if (c.pinned_bytes < bytes) {
    if (c.pinned) CB200_CUDA(cudaFreeHost(c.pinned));
    c.pinned = nullptr;
    c.pinned_bytes = 0;
    CB200_CUDA(cudaHostAlloc(&c.pinned, bytes, cudaHostAllocDefault));
    c.pinned_bytes = bytes;
  }
  *out = c.pinned;
  return 0;
}

int ensure_smem_attr(const void* func, int bytes) {
  Dev& c = ctx();
  std::lock_guard<std::mutex> lock(c.attr_mu);
  if (c.attr_done.count(func)) return 0;
  CB200_CUDA(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  c.attr_done.insert(func);
  return 0;
}

// ---------------------------------------------------------------- work sets and devices
static int wset_create(WorkSet& w) {  // the owning device is current
  CB200_CUDA(cudaEventCreateWithFlags(&w.ev_fork, cudaEventDisableTiming));
  for (int l = 0; l < 2; l++) {
    CB200_CUDA(cudaStreamCreateWithFlags(&w.lane[l], cudaStreamNonBlocking));
    CB200_CUDA(cudaEventCreateWithFlags(&w.ev_join[l], cudaEventDisableTiming));
  }
  CB200_CUDA(cudaStreamCreateWithFlags(&w.copy, cudaStreamNonBlocking));
  CB200_CUDA(cudaEventCreateWithFlags(&w.ev_copy, cudaEventDisableTiming));
  CB200_CUDA(cudaMalloc(&w.small, 256));
  CB200_CUDA(cudaHostAlloc(&w.pin, 64, cudaHostAllocDefault));
  return 0;
}
static void wset_destroy(WorkSet& w) {
  for (int l = 0; l < 2; l++) {
    if (w.fix[l]) cudaFree(w.fix[l]);
    w.fix[l] = nullptr;
    w.fix_bytes[l] = 0;
    if (w.work[l]) cudaFree(w.work[l]);
    w.work[l] = nullptr;
    w.work_bytes[l] = 0;
    if (w.lane[l]) cudaStreamDestroy(w.lane[l]);
    if (w.ev_join[l]) cudaEventDestroy(w.ev_join[l]);
    w.lane[l] = nullptr;
    w.ev_join[l] = nullptr;
  }
  if (w.ev_fork) cudaEventDestroy(w.ev_fork);
  w.ev_fork = nullptr;
  if (w.copy) cudaStreamDestroy(w.copy);
  if (w.ev_copy) cudaEventDestroy(w.ev_copy);
  w.copy = nullptr;
  w.ev_copy = nullptr;
  if (w.small) cudaFree(w.small);
  if (w.pin) cudaFreeHost(w.pin);
  w.small = w.pin = nullptr;
}

// CPUs next to a GPU: /sys/bus/pci/devices/<bus id>/local_cpulist, intersected with what this process may use.
static bool local_cpus(int device, cpu_set_t* out) {
  char id[32] = "";
  if (cudaDeviceGetPCIBusId(id, sizeof id, device) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  for (char* p = id; *p; p++) *p = (char)tolower(*p);
  char path[128];
  snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/local_cpulist", id);
  FILE* f = fopen(path, "r");
  if (!f) return false;
  char line[1024] = "";
  const bool got = fgets(line, sizeof line, f) != nullptr;
  fclose(f);
  if (!got) return false;
  cpu_set_t allowed;
  CPU_ZERO(&allowed);
  if (sched_getaffinity(0, sizeof allowed, &allowed) != 0) return false;
  CPU_ZERO(out);
  int n = 0;
  for (char* tok = strtok(line, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
    int lo = 0, hi = 0;
    const int k = sscanf(tok, "%d-%d", &lo, &hi);
    if (k < 1) continue;
    if (k == 1) hi = lo;
    for (int c = lo; c <= hi && c < CPU_SETSIZE; c++)
      if (CPU_ISSET(c, &allowed)) {
        CPU_SET(c, out);
        n++;
      }
  }
  return n > 0;
}
static int bind_thread_near(int device) {
  if (getenv("CB200_NO_AFFINITY")) return 0;
  cpu_set_t set;
  if (!local_cpus(device, &set)) return 0;
  return sched_setaffinity(0, sizeof set, &set) == 0 ? CPU_COUNT(&set) : 0;
}

static void worker_main(Dev* d) {
  cudaSetDevice(d->device);
  bind_thread_near(d->device);  // staging copies from pageable memory and status scans stay on the GPU's NUMA node
  t_dev = d;
  for (;;) {
    std::function<void()> job;
    {
      std::unique_lock<std::mutex> lk(d->q_mu);
      d->q_cv.wait(lk, [&] { return d->stop || !d->q.empty(); });
      if (d->q.empty()) return;
      job = std::move(d->q.front());
      d->q.pop_front();
    }
    job();
  }
}

static int dev_create(int device, std::unique_ptr<Dev>* out) {
  CB200_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  CB200_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("cb200_init: device %d is sm_%d%d; this build contains only sm_90a code", device, prop.major, prop.minor);
    return CB200_ERR_NOT_INIT;
  }
  std::unique_ptr<Dev> d(new Dev);
  d->device = device;
  d->sm_count = prop.multiProcessorCount;
  CB200_CUDA(cudaStreamCreateWithFlags(&d->h2d, cudaStreamNonBlocking));
  CB200_CUDA(cudaStreamCreateWithFlags(&d->d2h, cudaStreamNonBlocking));
  for (int s = 0; s < Dev::kSlots; s++) {
    CB200_CUDA(cudaStreamCreateWithFlags(&d->pipe[s], cudaStreamNonBlocking));
    CB200_CUDA(cudaEventCreateWithFlags(&d->ev_in[s], cudaEventDisableTiming));
    CB200_CUDA(cudaEventCreateWithFlags(&d->ev_k[s], cudaEventDisableTiming));
    CB200_CUDA(cudaEventCreateWithFlags(&d->ev_out[s], cudaEventDisableTiming));
    int rc = wset_create(d->staging[s]);
    if (rc) return rc;
  }
  int32_t ktw[512];
  kyber_fill_twiddles(ktw);
  CB200_CUDA(cudaMalloc(&d->kyber_tw, sizeof ktw));
  CB200_CUDA(cudaMemcpy(d->kyber_tw, ktw, sizeof ktw, cudaMemcpyHostToDevice));
  int rc = init_extra_tables(*d);
  if (rc) return rc;
  d->worker = std::thread(worker_main, d.get());
  *out = std::move(d);
  return 0;
}
static void dev_destroy(Dev& d) {
  {
    std::lock_guard<std::mutex> lk(d.q_mu);
    d.stop = true;
  }
  d.q_cv.notify_all();
  if (d.worker.joinable()) d.worker.join();
  cudaSetDevice(d.device);
  cudaDeviceSynchronize();
  for (int s = 0; s < Dev::kSlots; s++) {
    if (d.scratch[s]) cudaFree(d.scratch[s]);
    if (d.pipe[s]) cudaStreamDestroy(d.pipe[s]);
    if (d.ev_in[s]) cudaEventDestroy(d.ev_in[s]);
    if (d.ev_k[s]) cudaEventDestroy(d.ev_k[s]);
    if (d.ev_out[s]) cudaEventDestroy(d.ev_out[s]);
    wset_destroy(d.staging[s]);
  }
  if (d.h2d) cudaStreamDestroy(d.h2d);
  if (d.d2h) cudaStreamDestroy(d.d2h);
  for (auto& kv : d.sets) wset_destroy(*kv.second);
  d.sets.clear();
  if (d.pinned) cudaFreeHost(d.pinned);
  if (d.kyber_tw) cudaFree(d.kyber_tw);
  if (d.dil_tw) cudaFree(d.dil_tw);
  if (d.x25519_table) cudaFree(d.x25519_table);
  if (d.ed448_table) cudaFree(d.ed448_table);
  if (d.p256_table) cudaFree(d.p256_table);
  if (d.p384_table) cudaFree(d.p384_table);
  if (d.p521_table) cudaFree(d.p521_table);
}
static Dev* dev_by_ordinal(int device) {
  for (auto& d : rt().devs)
    if (d->device == device) return d.get();
  return nullptr;
}

DeviceCall::DeviceCall(const void* buf) : prev_dev_(t_dev), prev_ws_(t_ws3) {
  int ordinal = -1;
  if (!is_device_ptr(buf, &ordinal)) {
    set_error("cb200: internal error: DeviceCall on a host pointer");
    rc = CB200_ERR_ARG;
    return;
  }
  dev = dev_by_ordinal(ordinal);
  if (!dev) {
    set_error("cb200: the buffers live on GPU %d, which this library was not initialised on", ordinal);
    rc = CB200_ERR_NOT_INIT;
    return;
  }
  cudaGetDevice(&prev_device_);
  if (prev_device_ != ordinal && cudaSetDevice(ordinal) != cudaSuccess) {
    set_error("cb200: cudaSetDevice(%d) failed: %s", ordinal, cudaGetErrorString(cudaGetLastError()));
    rc = CB200_ERR_NOT_INIT;
    return;
  }
  st = t_stream;
  {
    std::lock_guard<std::mutex> lk(dev->sets_mu);
    std::unique_ptr<WorkSet>& slot = dev->sets[st];
    if (!slot) {
      slot.reset(new WorkSet);
      rc = wset_create(*slot);
      if (rc) {
        wset_destroy(*slot);
        dev->sets.erase(st);
        return;
      }
    }
    ws = slot.get();
  }
  lock_ = std::unique_lock<std::mutex>(ws->mu);
  t_dev = dev;
  t_ws3 = ws;
}
DeviceCall::~DeviceCall() {
  if (lock_.owns_lock()) lock_.unlock();
  t_dev = prev_dev_;
  t_ws3 = prev_ws_;
  if (prev_device_ >= 0 && dev && prev_device_ != dev->device) cudaSetDevice(prev_device_);
}

// ---------------------------------------------------------------- host-pointer calls
static void post(Dev& d, std::function<void()> job) {
  {
    std::lock_guard<std::mutex> lk(d.q_mu);
    d.q.push_back(std::move(job));
  }
  d.q_cv.notify_one();
}

int for_each_shard(size_t n, size_t min_shard, const std::function<int(size_t first, size_t count)>& fn) {
  Runtime& r = rt();
  const size_t nd = r.devs.size();
  if (nd == 0) return require_ready();
  if (min_shard == 0) min_shard = 1;
  size_t shards = 1;
  if (nd > 1 && n >= 2 * min_shard) shards = std::min(nd, n / min_shard);
  struct Res {
    int rc = 0;
    std::string err;
  };
  std::vector<Res> res(shards);
  std::mutex mu;
  std::condition_variable cv;
  size_t done = 0;
  const size_t rot = shards == 1 ? r.next_dev.fetch_add(1, std::memory_order_relaxed) % nd : 0;
  for (size_t s = 0; s < shards; s++) {
    const size_t first = n * s / shards, cnt = n * (s + 1) / shards - first;
    Dev& d = *r.devs[(s + rot) % nd];
    post(d, [&, s, first, cnt] {
      g_err[0] = 0;
      const int rc = cnt ? fn(first, cnt) : 0;
      res[s].rc = rc;
      if (rc) res[s].err = g_err;
      std::lock_guard<std::mutex> lk(mu);
      done++;
      cv.notify_one();
    });
  }
  {
    std::unique_lock<std::mutex> lk(mu);
    cv.wait(lk, [&] { return done == shards; });
  }
  for (size_t s = 0; s < shards; s++)
    if (res[s].rc) {
      set_error("%s", res[s].err.c_str());
      return res[s].rc;
    }
  return 0;
}

int run_staged(std::vector<Buf>& bufs, size_t first0, size_t n, size_t chunk,
               const std::function<int(void** dev, size_t count, size_t first, cudaStream_t st, int slot)>& body) {
  Dev& c = ctx();
  if (chunk == 0 || chunk > n) chunk = n;
  const size_t nb = bufs.size();
  std::vector<size_t> off(nb + 1, 0);
  for (size_t i = 0; i < nb; i++) {
    size_t sz = bufs[i].shared ? bufs[i].unit : bufs[i].unit * chunk;
    off[i + 1] = off[i] + ((sz + 255) & ~(size_t)255);
  }
  std::vector<size_t> sched;
  // Chunk schedule: the first and the last chunks are short (1/4, 1/4, 1/2 of `chunk` on the way up, the mirror
  // image on the way down) so that the part of the pipeline that cannot overlap -- the first input copy and the last
  // kernels + output copy -- is a quarter of a chunk instead of a whole one.  Only worth it for long batches.
  {
    const size_t ramp[3] = {chunk / 4, chunk / 4, chunk / 2};
    size_t left = n;
    std::vector<size_t> tail;
    if (n >= 6 * chunk && chunk >= 4096) {
      for (size_t r : ramp) {
        sched.push_back(r);
        tail.push_back(r);
        left -= 2 * r;
      }
    }
    while (left > 0) {
      const size_t cnt = left < chunk ? left : chunk;
      sched.push_back(cnt);
      left -= cnt;
    }
    for (size_t k = tail.size(); k-- > 0;) sched.push_back(tail[k]);
  }
  constexpr int S = Dev::kSlots;
  const int used = (int)std::min<size_t>(S, sched.size());
  for (int s = 0; s < used; s++) {
    int rc = ensure_scratch(s, off[nb]);
    if (rc) return rc;
  }
  // a buffer that is copied in AND out (in-place ring ops) must not be refilled before its output copy is done
  bool inout = false;
  for (size_t i = 0; i < nb; i++) inout |= (bufs[i].host_in && bufs[i].host_out);
  std::vector<void*> dev(nb);
  int rc = 0;
  size_t first = first0;
  for (size_t ci = 0; ci < sched.size() && rc == 0; first += sched[ci], ci++) {
    const int slot = (int)(ci % S);
    const size_t count = sched[ci];
    cudaStream_t st = c.pipe[slot];
    // inputs: the slot's previous occupant (chunk ci - S) has finished reading them once its kernels are done
    if (ci >= (size_t)S) CB200_CUDA(cudaStreamWaitEvent(c.h2d, inout ? c.ev_out[slot] : c.ev_k[slot], 0));
    for (size_t i = 0; i < nb; i++) {
      dev[i] = (char*)c.scratch[slot] + off[i];
      if (bufs[i].host_in) {
        const size_t hs = bufs[i].host_stride ? bufs[i].host_stride : bufs[i].unit;
        const char* src = (const char*)bufs[i].host_in + (bufs[i].shared ? 0 : first * hs);
        if (bufs[i].shared || hs == bufs[i].unit) {
          size_t sz = bufs[i].shared ? bufs[i].unit : count * bufs[i].unit;
          CB200_CUDA(cudaMemcpyAsync(dev[i], src, sz, cudaMemcpyHostToDevice, c.h2d));
        } else {
          CB200_CUDA(cudaMemcpy2DAsync(dev[i], bufs[i].unit, src, hs, bufs[i].unit, count, cudaMemcpyHostToDevice, c.h2d));
        }
      }
    }
    CB200_CUDA(cudaEventRecord(c.ev_in[slot], c.h2d));
    // kernels: after this chunk's inputs, and after the output copy of the slot's previous occupant
    CB200_CUDA(cudaStreamWaitEvent(st, c.ev_in[slot], 0));
    if (ci >= (size_t)S) CB200_CUDA(cudaStreamWaitEvent(st, c.ev_out[slot], 0));
    rc = body(dev.data(), count, first, st, slot);
    if (rc) break;
    CB200_CUDA(cudaEventRecord(c.ev_k[slot], st));
    // outputs
    CB200_CUDA(cudaStreamWaitEvent(c.d2h, c.ev_k[slot], 0));
    for (size_t i = 0; i < nb; i++)
      if (bufs[i].host_out && !bufs[i].shared)
        CB200_CUDA(cudaMemcpyAsync((char*)bufs[i].host_out + first * bufs[i].unit, dev[i], count * bufs[i].unit,
                                   cudaMemcpyDeviceToHost, c.d2h));
    CB200_CUDA(cudaEventRecord(c.ev_out[slot], c.d2h));
  }
  CB200_CUDA(cudaStreamSynchronize(c.h2d));
  for (int s = 0; s < S; s++) CB200_CUDA(cudaStreamSynchronize(c.pipe[s]));
  CB200_CUDA(cudaStreamSynchronize(c.d2h));
  return rc;
}

int HostCall::run(size_t n) {
  bit0 = 0;
  bit1 = 0;
  nonzero = 0;
  return for_each_shard(n, min_shard, [&](size_t first0, size_t cnt) -> int {
    std::vector<Buf> b = bufs;
    uint8_t* pin = nullptr;
    if (status_buf >= 0) {
      void* p = nullptr;
      int rc = ensure_pinned(cnt, &p);
      if (rc) return rc;
      pin = (uint8_t*)p;
      b[status_buf].host_out = pin - first0;  // element `first` of the batch lands at pin[first - first0]
    }
    int rc = run_staged(b, first0, cnt, chunk, body);
    if (rc) return rc;
    if (pin) {
      size_t c0 = 0, c1 = 0, cz = 0;
      for (size_t i = 0; i < cnt; i++) {
        c0 += (pin[i] & 1) != 0;
        c1 += (pin[i] & 2) != 0;
        cz += pin[i] != 0;
      }
      bit0 += c0;
      bit1 += c1;
      nonzero += cz;
      if (user_status) memcpy(user_status + first0, pin, cnt);
    }
    return 0;
  });
}

// number of polynomials per staging chunk: 64 MiB of int16 polys keeps three
// chunks in flight well under any memory pressure and amortises launch latency.
static constexpr size_t kPolyChunk = 1u << 17;

}  // namespace cb200

using namespace cb200;

extern "C" {

const char* cb200_version(void) { return "circl_b200 0.2 (sm_90a)"; }
const char* cb200_last_error(void) { return g_err; }

int cb200_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

static int init_list(const int* ordinals, int count) {
  Runtime& r = rt();
  std::lock_guard<std::mutex> lock(r.init_mu);
  if (r.ready) {
    bool same = (int)r.devs.size() == count;
    for (int i = 0; same && i < count; i++) same = r.devs[i]->device == ordinals[i];
    if (same) return 0;
    r.ready = false;
    for (auto& d : r.devs) dev_destroy(*d);
    r.devs.clear();
  }
  int prev = -1;
  cudaGetDevice(&prev);
  for (int i = 0; i < count; i++) {
    std::unique_ptr<Dev> d;
    int rc = dev_create(ordinals[i], &d);
    if (rc) {
      for (auto& e : r.devs) dev_destroy(*e);
      r.devs.clear();
      return rc;
    }
    r.devs.push_back(std::move(d));
  }
  // leave the caller's current device as it was (first GPU of the set if it had none of ours selected)
  cudaSetDevice(dev_by_ordinal(prev) ? prev : ordinals[0]);
  r.launches = 0;
  r.ready = true;
  return 0;
}

int cb200_init(int device) {
  const int n = cb200_device_count();
  if (n <= 0) {
    set_error("cb200_init: no CUDA device visible (this library has no CPU fallback)");
    return CB200_ERR_NOT_INIT;
  }
  if (device < 0 || device >= n) {
    set_error("cb200_init: device %d out of range (have %d)", device, n);
    return CB200_ERR_ARG;
  }
  const int rc = init_list(&device, 1);
  if (rc == 0) cudaSetDevice(device);
  return rc;
}

int cb200_init_devices(int ndev) {
  const int n = cb200_device_count();
  if (n <= 0) {
    set_error("cb200_init_devices: no CUDA device visible (this library has no CPU fallback)");
    return CB200_ERR_NOT_INIT;
  }
  if (ndev <= 0) ndev = n;
  if (ndev > n) {
    set_error("cb200_init_devices: %d GPUs requested, %d visible", ndev, n);
    return CB200_ERR_ARG;
  }
  std::vector<int> ord(ndev);
  for (int i = 0; i < ndev; i++) ord[i] = i;
  return init_list(ord.data(), ndev);
}

int cb200_active_devices(void) { return rt().ready ? (int)rt().devs.size() : 0; }

void cb200_shutdown(void) {
  Runtime& r = rt();
  std::lock_guard<std::mutex> lock(r.init_mu);
  if (!r.ready) return;
  r.ready = false;
  int prev = -1;
  cudaGetDevice(&prev);
  for (auto& d : r.devs) dev_destroy(*d);
  r.devs.clear();
  if (prev >= 0) cudaSetDevice(prev);
}

int cb200_set_stream(void* s) {
  int rc = require_ready();
  if (rc) return rc;
  t_stream = (cudaStream_t)s;
  return 0;
}

int cb200_release_stream(void* s) {
  int rc = require_ready();
  if (rc) return rc;
  int prev = -1;
  cudaGetDevice(&prev);
  for (auto& d : rt().devs) {
    std::unique_ptr<WorkSet> w;
    {
      std::lock_guard<std::mutex> lk(d->sets_mu);
      auto it = d->sets.find((cudaStream_t)s);
      if (it == d->sets.end()) continue;
      w = std::move(it->second);
      d->sets.erase(it);
    }
    std::lock_guard<std::mutex> lk(w->mu);
    cudaSetDevice(d->device);
    cudaStreamSynchronize((cudaStream_t)s);
    wset_destroy(*w);
  }
  if (prev >= 0) cudaSetDevice(prev);
  return 0;
}

int cb200_synchronize(void) {
  int rc = require_ready();
  if (rc) return rc;
  CB200_CUDA(cudaStreamSynchronize(t_stream));
  return 0;
}

int cb200_bind_thread_to_device(int device) {
  const int n = bind_thread_near(device);
  if (n == 0) set_error("cb200_bind_thread_to_device: no local_cpulist for GPU %d (affinity unchanged)", device);
  return n;
}

void* cb200_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes, cudaHostAllocPortable) != cudaSuccess) {
    set_error("cb200_host_alloc(%zu) failed: %s", bytes, cudaGetErrorString(cudaGetLastError()));
    return nullptr;
  }
  return p;
}
// One pinned buffer for a batch that cb200_* host-pointer calls will split over all active GPUs: the rows of shard s
// (the split of for_each_shard) are first touched by the worker thread of the GPU that will copy them, which runs on
// that GPU's NUMA node, so every GPU's copies stay on its own socket.
static std::mutex g_map_mu;
static std::map<void*, size_t> g_mapped;  // buffers of cb200_host_alloc_batch: mmap + cudaHostRegister

void* cb200_host_alloc_batch(size_t n, size_t unit_bytes) {
  if (require_ready()) return nullptr;
  Runtime& r = rt();
  const size_t nd = r.devs.size();
  const size_t bytes = n * unit_bytes;
  if (bytes == 0) return nullptr;
  const size_t page = 4096, len = (bytes + page - 1) / page * page;
  void* p = mmap(nullptr, len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
  if (p == MAP_FAILED) {
    set_error("cb200_host_alloc_batch(%zu x %zu): mmap failed", n, unit_bytes);
    return nullptr;
  }
  std::mutex mu;
  std::condition_variable cv;
  size_t done = 0;
  for (size_t s = 0; s < nd; s++) {
    // page-rounded byte range of rows [n s / nd, n (s + 1) / nd)
    size_t lo = (n * s / nd) * unit_bytes / page * page, hi = (n * (s + 1) / nd) * unit_bytes / page * page;
    if (s + 1 == nd) hi = len;
    post(*r.devs[s], [&, lo, hi] {
      if (hi > lo) memset((char*)p + lo, 0, hi - lo);
      std::lock_guard<std::mutex> lk(mu);
      done++;
      cv.notify_one();
    });
  }
  {
    std::unique_lock<std::mutex> lk(mu);
    cv.wait(lk, [&] { return done == nd; });
  }
  if (cudaHostRegister(p, len, cudaHostRegisterPortable) != cudaSuccess) {
    set_error("cb200_host_alloc_batch: cudaHostRegister(%zu) failed: %s", len, cudaGetErrorString(cudaGetLastError()));
    munmap(p, len);
    return nullptr;
  }
  std::lock_guard<std::mutex> lk(g_map_mu);
  g_mapped[p] = len;
  return p;
}
void cb200_host_free(void* p) {
  if (!p) return;
  {
    std::lock_guard<std::mutex> lk(g_map_mu);
    auto it = g_mapped.find(p);
    if (it != g_mapped.end()) {
      cudaHostUnregister(p);
      munmap(p, it->second);
      g_mapped.erase(it);
      return;
    }
  }
  cudaFreeHost(p);
}

uint64_t cb200_launch_count(void) { return rt().launches.load(); }

int cb200_profile_enable(int on) {
  int rc = require_ready();
  if (rc) return rc;
  rt().profiling = on != 0;
  return 0;
}
int cb200_profile_kernel_count(void) { return KID_COUNT; }
const char* cb200_profile_kernel_name(int id) { return kernel_name(id); }
int cb200_profile_read(double* ms_total, uint64_t* launches, int n) {
  int rc = require_ready();
  if (rc) return rc;
  Runtime& r = rt();
  int prev = -1;
  cudaGetDevice(&prev);
  for (auto& d : r.devs) {
    cudaSetDevice(d->device);
    CB200_CUDA(cudaDeviceSynchronize());
  }
  if (prev >= 0) cudaSetDevice(prev);
  std::lock_guard<std::mutex> lock(r.prof_mu);
  for (int i = 0; i < n; i++) {
    ms_total[i] = 0;
    launches[i] = 0;
  }
  for (ProfRec& p : r.prof) {
    float ms = 0;
    cudaEventElapsedTime(&ms, p.a, p.b);
    if (p.id < n) {
      ms_total[p.id] += ms;
      launches[p.id] += 1;
    }
    cudaEventDestroy(p.a);
    cudaEventDestroy(p.b);
  }
  r.prof.clear();
  return 0;
}

// ---------------------------------------------------------------- Kyber ring ops
int cb200_kyber_ntt(int16_t* polys, size_t n, int inverse) {
  int rc = require_ready();
  if (rc) return rc;
  if (n == 0) return 0;
  if (!polys) {
    set_error("cb200_kyber_ntt: null pointer");
    return CB200_ERR_ARG;
  }
  Batch b{"cb200_kyber_ntt", n, polys, kPolyChunk, 1u << 15, {{polys, 512, 512, kInOut}},
          {{!aligned({polys}, {}, 16), "%s: device buffers must be 16-byte aligned"}}};
  return run_batch(b, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return launch_kyber_ntt((int16_t*)r[0].p, cnt, inverse, ctx().kyber_tw, st);
  });
}

int cb200_kyber_dot(int16_t* out, const int16_t* a, const int16_t* b, int k, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (n == 0) return 0;
  if (!out || !a || !b || k < 1 || k > 8) {
    set_error("cb200_kyber_dot: bad argument");
    return CB200_ERR_ARG;
  }
  const size_t ku = 512 * (size_t)k;
  Batch bt{"cb200_kyber_dot", n, out, kPolyChunk / k, (1u << 15) / k, {{out, 512, 512, kOut}, {a, ku, ku, kIn}, {b, ku, ku, kIn}},
           {{!aligned({out, a, b}, {}, 16), "%s: device buffers must be 16-byte aligned"}}};
  return run_batch(bt, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return launch_kyber_dot((int16_t*)r[0].p, (const int16_t*)r[1].p, (const int16_t*)r[2].p, k, cnt, ctx().kyber_tw, st);
  });
}

int cb200_kyber_mulhat(int16_t* out, const int16_t* a, const int16_t* b, size_t n) {
  return cb200_kyber_dot(out, a, b, 1, n);
}

int cb200_kyber_poly_op(int op, int16_t* out, const int16_t* a, const int16_t* b, size_t n) {
  int rc = require_ready();
  if (rc) return rc;
  if (n == 0) return 0;
  const bool binary = (op == CB200_OP_ADD || op == CB200_OP_SUB);
  if (!out || !a || (binary && !b) || op < 0 || op > CB200_OP_TOMONT) {
    set_error("cb200_kyber_poly_op: bad argument");
    return CB200_ERR_ARG;
  }
  if (!binary) b = nullptr;
  Batch bt{"cb200_kyber_poly_op", n, out, kPolyChunk, 1u << 15, {{out, 512, 512, kOut}, {a, 512, 512, kIn}, {b, 512, 512, kIn}},
           {{!aligned({out, a, b}, {}, 16), "%s: device buffers must be 16-byte aligned"}}};
  return run_batch(bt, [&](const Rows& r, size_t cnt, cudaStream_t st, int) {
    return launch_kyber_poly_op(op, (int16_t*)r[0].p, (const int16_t*)r[1].p, (const int16_t*)r[2].p, cnt, st);
  });
}

}  // extern "C"
