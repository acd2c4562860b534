// Engine internals: pinned ring, HBM staging arena, worker pool, jobs.  See include/tsnap_b200.h for
// the contract and DESIGN.md for the pipeline picture.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "kernels.h"
#include "plan.h"

namespace tsnap {

int set_err(int code, const std::string& msg);
const char* last_err();

// where one I/O worker runs: CPU set it is bound to (empty = unbound) and the queue it serves first
struct WorkerSpec {
    std::vector<int> cpus;
    int queue = 0;
};

class WorkerPool {
   public:
    // one queue per NUMA node when the workers are node-bound (else one queue): a task posted with the queue of the
    // node its pinned slot lives on is copied by a CPU of that node; an idle worker takes work from the other queues
    WorkerPool(const std::vector<WorkerSpec>& workers, int n_queues);
    ~WorkerPool();
    void post(std::function<void()> fn, int queue = -1);
    int size() const { return int(threads_.size()); }
    int queues() const { return int(q_.size()); }

   private:
    void run(int home);
    std::vector<std::thread> threads_;
    std::vector<std::deque<std::function<void()>>> q_;
    size_t rr_ = 0;
    std::mutex mu_;
    std::condition_variable cv_;
    bool stop_ = false;
};

// fixed-size pinned slots handed out to in-flight chunks
class SlotRing {
   public:
    // every slot has `slack` extra bytes of capacity behind slot_bytes (O_DIRECT reads are widened to 4 KiB blocks).
    // `nodes` non-empty: slot i is placed on NUMA node nodes[i % size] (mmap + mbind + cudaHostRegister)
    int init(size_t slot_bytes, int n, bool pinned, size_t slack, const std::vector<int>& nodes);
    void destroy();
    char* acquire();  // blocks
    void release(char* p);
    int queue_of(const char* p) const;  // index into `nodes` of the slot's NUMA node, -1 when unplaced
    size_t slot_bytes() const { return slot_bytes_; }
    size_t total_bytes() const { return (slot_bytes_ + slack_) * all_.size(); }
    int count() const { return int(all_.size()); }

   private:
    size_t slot_bytes_ = 0, slack_ = 0;
    bool pinned_ = false;
    struct Placed {
        char* p;
        size_t len;   // mapping length when the slot was mmap'ed + registered (0: cudaHostAlloc / posix_memalign)
        int queue;
    };
    std::vector<Placed> placed_;
    std::vector<char*> all_;
    std::vector<char*> free_;
    std::mutex mu_;
    std::condition_variable cv_;
};

}  // namespace tsnap

struct tsnap_job;

struct tsnap_engine {
    tsnap_engine_config cfg{};
    int device = -1;
    int sm_count = 0;
    bool has_device = false;
    bool trace = false;      // TSNAP_ENGINE_TRACE
    bool odirect = false;    // TSNAP_ENGINE_ODIRECT
    bool no_arena = false;   // TSNAP_ENGINE_NO_ARENA
    std::vector<int> numa_cpus;  // CPUs of the NUMA node the GPU hangs off (empty = no binding)
    std::vector<int> ring_nodes; // NUMA nodes the ring slots are placed on, in queue order (empty = wherever they land)
    cudaStream_t s_kernel = nullptr;  // pack / unpack kernels
    cudaStream_t s_copy = nullptr;    // D2H / H2D payload copies
    tsnap::SlotRing ring;
    tsnap::WorkerPool* io = nullptr;
    // HBM staging arena (grow-only between jobs)
    char* arena = nullptr;
    size_t arena_bytes = 0;
    // the arena serves one device job at a time: the next one waits until the previous has fully completed
    std::mutex arena_mu;
    std::condition_variable arena_cv;
    bool arena_in_use = false;
    // cached whole-buffer pinned allocations for the stager seam, keyed by capacity
    std::mutex pin_mu;
    std::vector<std::pair<size_t, void*>> pin_cache;
    // job scheduling: one drain thread runs jobs FIFO; one completion thread retires chunk events
    std::thread drain_thread, completion_thread;
    std::mutex q_mu;
    std::condition_variable q_cv;
    std::deque<tsnap_job*> job_q;
    struct Pending {
        cudaEvent_t ev;
        std::function<void(bool ok)> done;
    };
    std::mutex c_mu;
    std::condition_variable c_cv;
    std::deque<Pending> pending;
    bool stopping = false;
    bool trim_arena = false;    // drain thread frees the HBM arena when it is idle
    bool busy = false;          // a job is being issued by the drain thread
    bool keep_arena = false;    // TSNAP_B200_KEEP_ARENA=1: do not give the engine-owned arena back when idle
    // device buffers for the member/tile tables of a launch (grow-only pool: no allocator call on the launch path)
    std::mutex tbl_mu;
    std::vector<std::pair<size_t, void*>> tbl_free;
    void* get_table(size_t bytes, size_t* cap);
    void put_table(void* p, size_t cap);
    // event pool
    std::mutex ev_mu;
    std::vector<cudaEvent_t> ev_free;
    cudaEvent_t get_event();
    void put_event(cudaEvent_t e);
    // stats
    std::atomic<int> active_jobs{0};  // submitted and not yet complete
    std::atomic<uint64_t> kernels_launched{0}, bytes_d2h{0}, bytes_h2d{0}, bytes_written{0}, bytes_read{0};
};

namespace tsnap {

struct FileSpec {
    std::string path;
    uint64_t offset = 0;  // load: first byte of the range inside the file
    uint64_t nbytes = 0;
    std::vector<tsnap_copy_desc> members;
    bool host_only = false;  // every member lives in HOST space
    bool mixed = false;      // a memory sink with HOST and DEVICE members
    bool dense = false;      // every device member is one dense, cast-free run: can be drained without staging
    bool direct = false;     // chosen for this job: D2H straight from the live tensors (no arena, no pack)
    // Device members on the wire: offset, tensor-side address of a dense run (else 0), length.  Save records every
    // device member's whole extent (quantisation trailer, per-channel header and parameters included); load only
    // the dense runs.  A direct file copies its runs one by one; a mixed sink copies back only these extents.
    struct Seg {
        uint64_t off, addr, bytes;
    };
    std::vector<Seg> segs;
    int fd = -1;
    bool opened = false, open_failed = false, direct_io = false;
    std::mutex open_mu;
    std::atomic<int64_t> parts_left{0};  // I/O parts not yet finished: the last one closes the file
    uint64_t arena_off = 0;  // offset inside the wave's arena region
    int wave = -1;
    int index = -1;                 // position in the job's files (trace records)
    const char* mem_src = nullptr;  // load: the "file" is caller memory (consumer seam)
    char* mem_dst = nullptr;        // save: the "file" is this pinned host buffer (stager seam)
};

struct Wave {
    std::vector<int> files;
    bool direct = false;      // pseudo-wave of direct files: no kernels, no arena region
    uint64_t bytes = 0;       // arena bytes (256B-aligned file regions)
    uint64_t region_off = 0;  // offset of the region inside the arena
    std::vector<Member> members;
    std::vector<Tile> tiles[kKernelCount];  // per kernel (kernels.h)
    std::vector<TmaPair> tmaps;  // tensor maps of the tensor-map kernels' members (Member.q_zero_point indexes this table)
    std::vector<QChannel> qch;   // parameters of the kModeQChannel members (Member.q_zero_point indexes this table)
    uint64_t qkey_bytes = 0;     // save: the key slots of all qch entries (QChannel.keys, filled in by launch_wave)
    void* d_tables = nullptr;
    size_t table_bytes = 0, table_cap = 0;
    cudaEvent_t ev_bucket[kBucketCount + 1] = {};  // kernel timing: bucket b runs between ev_bucket[b] and ev_bucket[b + 1]
    bool timed = false;
    double kernel_ms = 0;
    cudaEvent_t ev_done = nullptr;                                    // kernels finished
    cudaEvent_t ev_copied = nullptr;                                  // all payload copies of the wave finished
    std::atomic<int64_t> chunks_to_upload{0};                         // load: H2D chunks not yet issued
};

enum JobKind { kSave = 0, kLoad = 1 };

}  // namespace tsnap

struct tsnap_job {
    tsnap_engine* eng = nullptr;
    int kind = tsnap::kSave;
    std::deque<tsnap::FileSpec> files;
    std::deque<tsnap::Wave> waves;   // staged waves first, then at most one direct pseudo-wave
    size_t n_staged_waves = 0;
    cudaEvent_t ev_producer = nullptr;
    cudaEvent_t ev_copy_begin = nullptr, ev_copy_end = nullptr;  // timing of the payload D2H span
    void* consumer_stream = nullptr;
    bool submitted = false;
    bool holds_arena = false;  // released in part_done when the job completes
    // HBM staging of this job: lent by the caller (tsnap_job_set_arena) or the engine's own
    char* arena = nullptr;
    uint64_t arena_bytes = 0;
    bool arena_set = false;   // caller supplied one (possibly of 0 bytes = arena-less)
    cudaEvent_t ev_consumer = nullptr;  // load: recorded on the consumer stream at submit
    // timeline (TSNAP_ENGINE_TRACE)
    std::mutex trace_mu;
    std::vector<tsnap_trace_rec> trace;
    double last_copy_done_ms = 0;  // completion thread only
    void add_trace(int kind, int lane, int file, double t0, double t1, uint64_t bytes);
    double now_ms() const { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_submit).count(); }
    // completion state
    std::mutex mu;
    std::condition_variable cv;
    bool device_done = false;
    bool done = false;
    int err_code = 0;
    std::string err_msg;
    // outstanding work: the drain thread's token (set at submit) plus one part per task handed out and not yet
    // finished.  A task is handed out only by a holder of a part, so the count reaches zero once, when all is done.
    std::atomic<int64_t> parts_left{0};
    // per-channel descriptors: the job's own copies of their tsnap_qchannel records (the caller's are only read during
    // add_member), and the host-mapped word the parameter kernel raises on a NaN / Inf channel
    std::deque<tsnap_qchannel> qrecs;
    int* qflag = nullptr;
    // stats
    tsnap_job_stats stats{};
    bool timing_collected = false;
    std::atomic<int64_t> slot_wait_us{0}, io_busy_us{0}, io_queue_us{0}, n_memcpy{0}, link_starved_us{0};
    std::atomic<int> copies_in_flight{0};  // payload chunks issued on s_copy and not yet retired
    // host-memory budget: ring slots this job may hold at once (0 = unlimited)
    int max_slots = 0;
    int slots_held = 0, slots_peak = 0;
    std::mutex slot_mu;
    std::condition_variable slot_cv;
    char* take_slot();             // blocks on the budget, then on the ring
    void give_slot(char* p);
    std::chrono::steady_clock::time_point t_submit;

    void fail(int code, const std::string& msg);
    bool failed();
    void hold() { parts_left.fetch_add(1, std::memory_order_relaxed); }
    void part_done();
};

// stager seam: a save job whose one file is a pinned block of the pin cache
struct tsnap_buffer {
    tsnap_job* job;
    char* stage_buf;
    size_t stage_cap;
};
