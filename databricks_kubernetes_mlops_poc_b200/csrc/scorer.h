/*
 * scorer.h -- the columnar request pipeline behind `model.predict(DataFrame)`: columns in, probabilities out, ONE C call to
 * start it and one per chunk to collect it (included by b2f_api.cu; host code, no kernels of its own).
 *
 * Reference counterpart: everything between `pd.DataFrame(data)` and `.tolist()` around the classifier call
 * (reference app/main.py:54-72, databricks/src/02-register-model.ipynb:330-337) -- pandas column selection, SimpleImputer /
 * OneHotEncoder lookups, the float32 cast, the tree walk.  Here a request is cut into chunks and every chunk flows through
 *
 *     encode (worker threads: Arrow string buffers + float64 columns -> encoded rows, straight into a pinned staging buffer)
 *       -> cudaMemcpyAsync H2D -> fused scoring kernel -> cudaMemcpyAsync D2H (pinned results)        [issued by the worker
 *          that finished the chunk's last part, on one of the model's streams]
 *
 * so chunk c+1 is being encoded while chunk c crosses PCIe and is scored, and the caller can consume chunk c (build its
 * Python floats) while the rest is still in flight.  Worker threads are created once per scorer, bound to the CPUs of the
 * GPU's NUMA node (sysfs: /sys/bus/pci/devices/<bdf>/numa_node), and the pinned staging is allocated from one of them so the
 * pages are local to the PCIe root the copies leave from.
 */
#pragma once
#include <pthread.h>
#include <sched.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <mutex>

/* ------------------------------------------------------------------ NUMA placement (no libnuma in the image: sysfs + affinity) */
static bool numa_cpus_of_device(int device, cpu_set_t *set) {
    char bdf[32] = "";
    if (cudaDeviceGetPCIBusId(bdf, sizeof(bdf), device) != cudaSuccess) return false;
    for (char *c = bdf; *c; ++c) *c = (char)tolower(*c);
    char path[128];
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bdf);
    FILE *f = fopen(path, "r");
    if (!f) return false;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    if (node < 0) return false;
    snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
    f = fopen(path, "r");
    if (!f) return false;
    char list[1024] = "";
    if (!fgets(list, sizeof(list), f)) list[0] = 0;
    fclose(f);
    cpu_set_t allowed;
    CPU_ZERO(&allowed);
    if (sched_getaffinity(0, sizeof(allowed), &allowed) != 0) return false;
    CPU_ZERO(set);
    int n = 0;
    for (const char *p = list; *p;) {
        while (*p == ',' || *p == ' ' || *p == '\n') ++p;
        if (!*p) break;
        char *end;
        long a = strtol(p, &end, 10), b = a;
        if (end == p) break;
        p = end;
        if (*p == '-') {
            b = strtol(p + 1, &end, 10);
            p = end;
        }
        for (long c = a; c <= b && c < CPU_SETSIZE; ++c)
            if (CPU_ISSET((int)c, &allowed)) {
                CPU_SET((int)c, set);
                ++n;
            }
    }
    return n > 0;
}

static void bind_thread_near(int device) {
    static const bool off = getenv("B2F_NO_NUMA") != nullptr;
    cpu_set_t set;
    if (!off && numa_cpus_of_device(device, &set)) pthread_setaffinity_np(pthread_self(), sizeof(set), &set);
}

/* CPUs this process may actually burn: the cgroup's CFS bandwidth (v2 cpu.max "quota period", v1 cpu.cfs_quota_us /
 * cpu.cfs_period_us) next to its affinity mask.  A pool of polling workers larger than the quota gets the WHOLE cgroup
 * throttled for the rest of the 100 ms period, and the request that was running waits for it (tools/e2e_stalls.py shows it).
 * 0 = no limit found. */
static double cgroup_cpu_limit() {
    double best = 0.0;
    if (FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
        char q[32] = "";
        long long period = 0;
        if (fscanf(f, "%31s %lld", q, &period) == 2 && strcmp(q, "max") != 0 && period > 0) best = (double)atoll(q) / (double)period;
        fclose(f);
    }
    if (best <= 0.0) {
        long long quota = -1, period = 0;
        if (FILE *f = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r")) {
            if (fscanf(f, "%lld", &quota) != 1) quota = -1;
            fclose(f);
        }
        if (FILE *f = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r")) {
            if (fscanf(f, "%lld", &period) != 1) period = 0;
            fclose(f);
        }
        if (quota > 0 && period > 0) best = (double)quota / (double)period;
    }
    return best;
}

/* worker threads a scorer may start by default: the GPU's NUMA node (its cores and half of their hyper-threads), capped at 48
 * and at the cgroup's CPU bandwidth minus two (the caller's thread builds the response while the workers encode; more polling
 * workers than the quota allows get the whole cgroup throttled, and the request in flight stalls for the rest of the period) */
static int default_host_threads(int device) {
    cpu_set_t set;
    int local = numa_cpus_of_device(device, &set) ? CPU_COUNT(&set) : (int)std::thread::hardware_concurrency();
    int threads = std::max(1, std::min(48, local * 3 / 4));
    const double lim = cgroup_cpu_limit();
    if (lim > 0.0) threads = std::max(1, std::min(threads, (int)lim - 2));
    return threads;
}

/* bind the CALLING thread to the CPUs of a GPU's NUMA node (threads it creates afterwards inherit the mask; memory it touches
 * first lands on that node).  For a process that serves one GPU: call it before building the request data, so that the
 * DataFrame the encoder threads read, the Python heap the response is built in and the pinned staging all sit on the GPU's
 * socket.  Returns the number of CPUs bound to, 0 when the topology is not exposed (nothing changed). */
extern "C" int b2f_bind_caller_near(int device) {
    cpu_set_t set;
    if (!numa_cpus_of_device(device, &set)) return 0;
    if (pthread_setaffinity_np(pthread_self(), sizeof(set), &set) != 0) return 0;
    return CPU_COUNT(&set);
}

/* NUMA node of a GPU (sysfs numa_node of its PCI device), -1 when the topology is not exposed; *n_cpus = logical CPUs of that
 * node this process may run on */
extern "C" int b2f_device_numa_node(int device, int *n_cpus) {
    if (n_cpus) *n_cpus = 0;
    char bdf[32] = "";
    if (cudaDeviceGetPCIBusId(bdf, sizeof(bdf), device) != cudaSuccess) return -1;
    for (char *c = bdf; *c; ++c) *c = (char)tolower(*c);
    char path[128];
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bdf);
    int node = -1;
    if (FILE *f = fopen(path, "r")) {
        if (fscanf(f, "%d", &node) != 1) node = -1;
        fclose(f);
    }
    cpu_set_t set;
    if (node >= 0 && n_cpus && numa_cpus_of_device(device, &set)) *n_cpus = CPU_COUNT(&set);
    return node;
}

extern "C" double b2f_host_cpu_limit(void) { return cgroup_cpu_limit(); }
extern "C" int b2f_host_threads_default(int device) { return default_host_threads(device); }

/* page-locked host memory whose pages sit on the GPU's NUMA node: allocated from a thread bound to that node's CPUs */
static void *pinned_alloc_near(int device, size_t nbytes) {
    void *p = nullptr;
    cudaError_t err = cudaSuccess;
    static const bool off = getenv("B2F_NO_NUMA") != nullptr;
    std::thread t([&] {
        cpu_set_t set;
        if (!off && numa_cpus_of_device(device, &set)) pthread_setaffinity_np(pthread_self(), sizeof(set), &set);
        cudaSetDevice(device);
        err = cudaHostAlloc(&p, nbytes ? nbytes : 1, cudaHostAllocPortable);
        if (err == cudaSuccess && nbytes) memset(p, 0, nbytes); /* first touch from the bound thread */
    });
    t.join();
    if (err != cudaSuccess) {
        set_err(B2F_ENOMEM, "cudaHostAlloc(%zu) failed: %s", nbytes, cudaGetErrorString(err));
        return nullptr;
    }
    return p;
}

extern "C" void *b2f_pinned_alloc_near(int device, size_t nbytes) { return pinned_alloc_near(device, nbytes); }

/* One buffer for a stream that is dealt round-robin over several GPUs (b2f_predict_stream): stripe s = bytes
 * [s * stripe_bytes, (s + 1) * stripe_bytes) is the part GPU (s mod n) will copy, so its pages are first-touched from a thread
 * bound to THAT GPU's NUMA node, and only then is the whole range page-locked (cudaHostRegister keeps pages where they are).
 * A single cudaHostAlloc puts everything on the allocating thread's node, and the GPUs of the other socket then copy across the
 * socket interconnect. */
#include <sys/mman.h>
#include <map>
static std::mutex g_striped_mu;
static std::map<void *, size_t> g_striped;

extern "C" void *b2f_pinned_alloc_striped(b2f_model **models, int n_models, size_t stripe_bytes, size_t total_bytes) {
    if (!models || n_models <= 0 || stripe_bytes == 0 || total_bytes == 0) {
        set_err(B2F_EINVAL, "bad argument");
        return nullptr;
    }
    const size_t page = 4096, len = (total_bytes + page - 1) / page * page;
    void *p = mmap(nullptr, len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (p == MAP_FAILED) {
        set_err(B2F_ENOMEM, "mmap(%zu) failed", len);
        return nullptr;
    }
    static const bool off = getenv("B2F_NO_NUMA") != nullptr;
    std::vector<std::thread> th;
    for (int d = 0; d < n_models; ++d)
        th.emplace_back([=] {
            cpu_set_t set;
            if (!off && numa_cpus_of_device(models[d]->device, &set)) pthread_setaffinity_np(pthread_self(), sizeof(set), &set);
            uint8_t *b = static_cast<uint8_t *>(p);
            for (size_t s = (size_t)d * stripe_bytes; s < total_bytes; s += (size_t)n_models * stripe_bytes) {
                const size_t lo = (s + page - 1) / page * page; /* a page shared by two stripes belongs to the earlier one */
                const size_t hi = std::min(total_bytes, s + stripe_bytes);
                if (s == 0 || lo < hi)
                    for (size_t o = (s == 0 ? 0 : lo); o < hi; o += page) b[o] = 0; /* first touch */
            }
        });
    for (auto &t : th) t.join();
    cudaSetDevice(models[0]->device);
    cudaError_t e = cudaHostRegister(p, len, cudaHostRegisterPortable);
    if (e != cudaSuccess) {
        munmap(p, len);
        set_err(B2F_ENOMEM, "cudaHostRegister(%zu) failed: %s", len, cudaGetErrorString(e));
        return nullptr;
    }
    std::lock_guard<std::mutex> lk(g_striped_mu);
    g_striped[p] = len;
    return p;
}

extern "C" void b2f_pinned_free_striped(void *p) {
    if (!p) return;
    size_t len = 0;
    {
        std::lock_guard<std::mutex> lk(g_striped_mu);
        auto it = g_striped.find(p);
        if (it == g_striped.end()) return;
        len = it->second;
        g_striped.erase(it);
    }
    cudaHostUnregister(p);
    munmap(p, len);
}

/* ------------------------------------------------------------------ scorer */
#define B2F_SCORER_MAX_CHUNKS 64

struct b2f_scorer {
    b2f_model *m = nullptr;
    const b2f_encoder *e = nullptr;
    int n_threads = 0;
    std::vector<std::thread> workers;
    std::mutex mu;              /* job hand-over + CUDA submission (the model's slots are single-threaded) */
    std::condition_variable cv; /* workers sleep here between jobs */
    std::atomic<uint64_t> generation{0};
    bool stop = false;
    int spin_us = 1500; /* how long an idle worker polls for the next job before it sleeps (B200_SPIN_US) */
    /* pinned staging, grown on demand */
    uint8_t *h_rows = nullptr;
    uint8_t *h_out = nullptr;
    int64_t cap_rows = 0;
    /* current job */
    int64_t n = 0, chunk_rows = 0;
    int64_t chunk_lo[B2F_SCORER_MAX_CHUNKS + 1] = {}; /* chunk c = rows [chunk_lo[c], chunk_lo[c + 1]) */
    int n_chunks = 0, parts_per_chunk = 1;
    int row_format = 0;
    HostJob job{}; /* score_job of the output kind */
    const b2f_str_column *cats = nullptr;
    const double *const *nums = nullptr;
    const int64_t *strides = nullptr;
    std::atomic<int> next_item{0};
    std::atomic<int> items_done{0};
    std::atomic<int> parts_left[B2F_SCORER_MAX_CHUNKS];
    std::atomic<int> chunk_state[B2F_SCORER_MAX_CHUNKS]; /* 0 = encoding, 1 = submitted to the GPU, < 0 = error code */
    std::atomic<int> bad_range{0};
    cudaEvent_t ev[B2F_SCORER_MAX_CHUNKS] = {};
    char err[256] = "";
    int64_t jobs = 0;
    /* timeline of the current job (b2f_scorer_trace), microseconds since b2f_scorer_start: per chunk, when its last part was
     * encoded (submission begins) and when its H2D / kernel / D2H had been enqueued */
    std::chrono::steady_clock::time_point t_start;
    double t_encoded[B2F_SCORER_MAX_CHUNKS] = {}, t_enqueued[B2F_SCORER_MAX_CHUNKS] = {};
};

static inline double scorer_us_since(const b2f_scorer *s) {
    return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - s->t_start).count();
}

static void scorer_submit_chunk(b2f_scorer *s, int c) {
    /* H2D -> kernel(s) -> D2H for chunk c on the stream of slot (c mod streams); called by the worker that finished it */
    b2f_model *m = s->m;
    const int64_t lo = s->chunk_lo[c], cnt = s->chunk_lo[c + 1] - lo;
    int rc = B2F_OK;
    s->t_encoded[c] = scorer_us_since(s);
    if (cnt <= 0) { /* cannot happen with the boundaries b2f_scorer_start computes; never hand CUDA an empty chunk */
        s->t_enqueued[c] = s->t_encoded[c];
        s->chunk_state[c].store(1, std::memory_order_release);
        return;
    }
    {
        std::lock_guard<std::mutex> lk(s->mu);
        Slot &sl = m->slots[c % B2F_STREAMS];
        rc = submit_chunk(m, sl, s->job, s->h_rows, s->row_format, s->h_out, nullptr, lo, cnt, nullptr);
        const cudaError_t e = rc == B2F_OK ? cudaEventRecord(s->ev[c], sl.stream) : cudaSuccess;
        if (e != cudaSuccess) {
            snprintf(s->err, sizeof(s->err), "CUDA error while submitting chunk %d: %s", c, cudaGetErrorString(e));
            rc = B2F_ECUDA;
        } else if (rc != B2F_OK) {
            snprintf(s->err, sizeof(s->err), "%s", b2f_last_error());
        }
    }
    s->t_enqueued[c] = scorer_us_since(s);
    s->chunk_state[c].store(rc == B2F_OK ? 1 : rc, std::memory_order_release);
}

/* take one (chunk, part) item, encode it, submit the chunk if it was its last part; false when every item is handed out */
static bool scorer_work_one(b2f_scorer *s) {
    const int n_items = s->n_chunks * s->parts_per_chunk;
    const int it = s->next_item.fetch_add(1, std::memory_order_relaxed);
    if (it >= n_items) return false;
    const int c = it / s->parts_per_chunk, part = it % s->parts_per_chunk; /* items go out in order: chunk 0 completes first */
    const int64_t c_lo = s->chunk_lo[c], c_cnt = s->chunk_lo[c + 1] - c_lo;
    const int64_t lo = c_lo + c_cnt * part / s->parts_per_chunk, hi = c_lo + c_cnt * (part + 1) / s->parts_per_chunk;
    if (hi > lo && enc_range(s->e, lo, hi, s->cats, s->nums, s->strides, s->row_format, reinterpret_cast<uint32_t *>(s->h_rows))) s->bad_range.store(1);
    if (s->parts_left[c].fetch_sub(1, std::memory_order_acq_rel) == 1) scorer_submit_chunk(s, c);
    s->items_done.fetch_add(1, std::memory_order_release);
    return true;
}
static void scorer_work(b2f_scorer *s) {
    while (scorer_work_one(s)) {
    }
}

static void scorer_worker(b2f_scorer *s, int idx) {
    static const bool off = getenv("B2F_NO_NUMA") != nullptr;
    cpu_set_t set;
    if (!off && numa_cpus_of_device(s->m->device, &set)) pthread_setaffinity_np(pthread_self(), sizeof(set), &set);
    cudaSetDevice(s->m->device);
    uint64_t seen = 0;
    for (;;) {
        /* spin for the next job for a while (a service under load gets the next request within a millisecond; waking 30
         * sleeping threads through a condition variable delays the request that does it), then sleep */
        uint64_t g = s->generation.load(std::memory_order_acquire);
        if (g == seen) {
            const auto until = std::chrono::steady_clock::now() + std::chrono::microseconds(s->spin_us);
            for (int spin = 0; g == seen; ++spin) {
                __builtin_ia32_pause();
                g = s->generation.load(std::memory_order_acquire);
                if ((spin & 255) == 255 && std::chrono::steady_clock::now() > until) break;
            }
        }
        if (g == seen) {
            std::unique_lock<std::mutex> lk(s->mu);
            s->cv.wait(lk, [&] { return s->stop || s->generation.load(std::memory_order_acquire) != seen; });
            if (s->stop) return;
            g = s->generation.load(std::memory_order_acquire);
        }
        if (s->stop) return;
        seen = g;
        scorer_work(s);
    }
}

extern "C" b2f_scorer *b2f_scorer_create(b2f_model *m, const b2f_encoder *e, int threads) {
    if (!m || !e) {
        set_err(B2F_EINVAL, "null argument");
        return nullptr;
    }
    if ((int)m->hdr.n_cat != e->n_cat || (int)m->hdr.n_num != e->n_num) {
        set_err(B2F_EINVAL, "encoder schema (%d, %d) differs from the model's (%u, %u)", e->n_cat, e->n_num, m->hdr.n_cat, m->hdr.n_num);
        return nullptr;
    }
    b2f_scorer *s = new (std::nothrow) b2f_scorer();
    if (!s) return nullptr;
    s->m = m;
    s->e = e;
    if (threads <= 0) {
        threads = default_host_threads(m->device);
    }
    s->n_threads = std::min(threads, 64);
    if (const char *sp = getenv("B200_SPIN_US")) s->spin_us = std::max(0, atoi(sp));
    cudaSetDevice(m->device);
    for (auto &e2 : s->ev)
        if (cudaEventCreateWithFlags(&e2, cudaEventDisableTiming) != cudaSuccess) {
            set_err(B2F_ECUDA, "cudaEventCreate failed");
            delete s;
            return nullptr;
        }
    for (int i = 0; i < s->n_threads - 1; ++i) s->workers.emplace_back(scorer_worker, s, i); /* the caller's thread is the last worker */
    return s;
}

extern "C" void b2f_scorer_destroy(b2f_scorer *s) {
    if (!s) return;
    {
        std::lock_guard<std::mutex> lk(s->mu);
        s->stop = true;
        s->generation.fetch_add(1);
    }
    s->cv.notify_all();
    for (auto &t : s->workers) t.join();
    cudaSetDevice(s->m->device);
    for (auto &e : s->ev)
        if (e) cudaEventDestroy(e);
    if (s->h_rows) cudaFreeHost(s->h_rows);
    if (s->h_out) cudaFreeHost(s->h_out);
    delete s;
}

/* Start scoring n rows given as columns (same column arguments as b2f_encoder_encode).
 *   row_format : what the rows are encoded as on their way to the GPU (B2F_ROWS_RANKED / PACKED64 / WORDS24)
 *   out_mode   : B2F_OUT_F32, B2F_OUT_F64 or B2F_OUT_FULL (b2f_scored_full records: needs an attached outlier forest)
 *   chunk_rows : rows per pipeline chunk (0 = choose: ~8 chunks for large requests)
 * Returns the number of chunks (>= 0) or a negative error.  Results appear in the scorer's pinned result buffer
 * (b2f_scorer_results) chunk by chunk; b2f_scorer_wait(chunk) blocks until that chunk is there.  The column buffers must stay
 * valid until the last chunk has been waited for.  One job at a time per scorer. */
/* out[2 c] / out[2 c + 1]: microseconds from b2f_scorer_start to "chunk c encoded" / "chunk c's GPU work enqueued" (last job) */
extern "C" int b2f_scorer_trace(const b2f_scorer *s, double *out, int max_chunks) {
    if (!s || !out) return 0;
    const int nc = std::min(s->n_chunks, max_chunks);
    for (int c = 0; c < nc; ++c) {
        out[2 * c] = s->t_encoded[c];
        out[2 * c + 1] = s->t_enqueued[c];
    }
    return nc;
}

extern "C" int b2f_scorer_start(b2f_scorer *s, int64_t n, const b2f_str_column *cat_cols, const double *const *num_cols, const int64_t *num_strides,
                                int row_format, int out_mode, int64_t chunk_rows) {
    if (!s || n < 0) return set_err(B2F_EINVAL, "bad argument");
    if (out_mode == B2F_OUT_PAIRS) return set_err(B2F_EINVAL, "out_mode must be B2F_OUT_F32, B2F_OUT_F64 or B2F_OUT_FULL");
    int rcf = check_row_format(s->m, row_format);
    if (rcf) return rcf;
    if (row_format == B2F_ROWS_RANKED && !s->e->ranker) return set_err(B2F_ESTATE, "the encoder has no ranker attached (b2f_encoder_attach_ranker)");
    if (row_format == B2F_ROWS_PACKED64 && !s->e->packed_ok) return set_err(B2F_EINVAL, "schema does not fit the packed row");
    rcf = out_check(s->m, out_mode, row_format, true); /* the results go to the scorer's own buffer */
    if (rcf) return rcf;
    if (n == 0) {
        s->n = 0;
        s->n_chunks = 0;
        return 0;
    }
    const bool auto_chunks = chunk_rows <= 0;
    if (chunk_rows <= 0) {
        chunk_rows = n <= 8192 ? n : std::max<int64_t>(4096, ((n + 7) / 8 + 255) / 256 * 256);
        /* a forest that STREAMS through shared memory (500 trees x depth 8) makes the GPU the bound of a big request, and its
         * tile kernel -- one pass over the forest per launch -- wants >= 24 576 rows per launch: two chunks instead of eight
         * (resident forests keep eight: each pass over the forest is cheap, so overlap of copies and kernels wins) */
        const bool streamed = s->m->tile_ok && s->m->tp.n_pieces > s->m->tp.n_slots;
        if (streamed && row_format != B2F_ROWS_RANKED && n >= 2 * s->m->tile_min_rows)
            chunk_rows = std::max<int64_t>(s->m->tile_min_rows, ((n + 1) / 2 + 255) / 256 * 256);
    }
    int n_chunks = (int)((n + chunk_rows - 1) / chunk_rows);
    if (n_chunks > B2F_SCORER_MAX_CHUNKS) {
        chunk_rows = ((n + B2F_SCORER_MAX_CHUNKS - 1) / B2F_SCORER_MAX_CHUNKS + 255) / 256 * 256;
        n_chunks = (int)((n + chunk_rows - 1) / chunk_rows);
    }
    /* chunk boundaries: equal chunks.  B200_FIRST_CHUNK_ROWS=<r> makes the first chunk of a library-chunked request r rows
     * (the caller turns results into Python objects more slowly than the pool encodes, so the request ends one list-building
     * time after the FIRST chunk is back).  A small first chunk pays only when its launch and copies cost less than
     * encoding the rows it saves, which is not the case for the default 8 192-row chunks -- so it is off by default (a choice
     * kept from the previous GPU generation, not re-measured on the H100) */
    static const int64_t first_rows = getenv("B200_FIRST_CHUNK_ROWS") ? atoll(getenv("B200_FIRST_CHUNK_ROWS")) : 0;
    if (auto_chunks && n_chunks >= 4 && first_rows >= 256 && first_rows * 4 <= chunk_rows * 2) {
        const int64_t rest = n - first_rows, each = ((rest + (n_chunks - 2)) / (n_chunks - 1) + 255) / 256 * 256;
        s->chunk_lo[0] = 0;
        for (int c = 1; c <= n_chunks; ++c) s->chunk_lo[c] = std::min(n, first_rows + (int64_t)(c - 1) * each);
        s->chunk_lo[n_chunks] = n;
    } else {
        for (int c = 0; c <= n_chunks; ++c) s->chunk_lo[c] = std::min(n, (int64_t)c * chunk_rows);
    }
    CUDA_TRY(cudaSetDevice(s->m->device));
    if (n > s->cap_rows) {
        if (s->h_rows) cudaFreeHost(s->h_rows);
        if (s->h_out) cudaFreeHost(s->h_out);
        s->h_rows = s->h_out = nullptr;
        s->cap_rows = 0;
        const int64_t cap = std::max<int64_t>(n + n / 2, 4096);
        s->h_rows = static_cast<uint8_t *>(pinned_alloc_near(s->m->device, (size_t)cap * B2F_ROW_BYTES));
        s->h_out = static_cast<uint8_t *>(pinned_alloc_near(s->m->device, (size_t)cap * sizeof(b2f_scored_full)));
        if (!s->h_rows || !s->h_out) return B2F_ENOMEM;
        s->cap_rows = cap;
    }
    s->n = n;
    s->chunk_rows = chunk_rows;
    s->n_chunks = n_chunks;
    s->row_format = row_format;
    s->job = score_job(out_mode);
    s->cats = cat_cols;
    s->nums = num_cols;
    s->strides = num_strides;
    s->parts_per_chunk = (int)std::max<int64_t>(1, std::min<int64_t>(s->n_threads, chunk_rows / 512));
    for (int c = 0; c < n_chunks; ++c) {
        s->parts_left[c].store(s->parts_per_chunk);
        s->chunk_state[c].store(0);
    }
    s->bad_range.store(0);
    s->items_done.store(0);
    s->next_item.store(0);
    s->err[0] = 0;
    s->jobs++;
    s->t_start = std::chrono::steady_clock::now();
    {
        std::lock_guard<std::mutex> lk(s->mu);
        s->generation.fetch_add(1, std::memory_order_release);
    }
    if (n_chunks * s->parts_per_chunk > 1) s->cv.notify_all();
    return n_chunks;
}

/* Block until chunk `chunk` of the current job is in the result buffer.  The calling thread helps with the encoding while it
 * waits (it is the pool's last worker), so a scorer with one thread is simply synchronous. */
extern "C" int b2f_scorer_wait(b2f_scorer *s, int chunk) {
    if (!s || chunk < 0 || chunk >= s->n_chunks) return set_err(B2F_EINVAL, "bad chunk index");
    /* the caller's thread helps with the encoding only while ITS chunk is not on the GPU yet -- then it goes back to the caller,
     * who has the previous chunk's Python objects to build while the workers carry on */
    int st;
    while ((st = s->chunk_state[chunk].load(std::memory_order_acquire)) == 0)
        if (!scorer_work_one(s)) __builtin_ia32_pause();
    if (st < 0) return set_err(st, "%s", s->err);
    CUDA_TRY(cudaSetDevice(s->m->device));
    CUDA_TRY(cudaEventSynchronize(s->ev[chunk]));
    if (chunk == s->n_chunks - 1) {
        /* the job is over once every worker has left the item loop: only then may the caller free the columns / start again */
        const int n_items = s->n_chunks * s->parts_per_chunk;
        while (s->items_done.load(std::memory_order_acquire) < n_items) __builtin_ia32_pause();
        if (s->bad_range.load()) return set_err(B2F_ERANGE, "a numeric input is infinite or too large for float32");
    }
    return B2F_OK;
}

extern "C" const void *b2f_scorer_results(const b2f_scorer *s) { return s ? s->h_out : nullptr; }
extern "C" int64_t b2f_scorer_chunk_rows(const b2f_scorer *s) { return s ? s->chunk_rows : 0; }
/* rows [*lo, *lo + *cnt) of the request are chunk c of the current job (chunks need not be equal: see b2f_scorer_start) */
extern "C" int b2f_scorer_chunk_range(const b2f_scorer *s, int c, int64_t *lo, int64_t *cnt) {
    if (!s || c < 0 || c >= s->n_chunks || !lo || !cnt) return set_err(B2F_EINVAL, "bad chunk index");
    *lo = s->chunk_lo[c];
    *cnt = s->chunk_lo[c + 1] - s->chunk_lo[c];
    return B2F_OK;
}
extern "C" int b2f_scorer_threads(const b2f_scorer *s) { return s ? s->n_threads : 0; }
