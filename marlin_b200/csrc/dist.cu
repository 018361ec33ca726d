// Multi-GPU BlockMatrix.multiply behind the C ABI (include/marlin_b200.h: mb_comm_*, mb_matmul_blocked_dist*).
//
// The reference replicates A tiles n times and B tiles m times through two Spark shuffles so that partition
// seq = i*n*k + j*k + kk holds exactly A(i,kk) and B(kk,j), multiplies there and sums the k partials of every C tile
// with reduceByKey (matrix/BlockMatrix.scala:159-178).  Here one process drives one GPU of an NVSwitch box:
//   * rendezvous and per-call metadata go through a POSIX shared-memory segment (one box, no network, no torch);
//   * tile replication = copy-engine PULLS over NVLink peer memory (CUDA IPC), band by band, on a side stream; the
//     persistent grouped DMMA kernel (gemm_f64.cu) starts at once and its TMA producer waits per band, so the tensor
//     cores run on whatever has landed;
//   * the reduceByKey of a C tile held as two partials (k split over two GPUs) is a REDUCE-SCATTER done by the GEMM
//     epilogues: each holder first computes the column half the OTHER one reduces, its epilogue storing straight into
//     the peer's staging buffer over NVLink, then its own half as acc + staged partial; the partner's reduced half is
//     stored, again by the epilogue, directly into the owner's C tile.  No add pass, no extra copy.  The two halves are
//     two launches of the same persistent kernel with the exchange flags between them, written by stream memory
//     operations at the kernel boundary: completion counted inside a kernel whose epilogue stores to peer memory was
//     measured faulty;
//   * anything else (three or more holders, bf16 / transposed tiles) takes the staged path: partials are stored into
//     a per-source slot of the owner's staging buffer and the owner adds them in rank order (deterministic).
// Processes are ordered by monotonic epoch flags in exported device memory, written and awaited by stream memory
// operations (cuStreamWriteValue64 / cuStreamWaitValue64) or polled inside the GEMM (ld.acquire).  In-kernel waits are
// bounded (MARLIN_B200_TIMEOUT_S, default 120 s); stream-side waits cannot time out on the device, so every host-side
// synchronisation is bounded instead and, on expiry, releases the queued waits (abort_local) and reports MB_ERR_TIMEOUT.
#include "internal.h"
#include "elementwise.h"
#include "gemm_f64.h"

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <time.h>
#include <unistd.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <new>
#include <string>
#include <vector>

namespace {

constexpr int MAXW = 16;              // ranks per box
constexpr int RING = 4;               // mailboxes per rank (epoch % RING); see publish()
constexpr int MAX_PUB = 448;          // tiles one rank can publish per call
constexpr int MAX_BANDS = 4;          // readiness bands per operand tile
constexpr int MAX_PAIR = 8;           // fused C tiles per (rank, peer) pair and call

// ---- device flag words (uint64).  [0, EXPORTED) is written by peers, the rest is local to the GPU ----
constexpr int CH_READY = 0, CH_DONE = 1, CH_PARTIAL = 2, CH_FREE = 3;
constexpr int F_CH = 0;                               // [channel][src]            4 x MAXW
constexpr int F_PART2 = 64;                           // [src][slot]               MAXW x MAX_PAIR  (fused: peer's half landed)
constexpr int F_FINAL2 = F_PART2 + MAXW * MAX_PAIR;   // [src][slot]               (fused: partner's reduced half is in my C tile)
constexpr int F_UPREADY = F_FINAL2 + MAXW * MAX_PAIR; // [src][tile slot][band]    host path: a band of src's uploaded tile is in its HBM
constexpr int UP_SLOTS = 8;
constexpr int SUB_SLOTS = 64;                         // host path: sub-blocks per (src -> me) pair and call
constexpr int F_SUBDONE = F_UPREADY + MAXW * UP_SLOTS * MAX_BANDS;   // [src][sub-block]   host path: src's partial of the sub-block is in my staging
constexpr int F_LOCAL = F_SUBDONE + MAXW * SUB_SLOTS;             // ---- local from here ----
constexpr int F_BAND = F_LOCAL;                       // [operand tile][band]      2 * G2_MAX_OPS * MAX_BANDS
constexpr int F_CTR = F_BAND + 2 * mb::G2_MAX_OPS * MAX_BANDS;       // done counters, one per entry
constexpr int F_SIG = F_CTR + mb::G2_MAX_ENTRIES;                    // local completion flags, one per entry
constexpr int F_STATUS = F_SIG + mb::G2_MAX_ENTRIES;
constexpr int FLAG_WORDS = F_STATUS + 8;

struct ShmEntry {
    unsigned char handle[64];
    long long offset;                 // bytes from the allocation base to element 0 of the view
    int kind, idx;                    // 0 = A(i*k+kk), 1 = B(kk*n+j), 2 = C(i*n+j)
    int rows, cols, ld, trans, dtype, pad;
};
struct ShmMailbox {
    std::atomic<unsigned long long> seq;
    int n, pad;
    ShmEntry e[MAX_PUB];
};
struct ShmRank {
    std::atomic<unsigned long long> boot_seq;
    unsigned char flags_handle[64];
    long long flags_off;
    std::atomic<unsigned long long> staging_seq;
    unsigned char staging_handle[64];
    long long staging_off;
    unsigned long long staging_bytes;
    std::atomic<unsigned long long> abort_code;
    ShmMailbox mail[RING];
};
struct Shm {
    std::atomic<unsigned int> bar_count, bar_gen;
    ShmRank r[MAXW];
};

double now_s() {
    timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return ts.tv_sec + 1e-9 * ts.tv_nsec;
}
inline size_t up256(size_t b) { return (b + 255) & ~size_t(255); }
inline int even(int x) { return (x + 1) & ~1; }

}  // namespace

struct mb_comm {
    mb_ctx* ctx = nullptr;
    int rank = 0, world = 1;
    std::string name;
    Shm* shm = nullptr;
    size_t shm_bytes = 0;
    unsigned long long* flags = nullptr;             // local flag words (device)
    unsigned long long* flags_peer[MAXW] = {};
    cudaStream_t X = nullptr, R = nullptr, G = nullptr;   // copy stream, download stream, READY stream (tiles with ready events)
    char* staging = nullptr;                         // [src][slot_bytes]
    size_t slot_bytes = 0;
    char* staging_peer[MAXW] = {};
    unsigned long long staging_gen = 0;
    char* arena = nullptr;                           // pulled tiles
    size_t arena_bytes = 0;
    unsigned long long epoch = 0;
    unsigned long long last_write_epoch[MAXW] = {};  // last epoch in which I stored into dst's staging
    cudaEvent_t ev_compute = nullptr, ev_tmp = nullptr;
    bool have_compute = false;
    cudaEvent_t ev_half[2] = {nullptr, nullptr};     // device path: the products that read arena half p have been issued
    bool have_half[2] = {false, false};
    unsigned long long* status_host = nullptr;       // pinned copy of flags[F_STATUS]
    double timeout_s = 120.0;
    bool aborted = false;                            // abort_local() ran: every later call fails
    bool remote_write_ok = true;                     // cuStreamWriteValue64 accepted a peer address (else: 8-byte copies)
    unsigned long long* ring = nullptr;              // pinned host values for the copy-based flag writes
    size_t ring_pos = 0;
};
constexpr size_t RING_SLOTS = 8192;

namespace {

inline unsigned long long* flag_ch(mb_comm* c, int on_rank, int ch, int src) { return c->flags_peer[on_rank] + F_CH + ch * MAXW + src; }
inline long long timeout_ns(const mb_comm* c) { return (long long)(c->timeout_s * 1e9); }

int32_t host_barrier(mb_comm* c) {
    Shm* s = c->shm;
    const unsigned gen = s->bar_gen.load(std::memory_order_acquire);
    if (s->bar_count.fetch_add(1, std::memory_order_acq_rel) + 1 == (unsigned)c->world) {
        s->bar_count.store(0, std::memory_order_relaxed);
        s->bar_gen.fetch_add(1, std::memory_order_release);
        return MB_OK;
    }
    const double t0 = now_s();
    while (s->bar_gen.load(std::memory_order_acquire) == gen) {
        if (now_s() - t0 > c->timeout_s) return fail(MB_ERR_TIMEOUT, "mb_comm: host barrier timed out after %.0f s (a rank died?)", c->timeout_s);
        usleep(50);
    }
    return MB_OK;
}

template <class Pred>
int32_t spin_until(mb_comm* c, Pred p, const char* what) {
    const double t0 = now_s();
    int spins = 0;
    while (!p()) {
        if (++spins > 2000) usleep(20);
        if (now_s() - t0 > c->timeout_s) return fail(MB_ERR_TIMEOUT, "mb_comm: timed out waiting for %s after %.0f s", what, c->timeout_s);
    }
    return MB_OK;
}

// Flag writes and stream-side waits are STREAM MEMORY OPERATIONS (cuStreamWriteValue64 / cuStreamWaitValue64), executed
// by the front end in stream order — never kernels: a kernel that becomes runnable while the persistent GEMM holds every
// SM may not be scheduled until that GEMM retires (scripts/probe_copy_under_persistent.cu), and the GEMM may be waiting for
// exactly that flag.  Copies (copy engines) and memory operations are the only things the resident GEMM ever waits for.
// Writes to a peer's flag word fall back to an 8-byte copy if the driver refuses memory operations on peer addresses.
cudaError_t sig(mb_comm* c, unsigned long long* flag, unsigned long long v, cudaStream_t st) {
    const bool local = flag >= c->flags && flag < c->flags + FLAG_WORDS;
    if (local || c->remote_write_ok) {
        cudaError_t e = mb::stream_write64(flag, v, st);
        if (e == cudaSuccess || local) return e;
        c->remote_write_ok = false;
        cudaGetLastError();
    }
    unsigned long long* slot = c->ring + (c->ring_pos++ % RING_SLOTS);
    *slot = v;
    return cudaMemcpyAsync(flag, slot, 8, cudaMemcpyDefault, st);
}
// Unbounded on the device (a memory operation cannot time out); a rank that loses its peers notices at the next host-side
// rendezvous (bounded) and mb_comm_abort() releases whatever is still queued.
cudaError_t waitf(mb_comm* c, const unsigned long long* flag, unsigned long long v, cudaStream_t st) {
    (void)c;
    return mb::stream_wait64_geq(flag, v, st);
}
// Release everything this rank still has queued behind flag waits: every local flag word jumps far ahead of any epoch
// (the waits are cyclic >=), the streams drain with garbage results, the communicator is dead afterwards.
void abort_local(mb_comm* c) {
    if (c->aborted) return;
    c->aborted = true;
    cudaStream_t t = nullptr;
    if (cudaStreamCreateWithFlags(&t, cudaStreamNonBlocking) != cudaSuccess) return;
    std::vector<unsigned long long> big(FLAG_WORDS, 1ull << 62);
    cudaMemcpyAsync(c->flags, big.data(), sizeof(unsigned long long) * FLAG_WORDS, cudaMemcpyHostToDevice, t);
    cudaStreamSynchronize(t);
    cudaStreamDestroy(t);
}
// cudaStreamSynchronize with a deadline: a peer that died leaves this rank's streams parked on a memory-operation wait
// that no API call can cancel — so poll, and on timeout release the waits ourselves and report.
int32_t sync_bounded(mb_comm* c, cudaStream_t st, const char* what) {
    const double t0 = now_s();
    for (int spins = 0;; ++spins) {
        cudaError_t e = cudaStreamQuery(st);
        if (e == cudaSuccess) return MB_OK;
        if (e != cudaErrorNotReady) return cuda_fail(e, what);
        if (spins > 200) usleep(50);
        if (now_s() - t0 > c->timeout_s) {
            // post-mortem for the log: which flag words have reached the current epoch
            {
                cudaStream_t t = nullptr;
                std::vector<unsigned long long> snap(FLAG_WORDS, 0);
                if (cudaStreamCreateWithFlags(&t, cudaStreamNonBlocking) == cudaSuccess) {
                    cudaMemcpyAsync(snap.data(), c->flags, sizeof(unsigned long long) * FLAG_WORDS, cudaMemcpyDeviceToHost, t);
                    cudaStreamSynchronize(t);
                    cudaStreamDestroy(t);
                    auto dump = [&](const char* name, int base, int count) {
                        fprintf(stderr, "[marlin_b200 rank %d epoch %llu] %s:", c->rank, c->epoch, name);
                        for (int i = 0; i < count; ++i) if (snap[base + i]) fprintf(stderr, " [%d]=%llu", i, snap[base + i]);
                        fprintf(stderr, "\n");
                    };
                    dump("channels", F_CH, 4 * MAXW);
                    dump("upready", F_UPREADY, MAXW * UP_SLOTS * MAX_BANDS);
                    dump("subdone", F_SUBDONE, MAXW * SUB_SLOTS);
                    dump("band", F_BAND, 2 * mb::G2_MAX_OPS * MAX_BANDS);
                    dump("ctr", F_CTR, mb::G2_MAX_ENTRIES);
                    dump("sig", F_SIG, mb::G2_MAX_ENTRIES);
                    dump("status", F_STATUS, 8);
                    fprintf(stderr, "[marlin_b200 rank %d] stream states: S=%d X=%d R=%d U=%d (0 = idle, 600 = busy)\n", c->rank,
                            (int)cudaStreamQuery(c->ctx->stream), (int)cudaStreamQuery(c->X), (int)cudaStreamQuery(c->R),
                            c->ctx->h2d_stream ? (int)cudaStreamQuery(c->ctx->h2d_stream) : -1);
                }
            }
            abort_local(c);
            cudaStreamSynchronize(st);
            return fail(MB_ERR_TIMEOUT, "%s: no progress for %.0f s (a peer died or fell out of step); the communicator has been aborted", what,
                        c->timeout_s);
        }
    }
}

// ---------------------------------------------------------------------------------------- plan
struct MyC { int id, i, j; std::vector<int> kks; };   // a C tile (id = i*n + j) with the kk of one rank's products of it
struct Plan {
    int m, k, n, world;
    std::vector<int> prod_rank;                 // by seq = i*n*k + j*k + kk  (matrix/BlockMatrix.scala:163,168)
    std::vector<std::vector<int>> holders;      // per C tile (i*n + j): ranks holding a partial, in kk order of first appearance
    // the C tiles rank r computes partials of, in (i, j) order
    std::vector<MyC> c_tiles_of(int r) const {
        std::vector<MyC> out;
        for (int i = 0; i < m; ++i)
            for (int j = 0; j < n; ++j) {
                MyC mc{i * n + j, i, j, {}};
                for (int kk = 0; kk < k; ++kk) if (prod_rank[i * n * k + j * k + kk] == r) mc.kks.push_back(kk);
                if (!mc.kks.empty()) out.push_back(mc);
            }
        return out;
    }
};
// Products are dealt to ranks in contiguous seq ranges: the kk partials of a C tile stay on one rank whenever ranks get
// whole C tiles; with G = m*k*n this is the reference's partition -> executor identity (MatrixMultPartitioner).
inline int product_rank(int seq, int P, int world) { return P >= world ? (int)(((long long)seq * world) / P) : seq; }
Plan make_plan(int m, int k, int n, int world) {
    Plan p{m, k, n, world, {}, {}};
    const int P = m * k * n;
    p.prod_rank.resize(P);
    p.holders.resize(m * n);
    for (int i = 0; i < m; ++i)
        for (int j = 0; j < n; ++j)
            for (int kk = 0; kk < k; ++kk) {
                const int seq = i * n * k + j * k + kk, r = product_rank(seq, P, world);
                p.prod_rank[seq] = r;
                auto& h = p.holders[i * n + j];
                if (std::find(h.begin(), h.end(), r) == h.end()) h.push_back(r);
            }
    return p;
}

// Do the distinct A and B tiles that one rank's products read (its C tiles `cs`) fit the operand tables of a grouped
// launch?  The grouped launch has fixed-size tables, and whether EVERY rank's share fits is decided from the plan alone,
// so all ranks take the same path (a rank-local fallback would leave its partner waiting for flags that never come).
// Both entries run this check for every rank together with their own entry limits; the launch builders rely on it and
// fill the tables unchecked.
bool operands_fit(const Plan& p, const std::vector<MyC>& cs) {
    std::vector<char> ua(p.m * p.k, 0), ub(p.k * p.n, 0);
    int na = 0, nb = 0;
    for (const MyC& mc : cs)
        for (int kk : mc.kks) {
            if (!ua[mc.i * p.k + kk]) { ua[mc.i * p.k + kk] = 1; ++na; }
            if (!ub[kk * p.n + mc.j]) { ub[kk * p.n + mc.j] = 1; ++nb; }
        }
    return na <= mb::G2_MAX_OPS && nb <= mb::G2_MAX_OPS;
}

// Readiness bands along an operand tile's extent (A: rows, B: columns): up to `most` of them from an extent of 1024 on,
// each a multiple of 128 wide.
inline void bands_of(int extent, int most, int& band, int& nbands) {
    nbands = extent >= 1024 ? most : 1;
    band = ((extent + nbands - 1) / nbands + 127) / 128 * 128;
    nbands = (extent + band - 1) / band;
}

// Fused reduce-scatter: of a C tile N columns wide the owner reduces [0, half_cols(N)), the partner the rest.  The
// owner's half is never empty (at N = 1, N / 2 rounds to nothing): a grouped entry zero columns wide is refused.
inline int half_cols(int N) { return std::min(N, std::max(128, ((N / 2 + 127) / 128) * 128)); }

// ---------------------------------------------------------------------------------------- staging
// Per-source slots: src only ever writes [src * slot_bytes, +slot_bytes) of dst's buffer, so two sources can never
// collide whatever the sequence of plans; the FREE handshake orders a source against its OWN previous write.
int32_t ensure_staging(mb_comm* c, size_t need_slot) {
    if (need_slot <= c->slot_bytes) return MB_OK;
    // collective: every rank computes the same need from the same plan
    MB_CUDA(cudaDeviceSynchronize());
    int32_t r = host_barrier(c);
    if (r) return r;
    for (int p = 0; p < c->world; ++p)
        if (p != c->rank && c->staging_peer[p]) { mb::ipc_close(c->shm->r[p].staging_handle); c->staging_peer[p] = nullptr; }
    if ((r = host_barrier(c)) != MB_OK) return r;
    if (c->staging) { cudaFree(c->staging); c->staging = nullptr; }
    const size_t slot = up256(need_slot + need_slot / 4);
    MB_CUDA(cudaMalloc(&c->staging, slot * c->world));
    c->slot_bytes = slot;
    ShmRank& me = c->shm->r[c->rank];
    long long off = 0, bytes = 0;
    MB_CUDA(mb::ipc_export(c->staging, me.staging_handle, &off, &bytes));
    me.staging_off = off;
    me.staging_bytes = slot * c->world;
    const unsigned long long gen = ++c->staging_gen;
    me.staging_seq.store(gen, std::memory_order_release);
    if ((r = host_barrier(c)) != MB_OK) return r;
    for (int p = 0; p < c->world; ++p) {
        if (p == c->rank) { c->staging_peer[p] = c->staging; continue; }
        ShmRank& o = c->shm->r[p];
        if (o.staging_seq.load(std::memory_order_acquire) != gen) return fail(MB_ERR_INVALID_ARG, "mb_comm: staging generations differ across ranks");
        void* base = nullptr;
        MB_CUDA(mb::ipc_open_ex(o.staging_handle, &base, true));
        c->staging_peer[p] = static_cast<char*>(base) + o.staging_off;
    }
    for (int p = 0; p < c->world; ++p) c->last_write_epoch[p] = 0;
    return host_barrier(c);
}

int32_t ensure_arena(mb_comm* c, size_t bytes) {
    const cudaError_t e = grow(&c->arena, &c->arena_bytes, bytes, nullptr);
    return e == cudaSuccess ? MB_OK : cuda_fail(e, "mb_comm: arena");
}

// ---------------------------------------------------------------------------------------- metadata exchange
// Every rank writes the tiles it owns into mailbox[epoch % RING] and then reads EVERY rank's mailbox of this epoch.
// Ring safety without acknowledgements: a rank that publishes epoch e + RING has completed calls e+1 .. e+RING-1, each
// of which waited for every rank's mailbox of that epoch; a rank publishes e+1 only after it has read all of epoch e.
int32_t publish(mb_comm* c, unsigned long long e, const std::vector<ShmEntry>& mine) {
    if ((int)mine.size() > MAX_PUB) return fail(MB_ERR_UNSUPPORTED, "mb_matmul_blocked_dist: %d tiles on one rank (limit %d)", (int)mine.size(), MAX_PUB);
    ShmMailbox& mb_ = c->shm->r[c->rank].mail[e % RING];
    mb_.n = (int)mine.size();
    for (size_t i = 0; i < mine.size(); ++i) mb_.e[i] = mine[i];
    mb_.seq.store(e, std::memory_order_release);
    return MB_OK;
}
int32_t read_all(mb_comm* c, unsigned long long e, std::vector<std::vector<ShmEntry>>& out) {
    out.assign(c->world, {});
    for (int p = 0; p < c->world; ++p) {
        ShmMailbox& mb_ = c->shm->r[p].mail[e % RING];
        int32_t r = spin_until(c, [&] { return mb_.seq.load(std::memory_order_acquire) >= e; }, "a peer's tile directory");
        if (r) return r;
        if (mb_.seq.load(std::memory_order_acquire) != e)
            return fail(MB_ERR_INVALID_ARG, "mb_matmul_blocked_dist: rank %d is at call %llu, this rank at %llu (calls are collective)", p,
                        mb_.seq.load(), e);
        out[p].assign(mb_.e, mb_.e + mb_.n);
    }
    return MB_OK;
}
int32_t export_block(const mb_block* b, int kind, int idx, ShmEntry* out) {
    long long off = 0, bytes = 0;
    MB_CUDA(mb::ipc_export(b->data, out->handle, &off, &bytes));
    out->offset = off + b->offset * (long long)elem_size(b->dtype);
    out->kind = kind; out->idx = idx; out->rows = b->rows; out->cols = b->cols; out->ld = b->ld; out->trans = b->is_transpose;
    out->dtype = b->dtype; out->pad = 0;
    return MB_OK;
}
int32_t open_entry(const ShmEntry& en, char** ptr) {
    void* base = nullptr;
    MB_CUDA(mb::ipc_open(en.handle, &base));
    *ptr = static_cast<char*>(base) + en.offset;
    return MB_OK;
}

// Checks every entry runs first: the communicator, its context, the arguments (`args_ok`) and an earlier abort.
int32_t check_call(mb_comm* c, const char* who, bool args_ok) {
    if (!c) return fail(MB_ERR_INVALID_ARG, "null communicator");
    MB_CTX(c->ctx);
    if (!args_ok) return fail(MB_ERR_INVALID_ARG, "%s: bad argument", who);
    if (c->aborted) return fail(MB_ERR_TIMEOUT, "mb_comm: the communicator was aborted after a peer stopped answering");
    return MB_OK;
}

// Publish the tiles this rank offers in call e, read every rank's directory of that call, and map every peer allocation
// the directories name.
int32_t exchange_directory(mb_comm* c, unsigned long long e, const std::vector<ShmEntry>& mine, std::vector<std::vector<ShmEntry>>& dir) {
    int32_t rc = publish(c, e, mine);
    if (rc) return rc;
    if ((rc = read_all(c, e, dir)) != MB_OK) return rc;
    // Map every peer allocation this call will touch BEFORE any pointer is taken: opening a handle can evict stale
    // mappings (see ipc_open_ex), which would invalidate pointers handed out earlier in the same call.  A second pass
    // after an eviction only hits the cache.
    for (int attempt = 0; attempt < 3; ++attempt) {
        const unsigned long long gen = mb::ipc_evictions();
        char* dummy = nullptr;
        for (int p = 0; p < c->world; ++p)
            if (p != c->rank)
                for (const ShmEntry& en : dir[p])
                    if ((rc = open_entry(en, &dummy)) != MB_OK) return rc;
        if (mb::ipc_evictions() == gen) break;
    }
    return MB_OK;
}
// The directory entry of every tile of one kind, as published by the rank `owner` names (by any rank if owner is null);
// null where there is none.
std::vector<const ShmEntry*> entries_of(const std::vector<std::vector<ShmEntry>>& dir, int kind, int count, const int32_t* owner) {
    std::vector<const ShmEntry*> out(count, nullptr);
    for (size_t p = 0; p < dir.size(); ++p)
        for (const ShmEntry& en : dir[p])
            if (en.kind == kind && en.idx >= 0 && en.idx < count && (!owner || owner[en.idx] == (int)p)) out[en.idx] = &en;
    return out;
}

struct Tile {                         // an operand tile as this rank sees it during one call
    mb_block blk;                     // its local copy: the owner's block itself, or a packed copy in the arena
    int src = -1;                     // the rank it comes from: its owner (device tiles) or its uploader (host tiles)
    const ShmEntry* ent = nullptr;    // the source's directory entry, for tiles pulled from a peer
    bool need = false;                // one of this rank's products reads it
    bool remote = false;              // device tiles: pulled from a peer
    int up_slot = -1;                 // host tiles: index among the tiles its uploader uploads (F_UPREADY)
    cudaEvent_t landed = nullptr;     // device tiles: the whole tile is here (general path)
    int band = 0, nbands = 1;         // readiness bands (rows for A, columns for B); band 0 = resident, never polled
    int ready_base = -1;              // first band flag index relative to flags + F_BAND
    int op = -1;                      // operand index in the grouped launch
};

// Operand index of tile t in the A or B table of L, added on first use (operands_fit bounds the table).
int op_of(mb::G2Launch& L, Tile& t, bool is_a) {
    if (t.op >= 0) return t.op;
    int& cnt = is_a ? L.na : L.nb;
    mb::G2Operand& o = (is_a ? L.A : L.B)[cnt];
    o.ptr = f64_ptr(&t.blk); o.ld = t.blk.ld; o.rows = t.blk.rows; o.cols = t.blk.cols;
    o.band = t.band; o.ready_base = t.ready_base;
    return t.op = cnt++;
}

// Copy band b of tile t into its local copy from `src`, an array of the same shape and orientation with leading
// dimension `sld`.  Bands cut the logical rows (A) / columns (B); in the physical (minor x major) array that is the minor
// axis (rows [lo, hi) of every column) or the major one (columns [lo, hi)).
cudaError_t copy_band(const Tile& t, bool is_a, int b, const char* src, size_t sld, cudaMemcpyKind kind, cudaStream_t st) {
    const bool trans = t.blk.is_transpose != 0;
    const size_t es = elem_size(t.blk.dtype), dld = t.blk.ld;
    const int minor = trans ? t.blk.cols : t.blk.rows, major = trans ? t.blk.rows : t.blk.cols;
    const int lo = b * t.band, hi = std::min(is_a ? t.blk.rows : t.blk.cols, lo + t.band);
    char* dst = elem_ptr(&t.blk);
    if (hi <= lo || minor <= 0 || major <= 0) return cudaSuccess;
    if (is_a != trans)
        return cudaMemcpy2DAsync(dst + (size_t)lo * es, dld * es, src + (size_t)lo * es, sld * es, (size_t)(hi - lo) * es, major, kind, st);
    return cudaMemcpy2DAsync(dst + (size_t)lo * dld * es, dld * es, src + (size_t)lo * sld * es, sld * es, (size_t)minor * es, hi - lo,
                             kind, st);
}

// The status word is set by any bounded device-side wait that gave up.  read_status queues its copy into status_host
// behind the work on st; check_status reports the copy read last.
cudaError_t read_status(mb_comm* c, cudaStream_t st) {
    return cudaMemcpyAsync(c->status_host, c->flags + F_STATUS, 8, cudaMemcpyDeviceToHost, st);
}
int32_t check_status(const mb_comm* c, const char* who) {
    if (*c->status_host == 0) return MB_OK;
    return fail(MB_ERR_TIMEOUT, "%s: a device-side wait for a peer timed out (status %llu): a rank died or fell out of step; results since then "
                "are invalid", who, *c->status_host);
}
// My tiles may not be overwritten or freed until every consumer has finished pulling them.
int32_t wait_consumers(mb_comm* c, const std::vector<char>& consumer, unsigned long long e, cudaStream_t st) {
    for (int p = 0; p < c->world; ++p)
        if (consumer[p]) MB_CUDA(waitf(c, flag_ch(c, c->rank, CH_DONE, p), e, st));
    return MB_OK;
}

// The grouped-launch tables are about 20 KB each: one pair per thread serves both entries.
thread_local mb::G2Launch launch_tables[2];

// mb_matmul_blocked_dist's products on the fast path (plain fp64 tiles, C tiles with two holders fused).
// Two launches of the grouped kernel with the exchange flags between them: L0 computes the halves the peers reduce
// (stored into their staging buffers) and the plain regions, L2 the halves reduced here (acc + the peer's staged
// partial).  Completion counted inside a kernel whose epilogue stores to peer memory was measured faulty — at 8192^2
// about one call in three came back with one 16 x 32 patch off by a single product term — so the kernel boundary is
// the completion point and the flags are stream memory operations.  Both launches share one operand table.
int32_t products_fused(mb_comm* c, unsigned long long e, const Plan& plan, const std::vector<MyC>& myc, std::vector<Tile>& tA,
                       std::vector<Tile>& tB, const int32_t* row_len, const int32_t* col_len, mb_block* const* C_tiles,
                       const std::vector<const ShmEntry*>& entC, const std::vector<size_t>& slot_off, const std::vector<int>& pair_slot,
                       std::vector<char>& partial_to, std::vector<char>& fused_free_to) {
    mb_ctx* ctx = c->ctx;
    const int rank = c->rank, k = plan.k, n = plan.n;
    mb::G2Launch& L0 = launch_tables[0];
    mb::G2Launch& L2 = launch_tables[1];
    L0 = mb::G2Launch();
    L2 = mb::G2Launch();
    // entries: regions that peers wait for first, plain regions next, regions that wait for a peer last; at most two per
    // C tile, which the plan-wide check keeps within the table
    struct Reg { const MyC* mc; int n_off, N; int phase; };   // phase 0 = peer's half (store remote), 1 = plain, 2 = my half (needs the peer's)
    std::vector<Reg> regs;
    for (const MyC& mc : myc) {
        const int N_ = col_len[mc.j];
        if (plan.holders[mc.id].size() == 2) {
            const int nh = half_cols(N_);
            const bool owner = plan.holders[mc.id][0] == rank;
            // the owner reduces the left half [0, nh), the partner the right half [nh, N)
            if (owner) { if (N_ > nh) regs.push_back({&mc, nh, N_ - nh, 0}); regs.push_back({&mc, 0, nh, 2}); }
            else { regs.push_back({&mc, 0, nh, 0}); if (N_ > nh) regs.push_back({&mc, nh, N_ - nh, 2}); }
        } else {
            regs.push_back({&mc, 0, N_, 1});
        }
    }
    std::stable_sort(regs.begin(), regs.end(), [](const Reg& a, const Reg& b) { return a.phase < b.phase; });
    struct Note { int peer, slot; };
    std::vector<Note> wrote, need, final_to;              // F_PART2 to signal / F_PART2 to wait for / F_FINAL2 to signal
    for (const Reg& rg : regs) {
        const MyC& mc = *rg.mc;
        const int id = mc.id;
        mb::G2Launch& L = rg.phase == 2 ? L2 : L0;
        mb::G2Entry& en = L.E[L.ne++];
        en.nseg = (int)mc.kks.size();
        for (int s = 0; s < en.nseg; ++s) {
            en.a_op[s] = op_of(L0, tA[mc.i * k + mc.kks[s]], true);
            en.b_op[s] = op_of(L0, tB[mc.kks[s] * n + mc.j], false);
        }
        en.m_off = 0; en.n_off = rg.n_off; en.M = row_len[mc.i]; en.N = rg.N;
        const auto& h = plan.holders[id];
        const int ldst = even(row_len[mc.i]);               // leading dimension of a staged partial
        if (rg.phase == 1) {
            if (h[0] == rank) {                          // my own tile (other holders, if any, are added in step 4)
                en.D = f64_ptr(C_tiles[id]); en.ldd = C_tiles[id]->ld;
            } else {                                     // staged path: straight into my slot of the owner's staging buffer
                en.D = reinterpret_cast<double*>(c->staging_peer[h[0]] + (size_t)rank * c->slot_bytes + slot_off[id]);
                en.ldd = ldst;
                partial_to[h[0]] = 1;
            }
            continue;
        }
        const int peer = h[0] == rank ? h[1] : h[0];
        const int slot = pair_slot[id];
        if (rg.phase == 0) {
            // the half the PEER reduces: my partial of it goes over NVLink into my slot of the peer's staging buffer
            en.D = reinterpret_cast<double*>(c->staging_peer[peer] + (size_t)rank * c->slot_bytes + slot_off[id]);
            en.ldd = ldst;
            wrote.push_back({peer, slot});
        } else {
            // the half I reduce: acc + the peer's staged partial; the result belongs in the OWNER's C tile
            en.Cin = reinterpret_cast<const double*>(c->staging + (size_t)peer * c->slot_bytes + slot_off[id]);
            en.ldcin = ldst;
            need.push_back({peer, slot});
            if (h[0] == rank) {
                en.D = f64_ptr(C_tiles[id]) + (size_t)rg.n_off * C_tiles[id]->ld; en.ldd = C_tiles[id]->ld;
            } else {
                if (!entC[id]) return fail(MB_ERR_INVALID_ARG, "mb_matmul_blocked_dist: owner did not publish C tile %d", id);
                char* cp = nullptr;
                int32_t rc = open_entry(*entC[id], &cp);
                if (rc) return rc;
                en.D = reinterpret_cast<double*>(cp) + (size_t)rg.n_off * entC[id]->ld; en.ldd = entC[id]->ld;
                final_to.push_back({peer, slot});
            }
            fused_free_to[peer] = 1;
        }
    }
    L2.na = L0.na; L2.nb = L0.nb;
    std::copy_n(L0.A, L0.na, L2.A);
    std::copy_n(L0.B, L0.nb, L2.B);
    L0.ready = L2.ready = c->flags + F_BAND; L0.ready_val = L2.ready_val = e;
    L0.status = L2.status = c->flags + F_STATUS; L0.timeout_ns = L2.timeout_ns = timeout_ns(c);
    cudaError_t ce = mb::gemm_f64_grouped2(L0, ctx->num_sms, ctx->stream);
    if (ce != cudaSuccess) return cuda_fail(ce, "gemm_f64_grouped2 (first half)");
    for (const Note& w : wrote) MB_CUDA(sig(c, c->flags_peer[w.peer] + F_PART2 + rank * MAX_PAIR + w.slot, e, ctx->stream));
    for (const Note& w : need) MB_CUDA(waitf(c, c->flags + F_PART2 + w.peer * MAX_PAIR + w.slot, e, ctx->stream));
    ce = mb::gemm_f64_grouped2(L2, ctx->num_sms, ctx->stream);
    if (ce != cudaSuccess) return cuda_fail(ce, "gemm_f64_grouped2 (second half)");
    for (const Note& w : final_to) MB_CUDA(sig(c, c->flags_peer[w.peer] + F_FINAL2 + rank * MAX_PAIR + w.slot, e, ctx->stream));
    return MB_OK;
}

// mb_matmul_blocked_dist's products on the general path: per product (or per C tile when all kk are here), tile-level
// waits, staged partials.
int32_t products_general(mb_comm* c, const Plan& plan, const std::vector<MyC>& myc, std::vector<Tile>& tA, std::vector<Tile>& tB,
                         const int32_t* row_len, const int32_t* col_len, int out_dtype, mb_block* const* C_tiles,
                         const std::vector<size_t>& slot_off, std::vector<char>& partial_to) {
    mb_ctx* ctx = c->ctx;
    const int rank = c->rank, m = plan.m, k = plan.k, n = plan.n;
    cudaStream_t S = ctx->stream;
    int32_t rc = MB_OK;
    for (const MyC& mc : myc) {
        const auto& h = plan.holders[mc.id];
        mb_block out;
        if (h[0] == rank) { out = *C_tiles[mc.id]; out.owns = 0; }
        else {
            out = mb_block();
            out.data = c->staging_peer[h[0]] + (size_t)rank * c->slot_bytes + slot_off[mc.id];
            out.rows = row_len[mc.i]; out.cols = col_len[mc.j]; out.ld = even(row_len[mc.i]); out.dtype = out_dtype; out.device = ctx->device;
            partial_to[h[0]] = 1;
        }
        for (int kk : mc.kks) {
            Tile& a = tA[mc.i * k + kk];
            Tile& b = tB[kk * n + mc.j];
            if (a.landed) MB_CUDA(cudaStreamWaitEvent(S, a.landed, 0));
            if (b.landed) MB_CUDA(cudaStreamWaitEvent(S, b.landed, 0));
        }
        if ((int)mc.kks.size() == k) {
            // every kk of this C tile is here: one launch per tile (bf16: K segments in one wgmma launch; fp64: grouped DMMA)
            std::vector<mb_block*> at(m * k, nullptr), bt(k * n, nullptr), ct(m * n, nullptr);
            for (int kk = 0; kk < k; ++kk) { at[mc.i * k + kk] = &tA[mc.i * k + kk].blk; bt[kk * n + mc.j] = &tB[kk * n + mc.j].blk; }
            ct[mc.id] = &out;
            const int32_t id = mc.id;
            if ((rc = mb_matmul_blocked_subset(ctx, at.data(), bt.data(), m, k, n, ct.data(), &id, 1)) != MB_OK) return rc;
        } else {
            bool first = true;
            for (int kk : mc.kks) {
                if ((rc = mb_block_gemm(ctx, &tA[mc.i * k + kk].blk, &tB[kk * n + mc.j].blk, &out, first ? 0 : 1)) != MB_OK) return rc;
                first = false;
            }
        }
    }
    return MB_OK;
}

}  // namespace

extern "C" {

int32_t mb_dist_plan(int32_t m, int32_t k, int32_t n, int32_t world, int32_t* product_rank_out, int32_t* c_owner_out) {
    if (m <= 0 || k <= 0 || n <= 0 || world <= 0) return fail(MB_ERR_INVALID_ARG, "mb_dist_plan: bad argument");
    Plan p = make_plan(m, k, n, world);
    if (product_rank_out) for (int s = 0; s < m * k * n; ++s) product_rank_out[s] = p.prod_rank[s];
    if (c_owner_out) for (int c = 0; c < m * n; ++c) c_owner_out[c] = p.holders[c][0];
    return MB_OK;
}

int32_t mb_comm_init(mb_ctx* ctx, int32_t rank, int32_t world, const char* session, mb_comm** out) {
    MB_CTX(ctx);
    if (!out || !session || world < 1 || world > MAXW || rank < 0 || rank >= world)
        return fail(MB_ERR_INVALID_ARG, "mb_comm_init: bad argument (world must be 1..%d)", MAXW);
    mb_comm* c = new (std::nothrow) mb_comm();
    if (!c) return fail(MB_ERR_OOM, "host allocation failed");
    c->ctx = ctx; c->rank = rank; c->world = world;
    c->name = std::string("/marlin_b200_") + session;
    if (const char* t = getenv("MARLIN_B200_TIMEOUT_S")) c->timeout_s = std::max(1.0, atof(t));
    const int fd = shm_open(c->name.c_str(), O_CREAT | O_RDWR, 0600);
    if (fd < 0) { delete c; return fail(MB_ERR_CUDA, "mb_comm_init: shm_open(%s) failed", c->name.c_str()); }
    c->shm_bytes = sizeof(Shm);
    if (ftruncate(fd, (off_t)c->shm_bytes) != 0) { close(fd); delete c; return fail(MB_ERR_CUDA, "mb_comm_init: ftruncate failed"); }
    void* p = mmap(nullptr, c->shm_bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    close(fd);
    if (p == MAP_FAILED) { delete c; return fail(MB_ERR_CUDA, "mb_comm_init: mmap failed"); }
    c->shm = static_cast<Shm*>(p);                      // a fresh segment is zero-filled: all sequence numbers start at 0
    auto bail = [&](int32_t code) { munmap(c->shm, c->shm_bytes); if (rank == 0) shm_unlink(c->name.c_str()); delete c; return code; };
    cudaError_t e = cudaMalloc(&c->flags, sizeof(unsigned long long) * FLAG_WORDS);
    if (e == cudaSuccess) e = cudaMemset(c->flags, 0, sizeof(unsigned long long) * FLAG_WORDS);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&c->X, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&c->R, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&c->G, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_half[0], cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_half[1], cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_compute, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_tmp, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaMallocHost(&c->status_host, 8);
    if (e == cudaSuccess) e = cudaMallocHost(&c->ring, RING_SLOTS * 8);
    if (e != cudaSuccess) return bail(cuda_fail(e, "mb_comm_init"));
    if (!mb::stream_memops_available())
        return bail(fail(MB_ERR_UNSUPPORTED, "mb_comm_init: the driver does not expose cuStreamWriteValue64 / cuStreamWaitValue64"));
    *c->status_host = 0;
    ShmRank& me = c->shm->r[rank];
    long long off = 0, bytes = 0;
    e = mb::ipc_export(c->flags, me.flags_handle, &off, &bytes);
    if (e != cudaSuccess) return bail(cuda_fail(e, "mb_comm_init: cudaIpcGetMemHandle (is this memory from cudaMalloc?)"));
    me.flags_off = off;
    me.boot_seq.store(1, std::memory_order_release);
    for (int q = 0; q < world; ++q) {
        int32_t r = spin_until(c, [&] { return c->shm->r[q].boot_seq.load(std::memory_order_acquire) >= 1; }, "all ranks to attach");
        if (r) return bail(r);
        if (q == rank) { c->flags_peer[q] = c->flags; continue; }
        void* base = nullptr;
        e = mb::ipc_open_ex(c->shm->r[q].flags_handle, &base, true);
        if (e != cudaSuccess) return bail(cuda_fail(e, "mb_comm_init: cudaIpcOpenMemHandle (peer access between the GPUs?)"));
        c->flags_peer[q] = reinterpret_cast<unsigned long long*>(static_cast<char*>(base) + c->shm->r[q].flags_off);
    }
    int32_t r = host_barrier(c);
    if (r) return bail(r);
    // does the driver accept stream memory operations on peer addresses?  (one probe write per peer into a spare word)
    for (int q = 0; q < world && c->remote_write_ok; ++q)
        if (q != rank && mb::stream_write64(c->flags_peer[q] + F_STATUS + 1 + (rank % 4), 1, c->X) != cudaSuccess) {
            c->remote_write_ok = false;
            cudaGetLastError();
        }
    cudaStreamSynchronize(c->X);
    if (cudaGetLastError() != cudaSuccess) c->remote_write_ok = false;
    if ((r = host_barrier(c)) != MB_OK) return bail(r);
    if (rank == 0) shm_unlink(c->name.c_str());          // everyone has mapped it; the name can go
    *out = c;
    return MB_OK;
}

int32_t mb_comm_destroy(mb_comm* c) {
    if (!c) return MB_OK;
    cudaSetDevice(c->ctx->device);
    cudaDeviceSynchronize();
    host_barrier(c);                                       // nobody is still reading my memory
    mb::ipc_close_all();
    if (c->staging) cudaFree(c->staging);
    if (c->arena) cudaFree(c->arena);
    if (c->flags) cudaFree(c->flags);
    if (c->status_host) cudaFreeHost(c->status_host);
    if (c->ring) cudaFreeHost(c->ring);
    if (c->ev_compute) cudaEventDestroy(c->ev_compute);
    if (c->ev_tmp) cudaEventDestroy(c->ev_tmp);
    if (c->X) cudaStreamDestroy(c->X);
    if (c->R) cudaStreamDestroy(c->R);
    if (c->G) cudaStreamDestroy(c->G);
    for (int p = 0; p < 2; ++p) if (c->ev_half[p]) cudaEventDestroy(c->ev_half[p]);
    if (c->shm) munmap(c->shm, c->shm_bytes);
    delete c;
    return MB_OK;
}

int32_t mb_comm_rank(const mb_comm* c) { return c ? c->rank : -1; }
int32_t mb_comm_world(const mb_comm* c) { return c ? c->world : 0; }
int32_t mb_comm_barrier(mb_comm* c) {
    if (!c) return fail(MB_ERR_INVALID_ARG, "null communicator");
    return host_barrier(c);
}

// Give up on the peers: releases every wait this rank has queued (results are garbage), later calls fail.
int32_t mb_comm_abort(mb_comm* c) {
    if (!c) return fail(MB_ERR_INVALID_ARG, "null communicator");
    MB_CTX(c->ctx);
    abort_local(c);
    return MB_OK;
}

// Has any bounded device-side wait given up since the communicator was created?  (Synchronises the context stream.)
int32_t mb_comm_check(mb_comm* c) {
    int32_t r = check_call(c, "mb_comm_check", true);
    if (r) return r;
    MB_CUDA(read_status(c, c->ctx->stream));
    if ((r = sync_bounded(c, c->ctx->stream, "mb_comm_check")) != MB_OK) return r;
    return check_status(c, "mb_comm_check");
}

// ------------------------------------------------------------------------------------------------------------------
// BlockMatrix.multiply(other: BlockMatrix) across the ranks of `comm` (matrix/BlockMatrix.scala:149-186), device tiles.
// Collective.  A_tiles[i*k+kk] / B_tiles[kk*n+j] are the blocks THIS rank owns (NULL elsewhere), a_owner / b_owner say
// where every block lives; C_tiles[i*n+j] must be a preallocated block wherever mb_dist_plan() names this rank as owner.
// ------------------------------------------------------------------------------------------------------------------
int32_t mb_matmul_blocked_dist(mb_comm* c, mb_block* const* A_tiles, const int32_t* a_owner, mb_block* const* B_tiles,
                               const int32_t* b_owner, int32_t m, int32_t k, int32_t n, const int32_t* row_len,
                               const int32_t* k_len, const int32_t* col_len, int32_t dtype, mb_block* const* C_tiles) {
    int32_t rc = check_call(c, "mb_matmul_blocked_dist", A_tiles && B_tiles && C_tiles && a_owner && b_owner && row_len && k_len && col_len &&
                                                         m > 0 && k > 0 && n > 0);
    if (rc) return rc;
    mb_ctx* ctx = c->ctx;
    MB_LOCK(ctx);
    if (dtype != MB_F64 && dtype != MB_BF16) return fail(MB_ERR_UNSUPPORTED, "mb_matmul_blocked_dist: fp64 or bf16 tiles");
    const int rank = c->rank, world = c->world;
    const int out_dtype = dtype == MB_BF16 ? MB_F32 : MB_F64;
    const size_t osz = elem_size(out_dtype);
    cudaStream_t S = ctx->stream, X = c->X;
    const Plan plan = make_plan(m, k, n, world);
    // ---- local validation (before anything collective) ----
    for (int t = 0; t < m * k; ++t) {
        if (a_owner[t] < 0 || a_owner[t] >= world) return fail(MB_ERR_INVALID_ARG, "mb_matmul_blocked_dist: bad owner of A tile %d", t);
        if (a_owner[t] == rank) {
            const mb_block* b = A_tiles[t];
            if (!b || b->dtype != dtype || b->rows != row_len[t / k] || b->cols != k_len[t % k])
                return fail(MB_ERR_DIM_MISMATCH, "mb_matmul_blocked_dist: A(%d,%d) missing or not %dx%d", t / k, t % k, row_len[t / k], k_len[t % k]);
        }
    }
    for (int t = 0; t < k * n; ++t) {
        if (b_owner[t] < 0 || b_owner[t] >= world) return fail(MB_ERR_INVALID_ARG, "mb_matmul_blocked_dist: bad owner of B tile %d", t);
        if (b_owner[t] == rank) {
            const mb_block* b = B_tiles[t];
            if (!b || b->dtype != dtype || b->rows != k_len[t / n] || b->cols != col_len[t % n])
                return fail(MB_ERR_DIM_MISMATCH, "mb_matmul_blocked_dist: B(%d,%d) missing or not %dx%d", t / n, t % n, k_len[t / n], col_len[t % n]);
        }
    }
    for (int t = 0; t < m * n; ++t)
        if (plan.holders[t][0] == rank) {
            const mb_block* b = C_tiles[t];
            if (!b || b->rows != row_len[t / n] || b->cols != col_len[t % n] || b->dtype != out_dtype)
                return fail(MB_ERR_DIM_MISMATCH, "mb_matmul_blocked_dist: C(%d,%d) missing, or not a %dx%d block of the result type", t / n, t % n,
                            row_len[t / n], col_len[t % n]);
        }
    const unsigned long long e = ++c->epoch;
    ctx->events_used = 0;

    // ---- 0. publish the tiles I own, read everybody's ----
    std::vector<ShmEntry> mine;
    for (int t = 0; t < m * k; ++t)
        if (a_owner[t] == rank) { ShmEntry en; int32_t r = export_block(A_tiles[t], 0, t, &en); if (r) return r; mine.push_back(en); }
    for (int t = 0; t < k * n; ++t)
        if (b_owner[t] == rank) { ShmEntry en; int32_t r = export_block(B_tiles[t], 1, t, &en); if (r) return r; mine.push_back(en); }
    for (int t = 0; t < m * n; ++t)
        if (plan.holders[t][0] == rank && plan.holders[t].size() > 1) {
            ShmEntry en; int32_t r = export_block(C_tiles[t], 2, t, &en); if (r) return r; mine.push_back(en);
        }
    std::vector<std::vector<ShmEntry>> dir;
    if ((rc = exchange_directory(c, e, mine, dir)) != MB_OK) return rc;
    const std::vector<const ShmEntry*> entA = entries_of(dir, 0, m * k, a_owner), entB = entries_of(dir, 1, k * n, b_owner),
                                       entC = entries_of(dir, 2, m * n, nullptr);
    for (int t = 0; t < m * k; ++t) if (!entA[t]) return fail(MB_ERR_INVALID_ARG, "mb_matmul_blocked_dist: rank %d did not publish A tile %d", a_owner[t], t);
    for (int t = 0; t < k * n; ++t) if (!entB[t]) return fail(MB_ERR_INVALID_ARG, "mb_matmul_blocked_dist: rank %d did not publish B tile %d", b_owner[t], t);

    // ---- the same decision on every rank: can the whole call use the grouped DMMA launch / the fused reduce-scatter? ----
    bool fast = dtype == MB_F64 && k <= mb::G2_MAX_SEG;
    auto plain = [](const ShmEntry* en) { return en->dtype == MB_F64 && !en->trans && (en->ld % 2) == 0 && (en->offset % 16) == 0; };
    for (int t = 0; t < m * k && fast; ++t) fast = plain(entA[t]) && entA[t]->rows > 0 && entA[t]->cols > 0;
    for (int t = 0; t < k * n && fast; ++t) fast = plain(entB[t]) && entB[t]->cols > 0;
    for (int t = 0; t < m * n && fast; ++t) if (entC[t]) fast = plain(entC[t]);
    if (const char* env = getenv("MARLIN_B200_DIST_SLOW")) if (env[0] == '1') fast = false;
    // one grouped launch per rank: two entries per C tile at most
    for (int r = 0; r < world && fast; ++r) {
        const std::vector<MyC> cs = plan.c_tiles_of(r);
        fast = operands_fit(plan, cs) && 2 * (int)cs.size() <= mb::G2_MAX_ENTRIES;
    }
    const std::vector<MyC> myc = plan.c_tiles_of(rank);      // my products, my C regions
    // fused pairs: C tiles with exactly two holders.  slot = ordinal among the tiles this pair shares, in (i,j) order.
    auto fused_tile = [&](int id) { return fast && plan.holders[id].size() == 2; };
    std::map<std::pair<int, int>, int> pair_count;          // (lo rank, hi rank) -> tiles so far
    std::vector<int> pair_slot(m * n, -1);
    for (int id = 0; id < m * n; ++id)
        if (fused_tile(id)) {
            const int a = std::min(plan.holders[id][0], plan.holders[id][1]), b = std::max(plan.holders[id][0], plan.holders[id][1]);
            pair_slot[id] = pair_count[{a, b}]++;
            if (pair_slot[id] >= MAX_PAIR) { fast = false; break; }     // same on every rank
        }

    // ---- staging need per (src -> dst), identical arithmetic on every rank ----
    std::vector<size_t> slot_off(m * n, 0);                 // offset of tile id inside the (src -> dst) slot, for the pair that uses it
    size_t need_slot = 0;
    {
        std::map<std::pair<int, int>, size_t> used;         // (src, dst) -> bytes
        for (int id = 0; id < m * n; ++id) {
            const auto& h = plan.holders[id];
            if (h.size() < 2) continue;
            const size_t M_ = row_len[id / n], N_ = col_len[id % n];
            if (fused_tile(id)) {
                // owner h[0] receives the partner's partial of the left half; the partner receives the owner's partial of the right half
                const size_t nh = half_cols(col_len[id % n]);
                size_t& u0 = used[{h[1], h[0]}];
                size_t& u1 = used[{h[0], h[1]}];
                slot_off[id] = std::max(u0, u1);            // one offset for both directions keeps the bookkeeping simple
                u0 = u1 = slot_off[id] + up256((size_t)even((int)M_) * std::max(nh, N_ - nh) * osz);
            } else {
                size_t off = 0;
                for (size_t s = 1; s < h.size(); ++s) off = std::max(off, used[{h[s], h[0]}]);
                slot_off[id] = off;
                for (size_t s = 1; s < h.size(); ++s) used[{h[s], h[0]}] = off + up256((size_t)even((int)M_) * N_ * osz);
            }
        }
        for (auto& kv : used) need_slot = std::max(need_slot, kv.second);
    }
    if ((rc = ensure_staging(c, need_slot)) != MB_OK) return rc;

    // ---- 1. tell my consumers that my tiles are final (stream-ordered behind whatever produced them on S) ----
    std::vector<char> consumer(world, 0), source(world, 0);
    std::vector<Tile> tA(m * k), tB(k * n);
    for (int i = 0; i < m; ++i)
        for (int j = 0; j < n; ++j)
            for (int kk = 0; kk < k; ++kk) {
                const int r = plan.prod_rank[i * n * k + j * k + kk];
                if (r == rank) { tA[i * k + kk].need = true; tB[kk * n + j].need = true; }
                else {
                    if (a_owner[i * k + kk] == rank) consumer[r] = 1;
                    if (b_owner[kk * n + j] == rank) consumer[r] = 1;
                }
            }
    {
        // Tiles that carry a ready event are offered as soon as those events have completed (stream G), not after everything
        // queued on S — so the pulls of this multiply can run under the products of the previous one.
        bool all_events = true;
        std::vector<void*> evs;
        for (int i = 0; i < m && all_events; ++i)
            for (int j = 0; j < n && all_events; ++j)
                for (int kk = 0; kk < k && all_events; ++kk) {
                    if (plan.prod_rank[i * n * k + j * k + kk] == rank) continue;
                    if (a_owner[i * k + kk] == rank) { void* ev = A_tiles[i * k + kk]->ready_event; if (ev) evs.push_back(ev); else all_events = false; }
                    if (b_owner[kk * n + j] == rank) { void* ev = B_tiles[kk * n + j]->ready_event; if (ev) evs.push_back(ev); else all_events = false; }
                }
        // READY is always written from stream G, so the epochs reach a consumer in order whichever rule a call used
        if (all_events && !evs.empty()) {
            std::sort(evs.begin(), evs.end());
            evs.erase(std::unique(evs.begin(), evs.end()), evs.end());
            for (void* ev : evs) MB_CUDA(cudaStreamWaitEvent(c->G, static_cast<cudaEvent_t>(ev), 0));
        } else {
            MB_CUDA(cudaEventRecord(c->ev_tmp, S));
            MB_CUDA(cudaStreamWaitEvent(c->G, c->ev_tmp, 0));
        }
        for (int p = 0; p < world; ++p)
            if (consumer[p]) MB_CUDA(sig(c, flag_ch(c, p, CH_READY, rank), e, c->G));
    }

    // ---- 2. pull the tiles I need, in first-use order, band by band, on the copy stream ----
    size_t arena_need = 0;
    std::vector<std::pair<int, int>> pulls;                  // (0 = A / 1 = B, idx) in first-use order
    for (const MyC& mc : myc)
        for (int kk : mc.kks) {
            const int ia = mc.i * k + kk, ib = kk * n + mc.j;
            if (a_owner[ia] != rank && !tA[ia].remote) { tA[ia].remote = true; pulls.push_back({0, ia}); }
            if (b_owner[ib] != rank && !tB[ib].remote) { tB[ib].remote = true; pulls.push_back({1, ib}); }
        }
    int flag_slot = 0;
    auto setup_tile = [&](Tile& t, const ShmEntry* en, const mb_block* local, bool is_a, int owner) {
        t.ent = en; t.src = owner;
        if (!t.remote) { t.blk = *local; t.blk.owns = 0; return; }
        // packed local copy of the physical (minor x major) array, even leading dimension, same orientation flag
        const int minor = en->trans ? en->cols : en->rows, major = en->trans ? en->rows : en->cols;
        t.blk = mb_block();
        t.blk.rows = en->rows; t.blk.cols = en->cols; t.blk.ld = std::max(2, even(minor)); t.blk.is_transpose = en->trans;
        t.blk.dtype = en->dtype; t.blk.device = ctx->device;
        t.blk.offset = (long long)(arena_need / elem_size(en->dtype));      // patched to a pointer once the arena exists
        arena_need += up256((size_t)t.blk.ld * std::max(1, major) * elem_size(en->dtype));
        bands_of(is_a ? en->rows : en->cols, fast ? MAX_BANDS : 1, t.band, t.nbands);
        if (fast) { t.ready_base = flag_slot * MAX_BANDS; ++flag_slot; }
    };
    for (int t = 0; t < m * k; ++t) if (tA[t].need) setup_tile(tA[t], entA[t], A_tiles[t], true, a_owner[t]);
    for (int t = 0; t < k * n; ++t) if (tB[t].need) setup_tile(tB[t], entB[t], B_tiles[t], false, b_owner[t]);
    // two halves, alternating by epoch: the pulls of this call may land while the previous call's products still read theirs
    const int half = (int)(e & 1);
    const size_t half_need = up256(arena_need);
    if (2 * half_need > c->arena_bytes) { c->have_half[0] = c->have_half[1] = false; }       // regrown below (device sync inside)
    if ((rc = ensure_arena(c, 2 * half_need)) != MB_OK) return rc;
    char* const arena_base = c->arena + (size_t)half * (c->arena_bytes / 2 / 256 * 256);
    for (auto& pr : pulls) {
        Tile& t = pr.first == 0 ? tA[pr.second] : tB[pr.second];
        t.blk.data = arena_base + t.blk.offset * (long long)elem_size(t.blk.dtype);
        t.blk.offset = 0;
    }
    if (!pulls.empty()) {
        // this half was last read by the products of two calls ago (or by a host-path call, which is synchronous)
        if (c->have_half[half]) MB_CUDA(cudaStreamWaitEvent(X, c->ev_half[half], 0));
        std::vector<char> waited(world, 0);
        // tiles of one product are interleaved band by band (A0 B0 A1 B1 ...); products follow one another
        size_t p0 = 0;
        while (p0 < pulls.size()) {
            size_t p1 = std::min(pulls.size(), p0 + 2);
            int maxb = 1;
            for (size_t q = p0; q < p1; ++q) {
                Tile& t = pulls[q].first == 0 ? tA[pulls[q].second] : tB[pulls[q].second];
                maxb = std::max(maxb, t.nbands);
                if (!waited[t.src]) { MB_CUDA(waitf(c, flag_ch(c, rank, CH_READY, t.src), e, X)); waited[t.src] = 1; source[t.src] = 1; }
            }
            for (int b = 0; b < maxb; ++b)
                for (size_t q = p0; q < p1; ++q) {
                    const bool is_a = pulls[q].first == 0;
                    Tile& t = is_a ? tA[pulls[q].second] : tB[pulls[q].second];
                    if (b >= t.nbands) continue;
                    char* src = nullptr;
                    if ((rc = open_entry(*t.ent, &src)) != MB_OK) return rc;
                    MB_CUDA(copy_band(t, is_a, b, src, t.ent->ld, cudaMemcpyDeviceToDevice, X));
                    if (t.ready_base >= 0) MB_CUDA(sig(c, c->flags + F_BAND + t.ready_base + b, e, X));
                    if (b == t.nbands - 1) {
                        MB_CUDA(next_event(ctx, &t.landed));
                        MB_CUDA(cudaEventRecord(t.landed, X));
                    }
                }
            p0 = p1;
        }
        for (int p = 0; p < world; ++p)
            if (source[p]) MB_CUDA(sig(c, flag_ch(c, p, CH_DONE, rank), e, X));
    }

    // ---- before my epilogues store into a peer's staging slot again: it has consumed what I stored there last time ----
    std::vector<char> writes_to(world, 0);
    for (const MyC& mc : myc) {
        const auto& h = plan.holders[mc.id];
        if (h.size() < 2) continue;
        if (fused_tile(mc.id)) {
            // the owner stores the right half [nh, N) into the partner's slot (if there is one), the partner the left half
            if (h[0] != rank || col_len[mc.j] > half_cols(col_len[mc.j])) writes_to[h[0] == rank ? h[1] : h[0]] = 1;
        } else if (h[0] != rank) writes_to[h[0]] = 1;
    }
    for (int p = 0; p < world; ++p)
        if (writes_to[p] && c->last_write_epoch[p]) MB_CUDA(waitf(c, flag_ch(c, rank, CH_FREE, p), c->last_write_epoch[p], S));

    // ---- 3. my block products ----
    std::vector<char> partial_to(world, 0);                  // staged path: owners I have stored a partial for
    std::vector<char> fused_free_to(world, 0);               // fused path: peers whose staged half I have consumed
    rc = fast ? products_fused(c, e, plan, myc, tA, tB, row_len, col_len, C_tiles, entC, slot_off, pair_slot, partial_to, fused_free_to)
              : products_general(c, plan, myc, tA, tB, row_len, col_len, out_dtype, C_tiles, slot_off, partial_to);
    if (rc) return rc;
    MB_CUDA(cudaEventRecord(c->ev_compute, S));
    c->have_compute = true;
    MB_CUDA(cudaEventRecord(c->ev_half[half], S));
    c->have_half[half] = true;

    // ---- 4. the reduceByKey across ranks ----
    for (int p = 0; p < world; ++p) {
        if (partial_to[p]) MB_CUDA(sig(c, flag_ch(c, p, CH_PARTIAL, rank), e, S));
        if (partial_to[p] || (fast && writes_to[p])) c->last_write_epoch[p] = e;
    }
    // staged path, owner side: add the partials in holder order (deterministic), then free the slots
    std::vector<char> free_to(world, 0);
    for (const MyC& mc : myc) {
        const auto& h = plan.holders[mc.id];
        if (h.size() < 2 || h[0] != rank || fused_tile(mc.id)) continue;
        for (size_t s = 1; s < h.size(); ++s) {
            const int src = h[s];
            MB_CUDA(waitf(c, flag_ch(c, rank, CH_PARTIAL, src), e, S));
            mb_block part;
            part.data = c->staging + (size_t)src * c->slot_bytes + slot_off[mc.id];
            part.rows = row_len[mc.i]; part.cols = col_len[mc.j]; part.ld = even(row_len[mc.i]); part.dtype = out_dtype; part.device = ctx->device;
            if ((rc = mb_block_add(ctx, C_tiles[mc.id], &part, C_tiles[mc.id])) != MB_OK) return rc;
            free_to[src] = 1;
        }
    }
    // a C tile I own but hold no product of cannot exist: the owner is the holder of kk = 0
    for (int p = 0; p < world; ++p)
        if (free_to[p] || fused_free_to[p]) MB_CUDA(sig(c, flag_ch(c, p, CH_FREE, rank), e, S));
    // fused path, owner side: the partner's reduced half has landed in my C tile
    for (const MyC& mc : myc) {
        const auto& h = plan.holders[mc.id];
        if (fused_tile(mc.id) && h[0] == rank && col_len[mc.j] > half_cols(col_len[mc.j]))
            MB_CUDA(waitf(c, c->flags + F_FINAL2 + h[1] * MAX_PAIR + pair_slot[mc.id], e, S));
    }

    // ---- 5. my tiles may not be overwritten / freed until everyone has finished pulling them ----
    if ((rc = wait_consumers(c, consumer, e, S)) != MB_OK) return rc;
    // surface a timed-out wait of an EARLIER call (this call's status is read by the next one / mb_comm_check)
    if ((rc = check_status(c, "mb_matmul_blocked_dist")) != MB_OK) return rc;
    MB_CUDA(read_status(c, S));
    return MB_OK;
}


// ------------------------------------------------------------------------------------------------------------------
// Placement of HOST tiles for the end-to-end path: every input tile is uploaded (H2D) by exactly one of the ranks that
// need it, with the uploads spread as evenly as possible over the ranks' PCIe links; the other ranks that need the
// tile pull it over NVLink.  Deterministic: smallest feasible per-rank tile count, found by bipartite matching.
// ------------------------------------------------------------------------------------------------------------------
int32_t mb_dist_host_homes(int32_t m, int32_t k, int32_t n, int32_t world, int32_t* a_home, int32_t* b_home) {
    if (m <= 0 || k <= 0 || n <= 0 || world <= 0 || world > MAXW || !a_home || !b_home) return fail(MB_ERR_INVALID_ARG, "mb_dist_host_homes: bad argument");
    const Plan plan = make_plan(m, k, n, world);
    const int T = m * k + k * n;
    std::vector<std::vector<int>> cand(T);
    for (int i = 0; i < m; ++i)
        for (int j = 0; j < n; ++j)
            for (int kk = 0; kk < k; ++kk) {
                const int r = plan.prod_rank[i * n * k + j * k + kk];
                auto add = [&](int t) { if (std::find(cand[t].begin(), cand[t].end(), r) == cand[t].end()) cand[t].push_back(r); };
                add(i * k + kk);
                add(m * k + kk * n + j);
            }
    for (auto& cnd : cand) std::sort(cnd.begin(), cnd.end());
    for (int cap = (T + world - 1) / world; cap <= T; ++cap) {
        std::vector<std::vector<int>> held(world);              // rank -> tiles assigned
        std::vector<int> home(T, -1);
        // Kuhn's augmenting paths with rank capacity `cap`
        std::vector<char> seen;
        struct Rec { static bool go(int t, int cap, std::vector<std::vector<int>>& cand, std::vector<std::vector<int>>& held,
                                    std::vector<int>& home, std::vector<char>& seen) {
            for (int r : cand[t]) {
                if (seen[r]) continue;
                seen[r] = 1;
                if ((int)held[r].size() < cap) { held[r].push_back(t); home[t] = r; return true; }
                for (size_t x = 0; x < held[r].size(); ++x) {
                    const int other = held[r][x];
                    if (go(other, cap, cand, held, home, seen)) { held[r][x] = t; home[t] = r; return true; }
                }
            }
            return false;
        } };
        bool ok = true;
        for (int t = 0; t < T && ok; ++t) {
            seen.assign(world, 0);
            ok = Rec::go(t, cap, cand, held, home, seen);
        }
        if (ok) {
            for (int t = 0; t < m * k; ++t) a_home[t] = home[t];
            for (int t = 0; t < k * n; ++t) b_home[t] = home[m * k + t];
            return MB_OK;
        }
    }
    return fail(MB_ERR_UNSUPPORTED, "mb_dist_host_homes: no assignment");
}

// Pinned host memory shared by the ranks of one box (POSIX shm + cudaHostRegister): lets the ranks that reduce
// different parts of one C tile write them into ONE host array, and lets a test read the whole result in one process.
int32_t mb_host_alloc_shared(const char* name, int64_t bytes, void** out) {
    if (!name || bytes <= 0 || !out) return fail(MB_ERR_INVALID_ARG, "mb_host_alloc_shared: bad argument");
    std::string nm = std::string("/marlin_b200_h_") + name;
    const int fd = shm_open(nm.c_str(), O_CREAT | O_RDWR, 0600);
    if (fd < 0) return fail(MB_ERR_OOM, "mb_host_alloc_shared: shm_open(%s) failed", nm.c_str());
    if (ftruncate(fd, (off_t)bytes) != 0) { close(fd); return fail(MB_ERR_OOM, "mb_host_alloc_shared: ftruncate(%lld) failed", (long long)bytes); }
    void* p = mmap(nullptr, (size_t)bytes, PROT_READ | PROT_WRITE, MAP_SHARED | MAP_POPULATE, fd, 0);
    close(fd);
    if (p == MAP_FAILED) return fail(MB_ERR_OOM, "mb_host_alloc_shared: mmap failed");
    cudaError_t e = cudaHostRegister(p, (size_t)bytes, cudaHostRegisterPortable);
    if (e != cudaSuccess) { munmap(p, (size_t)bytes); return cuda_fail(e, "cudaHostRegister"); }
    *out = p;
    return MB_OK;
}
int32_t mb_host_free_shared(const char* name, void* ptr, int64_t bytes, int32_t unlink_name) {
    if (ptr) { cudaHostUnregister(ptr); munmap(ptr, (size_t)bytes); }
    if (unlink_name && name) shm_unlink((std::string("/marlin_b200_h_") + name).c_str());
    return MB_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// The same multiply END TO END: HOST tiles in, HOST tiles out, across the ranks of `comm` (bench.py's e2e at N > 1).
// A_host[i*k+kk] / B_host[kk*n+j]: packed column-major fp64 host tiles, non-NULL on the rank a_home / b_home names
// (mb_dist_host_homes spreads them over the PCIe links); C_host[i*n+j]: the packed (row_len[i] x col_len[j]) host tile,
// non-NULL on every rank that computes a partial of it (mb_dist_plan).  The two holders of a k-split tile each
// reduce and download a checkerboard of its (row band x column band) sub-blocks, so with one shared host array per tile
// (mb_host_alloc_shared) the tile is complete when every rank has returned.
//   upload stream   : my tiles, band by band (A: row bands, B: column bands), each band announced to its consumers;
//   pull stream     : the other tiles I need, band by band over NVLink as their uploaders announce them;
//   compute stream  : ONE grouped DMMA launch over the sub-blocks in wavefront order (sub-block (p,q) needs band p of
//                     the A tiles and band q of the B tiles); its producer waits per band, so the tensor cores start
//                     after a quarter of each tile has crossed PCIe; sub-blocks the peer reduces are stored by the
//                     epilogue straight into the peer's staging buffer;
//   reduce stream   : per finished sub-block: add the peer's staged partial, D2H — hidden behind the rest of the GEMM.
// Blocking: returns when this rank's part of C is in host memory.
// ------------------------------------------------------------------------------------------------------------------
int32_t mb_matmul_blocked_dist_host(mb_comm* c, const double* const* A_host, const int32_t* a_home, const double* const* B_host,
                                    const int32_t* b_home, int32_t m, int32_t k, int32_t n, const int32_t* row_len,
                                    const int32_t* k_len, const int32_t* col_len, double* const* C_host) {
    int32_t rc = check_call(c, "mb_matmul_blocked_dist_host", A_host && B_host && C_host && a_home && b_home && row_len && k_len && col_len &&
                                                              m > 0 && k > 0 && n > 0);
    if (rc) return rc;
    mb_ctx* ctx = c->ctx;
    MB_LOCK(ctx);
    const int rank = c->rank, world = c->world;
    if (k > mb::G2_MAX_SEG) return fail(MB_ERR_UNSUPPORTED, "mb_matmul_blocked_dist_host: k = %d > %d", k, mb::G2_MAX_SEG);
    for (int i = 0; i < m; ++i) if (row_len[i] <= 0) return fail(MB_ERR_UNSUPPORTED, "mb_matmul_blocked_dist_host: empty block row");
    for (int kk = 0; kk < k; ++kk) if (k_len[kk] <= 0) return fail(MB_ERR_UNSUPPORTED, "mb_matmul_blocked_dist_host: empty k segment");
    for (int j = 0; j < n; ++j) if (col_len[j] <= 0) return fail(MB_ERR_UNSUPPORTED, "mb_matmul_blocked_dist_host: empty block column");
    MB_CUDA(ensure_copy_streams(ctx));
    cudaStream_t S = ctx->stream, X = c->X, U = ctx->h2d_stream, R = c->R;
    const Plan plan = make_plan(m, k, n, world);
    // ---- global feasibility (the same verdict on every rank) ----
    std::vector<int> ups(world, 0);
    for (int t = 0; t < m * k; ++t) { if (a_home[t] < 0 || a_home[t] >= world) return fail(MB_ERR_INVALID_ARG, "bad a_home"); ++ups[a_home[t]]; }
    for (int t = 0; t < k * n; ++t) { if (b_home[t] < 0 || b_home[t] >= world) return fail(MB_ERR_INVALID_ARG, "bad b_home"); ++ups[b_home[t]]; }
    for (int r = 0; r < world; ++r) if (ups[r] > UP_SLOTS) return fail(MB_ERR_UNSUPPORTED, "mb_matmul_blocked_dist_host: rank %d would upload %d tiles (limit %d)", r, ups[r], UP_SLOTS);
    for (int id = 0; id < m * n; ++id) if (plan.holders[id].size() > 2) return fail(MB_ERR_UNSUPPORTED, "mb_matmul_blocked_dist_host: C tile %d has %d holders (limit 2)", id, (int)plan.holders[id].size());
    // one grouped launch per rank: one entry per sub-block
    for (int r = 0; r < world; ++r) {
        const std::vector<MyC> cs = plan.c_tiles_of(r);
        int subs = 0;
        std::map<int, int> pair_subs;
        for (const MyC& mc : cs) {
            int ba, nba, bb, nbb;
            bands_of(row_len[mc.i], MAX_BANDS, ba, nba); bands_of(col_len[mc.j], MAX_BANDS, bb, nbb);
            subs += nba * nbb;
            const auto& h = plan.holders[mc.id];
            if (h.size() == 2) pair_subs[h[0] == r ? h[1] : h[0]] += nba * nbb;
        }
        if (!operands_fit(plan, cs) || subs > mb::G2_MAX_ENTRIES)
            return fail(MB_ERR_UNSUPPORTED, "mb_matmul_blocked_dist_host: rank %d's share (%d sub-blocks) does not fit one grouped launch", r, subs);
        for (auto& kv : pair_subs) if (kv.second > SUB_SLOTS) return fail(MB_ERR_UNSUPPORTED, "mb_matmul_blocked_dist_host: too many shared sub-blocks");
    }
    // ---- local checks ----
    for (int t = 0; t < m * k; ++t) if (a_home[t] == rank && !A_host[t]) return fail(MB_ERR_INVALID_ARG, "mb_matmul_blocked_dist_host: A tile %d is homed here but NULL", t);
    for (int t = 0; t < k * n; ++t) if (b_home[t] == rank && !B_host[t]) return fail(MB_ERR_INVALID_ARG, "mb_matmul_blocked_dist_host: B tile %d is homed here but NULL", t);
    const std::vector<MyC> myc = plan.c_tiles_of(rank);
    for (const MyC& mc : myc)
        if (!C_host[mc.id]) return fail(MB_ERR_INVALID_ARG, "mb_matmul_blocked_dist_host: C tile %d is computed here but NULL", mc.id);
    const unsigned long long e = ++c->epoch;
    ctx->events_used = 0;

    // ---- device layout in the arena: tiles I upload, tiles I pull, my C tiles ----
    std::vector<Tile> tA(m * k), tB(k * n);
    for (const MyC& mc : myc)
        for (int kk : mc.kks) { tA[mc.i * k + kk].need = true; tB[kk * n + mc.j].need = true; }
    size_t total = 0;
    int nflag = 0;
    std::vector<int> slot_ctr(world, 0);
    auto place = [&](Tile& t, int rows, int cols, int home, bool is_a) {
        t.blk.rows = rows; t.blk.cols = cols; t.blk.ld = std::max(2, even(rows)); t.blk.dtype = MB_F64;
        t.src = home; t.up_slot = slot_ctr[home]++;
        bands_of(is_a ? rows : cols, MAX_BANDS, t.band, t.nbands);
        if (home == rank || t.need) { t.blk.offset = (long long)(total / 8); total += up256((size_t)t.blk.ld * cols * 8); }
        if (t.need) { t.ready_base = nflag * MAX_BANDS; ++nflag; }
    };
    for (int t = 0; t < m * k; ++t) place(tA[t], row_len[t / k], k_len[t % k], a_home[t], true);
    for (int t = 0; t < k * n; ++t) place(tB[t], k_len[t / n], col_len[t % n], b_home[t], false);
    std::vector<size_t> coff(m * n, 0);
    for (const MyC& mc : myc) { coff[mc.id] = total; total += up256((size_t)even(row_len[mc.i]) * col_len[mc.j] * 8); }
    // The arena may be regrown (device sync inside): peers cannot still be pulling from the old one, because every call
    // orders the DONE flags of its consumers on S before it ends.
    if ((rc = ensure_arena(c, total)) != MB_OK) return rc;
    for (Tile& t : tA) t.blk.data = c->arena;          // the tiles' offsets are arena offsets
    for (Tile& t : tB) t.blk.data = c->arena;

    // ---- staging: the partner's partial of a whole tile footprint per shared C tile ----
    std::vector<size_t> slot_off(m * n, 0);
    size_t need_slot = 0;
    std::vector<int> pair_base(m * n, 0);                     // first F_SUBDONE index of the tile for its pair
    {
        std::map<std::pair<int, int>, size_t> used;
        std::map<std::pair<int, int>, int> subs;
        for (int id = 0; id < m * n; ++id) {
            const auto& h = plan.holders[id];
            if (h.size() != 2) continue;
            const std::pair<int, int> key{std::min(h[0], h[1]), std::max(h[0], h[1])};
            slot_off[id] = used[key];
            used[key] += up256((size_t)even(row_len[id / n]) * col_len[id % n] * 8);
            int ba, nba, bb, nbb;
            bands_of(row_len[id / n], MAX_BANDS, ba, nba); bands_of(col_len[id % n], MAX_BANDS, bb, nbb);
            pair_base[id] = subs[key];
            subs[key] += nba * nbb;
        }
        for (auto& kv : used) need_slot = std::max(need_slot, kv.second);
    }
    if ((rc = ensure_staging(c, need_slot)) != MB_OK) return rc;

    // ---- publish my upload buffers, read everybody's ----
    std::vector<ShmEntry> mine;
    for (int t = 0; t < m * k; ++t)
        if (tA[t].src == rank) { ShmEntry en; if ((rc = export_block(&tA[t].blk, 0, t, &en)) != MB_OK) return rc; mine.push_back(en); }
    for (int t = 0; t < k * n; ++t)
        if (tB[t].src == rank) { ShmEntry en; if ((rc = export_block(&tB[t].blk, 1, t, &en)) != MB_OK) return rc; mine.push_back(en); }
    std::vector<std::vector<ShmEntry>> dir;
    if ((rc = exchange_directory(c, e, mine, dir)) != MB_OK) return rc;
    const std::vector<const ShmEntry*> entA = entries_of(dir, 0, m * k, a_home), entB = entries_of(dir, 1, k * n, b_home);
    for (int t = 0; t < m * k; ++t)
        if (tA[t].need && tA[t].src != rank && !(tA[t].ent = entA[t])) return fail(MB_ERR_INVALID_ARG, "mb_matmul_blocked_dist_host: a peer did not publish an A tile");
    for (int t = 0; t < k * n; ++t)
        if (tB[t].need && tB[t].src != rank && !(tB[t].ent = entB[t])) return fail(MB_ERR_INVALID_ARG, "mb_matmul_blocked_dist_host: a peer did not publish a B tile");

    // everything of the previous call that touches the arena / my uploads is ordered on S: fan that out
    MB_CUDA(cudaEventRecord(c->ev_tmp, S));
    MB_CUDA(cudaStreamWaitEvent(U, c->ev_tmp, 0));
    MB_CUDA(cudaStreamWaitEvent(X, c->ev_tmp, 0));
    MB_CUDA(cudaStreamWaitEvent(R, c->ev_tmp, 0));

    // ---- upload stream: my tiles band by band; every band is announced locally and to the ranks that pull it ----
    std::vector<std::vector<int>> consumers_a(m * k), consumers_b(k * n);
    std::vector<char> consumer(world, 0), source(world, 0);
    for (int i = 0; i < m; ++i)
        for (int j = 0; j < n; ++j)
            for (int kk = 0; kk < k; ++kk) {
                const int r = plan.prod_rank[i * n * k + j * k + kk];
                auto addc = [&](std::vector<int>& v) { if (r != rank && std::find(v.begin(), v.end(), r) == v.end()) v.push_back(r); };
                if (a_home[i * k + kk] == rank) addc(consumers_a[i * k + kk]);
                if (b_home[kk * n + j] == rank) addc(consumers_b[kk * n + j]);
            }
    for (int b = 0; b < MAX_BANDS; ++b) {
        for (int pass = 0; pass < 2; ++pass) {
            const int cnt = pass == 0 ? m * k : k * n;
            for (int t = 0; t < cnt; ++t) {
                Tile& ht = pass == 0 ? tA[t] : tB[t];
                if (ht.src != rank || b >= ht.nbands) continue;
                const double* src = pass == 0 ? A_host[t] : B_host[t];
                MB_CUDA(copy_band(ht, pass == 0, b, reinterpret_cast<const char*>(src), ht.blk.rows, cudaMemcpyHostToDevice, U));
                if (ht.need) MB_CUDA(sig(c, c->flags + F_BAND + ht.ready_base + b, e, U));
                for (int r : (pass == 0 ? consumers_a[t] : consumers_b[t])) {
                    MB_CUDA(sig(c, c->flags_peer[r] + F_UPREADY + (rank * UP_SLOTS + ht.up_slot) * MAX_BANDS + b, e, U));
                    consumer[r] = 1;
                }
            }
        }
    }
    // ---- pull stream: the other tiles I need, as their bands are announced ----
    for (int b = 0; b < MAX_BANDS; ++b) {
        for (int pass = 0; pass < 2; ++pass) {
            const int cnt = pass == 0 ? m * k : k * n;
            for (int t = 0; t < cnt; ++t) {
                Tile& ht = pass == 0 ? tA[t] : tB[t];
                if (!ht.need || ht.src == rank || b >= ht.nbands) continue;
                source[ht.src] = 1;
                MB_CUDA(waitf(c, c->flags + F_UPREADY + (ht.src * UP_SLOTS + ht.up_slot) * MAX_BANDS + b, e, X));
                char* peer = nullptr;
                if ((rc = open_entry(*ht.ent, &peer)) != MB_OK) return rc;
                if (pass == 0) {
                    MB_CUDA(copy_band(ht, true, b, peer, ht.blk.ld, cudaMemcpyDeviceToDevice, X));
                } else {            // a column band of the uploader's packed copy is one contiguous range
                    const size_t lo = (size_t)b * ht.band, hi = std::min((size_t)ht.blk.cols, lo + ht.band), ld = ht.blk.ld;
                    MB_CUDA(cudaMemcpyAsync(elem_ptr(&ht.blk) + lo * ld * 8, peer + lo * ld * 8, (hi - lo) * ld * 8, cudaMemcpyDeviceToDevice, X));
                }
                MB_CUDA(sig(c, c->flags + F_BAND + ht.ready_base + b, e, X));
            }
        }
    }
    for (int p = 0; p < world; ++p)
        if (source[p]) MB_CUDA(sig(c, flag_ch(c, p, CH_DONE, rank), e, X));

    // ---- compute stream: one grouped launch over my sub-blocks in wavefront order ----
    std::vector<char> writes_to(world, 0), reads_from(world, 0);
    for (const MyC& mc : myc) {
        const auto& h = plan.holders[mc.id];
        if (h.size() == 2) { const int peer = h[0] == rank ? h[1] : h[0]; writes_to[peer] = 1; reads_from[peer] = 1; }
    }
    // my partials of the sub-blocks the peer reduces are pushed into ITS staging buffer by my copy engine (stream R, below):
    // it must have consumed what I pushed there last time
    for (int p = 0; p < world; ++p)
        if (writes_to[p] && c->last_write_epoch[p]) MB_CUDA(waitf(c, flag_ch(c, rank, CH_FREE, p), c->last_write_epoch[p], R));
    mb::G2Launch& L = launch_tables[0];
    L = mb::G2Launch();
    struct Sub { const MyC* mc; int p, q, m_off, n_off, M, N, wave, sub_idx; bool mine; int entry; };
    std::vector<Sub> subs;
    for (const MyC& mc : myc) {
        int ba, nba, bb, nbb;
        bands_of(row_len[mc.i], MAX_BANDS, ba, nba); bands_of(col_len[mc.j], MAX_BANDS, bb, nbb);
        const auto& h = plan.holders[mc.id];
        const int my_pos = h[0] == rank ? 0 : 1;
        for (int p = 0; p < nba; ++p)
            for (int q = 0; q < nbb; ++q) {
                Sub sb{&mc, p, q, p * ba, q * bb, std::min(ba, row_len[mc.i] - p * ba), std::min(bb, col_len[mc.j] - q * bb), std::max(p, q),
                       pair_base[mc.id] + p * nbb + q, true, -1};
                if (h.size() == 2) sb.mine = ((p + q) % 2) == my_pos;        // checkerboard: both links carry half of the tile
                subs.push_back(sb);
            }
    }
    // wavefront order (the bands arrive in order); inside a wave the sub-blocks the PEER reduces come first, so that by the
    // time this rank reaches its own sub-blocks of the wave the peer — which runs the mirror-image order — has stored its
    // partials of them into this rank's staging buffer
    std::stable_sort(subs.begin(), subs.end(), [](const Sub& a, const Sub& b) {
        if (a.wave != b.wave) return a.wave < b.wave;
        if (a.mine != b.mine) return !a.mine;
        return a.mc->id != b.mc->id ? a.mc->id < b.mc->id : (a.p != b.p ? a.p < b.p : a.q < b.q);
    });
    for (Sub& sb : subs) {
        const MyC& mc = *sb.mc;
        sb.entry = L.ne;
        mb::G2Entry& en = L.E[L.ne++];
        en.nseg = (int)mc.kks.size();
        for (int sg = 0; sg < en.nseg; ++sg) {
            en.a_op[sg] = op_of(L, tA[mc.i * k + mc.kks[sg]], true);
            en.b_op[sg] = op_of(L, tB[mc.kks[sg] * n + mc.j], false);
        }
        en.m_off = sb.m_off; en.n_off = sb.n_off; en.M = sb.M; en.N = sb.N;
        const int ldc = even(row_len[mc.i]);
        en.done_ctr = c->flags + F_CTR + sb.entry;
        en.sig_val = e;
        const auto& h = plan.holders[mc.id];
        if (sb.mine) {
            en.D = reinterpret_cast<double*>(c->arena + coff[mc.id]) + (size_t)sb.n_off * ldc + sb.m_off; en.ldd = ldc;
            en.sig_local = c->flags + F_SIG + sb.entry;
            if (h.size() == 2) {
                // reduce in the epilogue: my partial + the peer's staged partial (no separate add kernel: a kernel launched
                // while this GEMM is resident might not be scheduled before it ends)
                const int peer = h[0] == rank ? h[1] : h[0];
                en.Cin = reinterpret_cast<const double*>(c->staging + (size_t)peer * c->slot_bytes + slot_off[mc.id]) + (size_t)sb.n_off * ldc + sb.m_off;
                en.ldcin = ldc;
                en.cin_flag = c->flags + F_SUBDONE + peer * SUB_SLOTS + sb.sub_idx;
                en.cin_val = e;
            }
        } else {
            // a sub-block the PEER reduces: my partial goes to the same place in my own C buffer (local stores: completion
            // counting next to peer stores proved unreliable, see mb_matmul_blocked_dist) and is pushed from there by the
            // copy engine once the entry's completion flag is up
            en.D = reinterpret_cast<double*>(c->arena + coff[mc.id]) + (size_t)sb.n_off * ldc + sb.m_off; en.ldd = ldc;
            en.sig_local = c->flags + F_SIG + sb.entry;
        }
    }
    L.ready = c->flags + F_BAND; L.ready_val = e; L.status = c->flags + F_STATUS; L.timeout_ns = timeout_ns(c);
    MB_CUDA(cudaMemsetAsync(c->flags + F_CTR, 0, sizeof(unsigned long long) * mb::G2_MAX_ENTRIES, S));
    if (const cudaError_t ce = mb::gemm_f64_grouped2(L, ctx->num_sms, S); ce != cudaSuccess)
        return cuda_fail(ce, "mb_matmul_blocked_dist_host: grouped launch");
    MB_CUDA(cudaEventRecord(c->ev_compute, S));
    c->have_compute = true;
    for (int p = 0; p < world; ++p) if (writes_to[p]) c->last_write_epoch[p] = e;

    // ---- copy-out stream, in entry order: a finished sub-block is either mine (already reduced in the epilogue) -> host,
    //      or the peer's -> pushed into its staging buffer over NVLink + its flag; all hidden behind the rest of the GEMM ----
    for (const Sub& sb : subs) {
        const int id = sb.mc->id, i = sb.mc->i;
        const int ldc = even(row_len[i]);
        MB_CUDA(waitf(c, c->flags + F_SIG + sb.entry, e, R));
        const double* src = reinterpret_cast<const double*>(c->arena + coff[id]) + (size_t)sb.n_off * ldc + sb.m_off;
        if (sb.mine) {
            MB_CUDA(cudaMemcpy2DAsync(C_host[id] + (size_t)sb.n_off * row_len[i] + sb.m_off, (size_t)row_len[i] * 8, src, (size_t)ldc * 8,
                                      (size_t)sb.M * 8, sb.N, cudaMemcpyDeviceToHost, R));
        } else {
            const auto& h = plan.holders[id];
            const int peer = h[0] == rank ? h[1] : h[0];
            double* dst = reinterpret_cast<double*>(c->staging_peer[peer] + (size_t)rank * c->slot_bytes + slot_off[id]) + (size_t)sb.n_off * ldc + sb.m_off;
            MB_CUDA(cudaMemcpy2DAsync(dst, (size_t)ldc * 8, src, (size_t)ldc * 8, (size_t)sb.M * 8, sb.N, cudaMemcpyDeviceToDevice, R));
            MB_CUDA(sig(c, c->flags_peer[peer] + F_SUBDONE + rank * SUB_SLOTS + sb.sub_idx, e, R));
        }
    }
    // the peer's staged partials have been consumed once my GEMM is done
    for (int p = 0; p < world; ++p)
        if (reads_from[p]) MB_CUDA(sig(c, flag_ch(c, p, CH_FREE, rank), e, S));
    // ---- my upload buffers may not be overwritten until everyone has pulled them; S is ordered behind R ----
    if ((rc = wait_consumers(c, consumer, e, S)) != MB_OK) return rc;
    MB_CUDA(cudaEventRecord(c->ev_tmp, R));
    MB_CUDA(cudaStreamWaitEvent(S, c->ev_tmp, 0));
    MB_CUDA(cudaEventRecord(c->ev_tmp, U));
    MB_CUDA(cudaStreamWaitEvent(S, c->ev_tmp, 0));
    MB_CUDA(read_status(c, S));
    if ((rc = sync_bounded(c, R, "mb_matmul_blocked_dist_host")) != MB_OK) return rc;
    if ((rc = sync_bounded(c, S, "mb_matmul_blocked_dist_host")) != MB_OK) return rc;
    return check_status(c, "mb_matmul_blocked_dist_host");
}

}  // extern "C"
