// The matrix-file writer on the device: the text of DenseVecMatrix.saveToFileSystem (matrix/DenseVecMatrix.scala:1042-1046)
// and BlockMatrix.saveToFileSystem(path, "blockmatrix") (matrix/BlockMatrix.scala:550-555), formatted by the tokens of
// text.h and streamed to a file.
//
// A segment is one view in file order: a row shard (row by row, one line per row, `id:DenseVector(v, v)`) or a block
// (column by column, one line, `r-c-rows-cols:v,v`).  Its values are cut into chunks of at most MB_TEXT_CHUNK_VALUES,
// which may split a line.  Each chunk takes two launches over tiles of TEXT_TILE values:
//   length  every thread computes the bytes of its values (prefix, token, separator); the CTA stores the tile's total.
//   write   the CTA sums the totals of the tiles before its own (its byte offset), recomputes its tokens in rounds of one
//           value per thread, scans their lengths and writes them into a shared-memory stage that has the output's
//           alignment mod 16, and stores the stage with 16-byte stores (byte stores only in the two edge words).
// The 5^q tables sit in shared memory: neighbouring threads index them differently.  The host pipelines the chunks:
// chunk k is formatted while chunk k - 1 is copied to pinned memory and chunk k - 2 is written to the file.
#include "text.h"
#include "../../include/marlin_b200.h"
#include "launch.h"
#include "stream_buffer.h"

#include <cerrno>
#include <cstring>
#include <string>
#include <vector>

namespace mb {
namespace {

using namespace text;

constexpr int TEXT_THREADS = 256;
constexpr int TEXT_ROUNDS = 8;
constexpr int TEXT_TILE = TEXT_THREADS * TEXT_ROUNDS;                 // values per CTA
constexpr int TEXT_PREFIX_MAX = 4 * 11 + 4;                            // r-c-rows-cols: of four int32; id:DenseVector( is 33
constexpr int TEXT_SEP_MAX = 2;                                        // ", " or ")\n"
constexpr int TEXT_VALUE_MAX = TEXT_PREFIX_MAX + TEXT_TOKEN_MAX + TEXT_SEP_MAX;
constexpr int TEXT_STAGE = TEXT_THREADS * TEXT_VALUE_MAX + 32;
static_assert(MB_TEXT_CHUNK_VALUES % TEXT_TILE == 0, "chunks are whole tiles");

__device__ const uint64_t g_pow5[] = MB_TEXT_POW5_TABLE;
__device__ const uint64_t g_pow5_inv[] = MB_TEXT_POW5_INV_TABLE;

struct Tables {
    uint64_t pow5[2 * MB_TEXT_POW5_COUNT];
    uint64_t pow5_inv[2 * MB_TEXT_POW5_INV_COUNT];
};

__device__ __forceinline__ void load_tables(Tables& t) {
    for (int i = threadIdx.x; i < 2 * MB_TEXT_POW5_COUNT; i += TEXT_THREADS) t.pow5[i] = g_pow5[i];
    for (int i = threadIdx.x; i < 2 * MB_TEXT_POW5_INV_COUNT; i += TEXT_THREADS) t.pow5_inv[i] = g_pow5_inv[i];
}

// The value at (r, c) of the view as fp64 bits; fp32 and bf16 widen exactly.
__device__ __forceinline__ uint64_t value_bits(const TextSegment& s, long long r, long long c) {
    const long long i = r * s.rs + c * s.cs;
    if (s.dtype == MB_F64) return __ldg(static_cast<const unsigned long long*>(s.data) + i);
    float f;
    if (s.dtype == MB_F32) f = __ldg(static_cast<const float*>(s.data) + i);
    else f = __uint_as_float((uint32_t)__ldg(static_cast<const unsigned short*>(s.data) + i) << 16);
    return (uint64_t)__double_as_longlong((double)f);
}

// Where a value sits: `major` is its line (row shard) or column (block), `minor` its place inside that.
struct Place {
    long long major;
    uint32_t minor;
};

// A chunk's values: n of them from place `first`.  `inner` is the length of a major step (cols of a shard, rows of a
// block) and `magic` = floor(2^64 / inner) + 1, so that x / inner = umulhi(x, magic) for every 32-bit x (inner > 1).
struct ChunkArgs {
    long long n;
    Place first;
    uint32_t inner;
    uint64_t magic;
};

// The place l values after c.first, for l < MB_TEXT_CHUNK_VALUES: integer multiplies only (no division instruction).
__device__ __forceinline__ Place place_at(const ChunkArgs& c, uint32_t l) {
    const uint32_t x = c.first.minor + l;                          // < 2^31 + 2^21: no wrap
    const uint32_t q = c.inner == 1 ? x : (uint32_t)__umul64hi(x, c.magic);
    return Place{c.first.major + q, x - q * c.inner};
}

// One value's text: the line's prefix before its first value, the token, and what follows it.
struct Piece {
    Token tok;
    int prefix;          // bytes of the prefix, 0 when none
    int sep;             // bytes after the token
    bool last;
};

__device__ __forceinline__ Piece piece_of(const TextSegment& s, const Place& p, const Tables& t) {
    Piece pc;
    const bool rows = s.ids != nullptr;
    const long long r = rows ? p.major : p.minor, c = rows ? p.minor : p.major;
    pc.tok = classify(value_bits(s, r, c), t.pow5, t.pow5_inv);
    const bool first = rows ? p.minor == 0 : (p.major == 0 && p.minor == 0);
    pc.last = rows ? p.minor == (uint32_t)s.cols - 1 : (p.major == s.cols - 1 && p.minor == (uint32_t)s.rows - 1);
    pc.prefix = 0;
    if (first) {
        pc.prefix = rows ? long_length(s.ids[p.major]) + 13
                         : long_length(s.block_row) + long_length(s.block_col) + long_length(s.rows) + long_length(s.cols) + 4;
    }
    pc.sep = rows ? 2 : 1;
    return pc;
}

__device__ __forceinline__ int piece_length(const Piece& pc) { return pc.prefix + token_length(pc.tok) + pc.sep; }

__device__ __forceinline__ int put(char* out, const char* s) {
    int n = 0;
    while (s[n]) {
        out[n] = s[n];
        ++n;
    }
    return n;
}

__device__ __forceinline__ void write_piece(const TextSegment& s, const Place& p, const Piece& pc, char* out) {
    const bool rows = s.ids != nullptr;
    int n = 0;
    if (pc.prefix) {
        if (rows) {
            n += write_long(s.ids[p.major], out);
            n += put(out + n, ":DenseVector(");
        } else {
            n += write_long(s.block_row, out);
            out[n++] = '-';
            n += write_long(s.block_col, out + n);
            out[n++] = '-';
            n += write_long(s.rows, out + n);
            out[n++] = '-';
            n += write_long(s.cols, out + n);
            out[n++] = ':';
        }
    }
    n += write_token(pc.tok, out + n);
    if (rows) {
        out[n] = pc.last ? ')' : ',';
        out[n + 1] = pc.last ? '\n' : ' ';
    } else {
        out[n] = pc.last ? '\n' : ',';
    }
}

// Sum over the CTA; every thread gets it.
__device__ __forceinline__ long long cta_sum(long long v, long long* warp_s) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) warp_s[threadIdx.x >> 5] = v;
    __syncthreads();
    long long s = 0;
#pragma unroll
    for (int w = 0; w < TEXT_THREADS / 32; ++w) s += warp_s[w];
    return s;
}

// The chunk's values: tile_bytes[tile] = the bytes of the tile's text.
__global__ void __launch_bounds__(TEXT_THREADS) text_length_kernel(TextSegment s, ChunkArgs c, int* __restrict__ tile_bytes) {
    __shared__ Tables t;
    __shared__ long long warp_s[TEXT_THREADS / 32];
    load_tables(t);
    __syncthreads();
    const uint32_t l0 = blockIdx.x * TEXT_TILE + threadIdx.x;
    long long sum = 0;
#pragma unroll 1
    for (int round = 0; round < TEXT_ROUNDS; ++round) {
        const uint32_t l = l0 + round * TEXT_THREADS;
        if (l < c.n) sum += piece_length(piece_of(s, place_at(c, l), t));
    }
    sum = cta_sum(sum, warp_s);
    if (threadIdx.x == 0) tile_bytes[blockIdx.x] = (int)sum;
}

// The same values' bytes at out[0 ..); *total = their count.
__global__ void __launch_bounds__(TEXT_THREADS) text_write_kernel(TextSegment s, ChunkArgs c,
                                                                  const int* __restrict__ tile_bytes, char* __restrict__ out,
                                                                  long long* __restrict__ total) {
    __shared__ Tables t;
    __shared__ __align__(16) char stage[TEXT_STAGE];
    __shared__ long long warp_s[TEXT_THREADS / 32];
    __shared__ int scan_s[TEXT_THREADS / 32];
    load_tables(t);
    long long before = 0;
    for (int i = threadIdx.x; i < (int)blockIdx.x; i += TEXT_THREADS) before += tile_bytes[i];
    long long base = cta_sum(before, warp_s);                       // also makes the tables visible
    if (threadIdx.x == 0 && blockIdx.x == gridDim.x - 1) *total = base + tile_bytes[blockIdx.x];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t l0 = blockIdx.x * TEXT_TILE + threadIdx.x;
#pragma unroll 1
    for (int round = 0; round < TEXT_ROUNDS; ++round) {
        const uint32_t l = l0 + round * TEXT_THREADS;
        const bool active = l < c.n;
        const Place p = place_at(c, l);
        if (!__syncthreads_or(active)) break;
        Piece pc{};
        int len = 0;
        if (active) {
            pc = piece_of(s, p, t);
            len = piece_length(pc);
        }
        int incl = len;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) scan_s[warp] = incl;
        __syncthreads();
        int excl = incl - len, round_bytes = 0;
#pragma unroll
        for (int w = 0; w < TEXT_THREADS / 32; ++w) {
            excl += w < warp ? scan_s[w] : 0;
            round_bytes += scan_s[w];
        }
        const int head = (int)(base & 15);                          // stage byte b is output byte (base & ~15) + b
        if (active) write_piece(s, p, pc, stage + head + excl);
        __syncthreads();
        char* dst = out + (base & ~15ll);
        const int end = head + round_bytes, words = (end + 15) >> 4;
        for (int w = threadIdx.x; w < words; w += TEXT_THREADS) {
            const int b0 = w << 4;
            if (b0 >= head && b0 + 16 <= end) {
                *reinterpret_cast<uint4*>(dst + b0) = *reinterpret_cast<const uint4*>(stage + b0);
            } else {
                for (int b = b0 > head ? b0 : head; b < b0 + 16 && b < end; ++b) dst[b] = stage[b];
            }
        }
        base += round_bytes;
        __syncthreads();                                            // the stage and scan_s are free again
    }
}

// A piece of the file: values [g0, g0 + n) of segment seg, or (n == 0) host-made text.
struct Chunk {
    int seg;
    long long g0, n;
    std::string host;
};

// The bytes a chunk of n values of s can take at most.
size_t chunk_bound(const TextSegment& s, long long n) {
    long long lines = 1;                                           // lines that start in the chunk
    if (s.ids) lines = n < n / s.cols + 2 ? n : n / s.cols + 2;
    return (size_t)n * (TEXT_TOKEN_MAX + TEXT_SEP_MAX) + (size_t)lines * TEXT_PREFIX_MAX;
}

// The text of a segment without values: zero-column rows or an empty block.
std::string empty_text(const TextSegment& s, const long long* host_ids) {
    char num[TEXT_LONG_MAX];
    std::string out;
    if (s.ids) {
        for (int r = 0; r < s.rows; ++r) {
            out.append(num, write_long(host_ids[r], num));
            out += ":DenseVector()\n";
        }
    } else {
        for (long long v : {(long long)s.block_row, (long long)s.block_col, (long long)s.rows, (long long)s.cols}) {
            out.append(num, write_long(v, num));
            out += '-';
        }
        out.back() = ':';
        out += '\n';
    }
    return out;
}

// Pinned host memory for the length of a call.
struct Pinned {
    char* p = nullptr;
    ~Pinned() { if (p) cudaFreeHost(p); }
};

}  // namespace

cudaError_t save_text(const TextSegment* segs, const long long* const* host_ids, int count, const TextIo& io, int* io_errno) {
    *io_errno = 0;
    std::vector<Chunk> chunks;
    size_t bound = 0;
    for (int i = 0; i < count; ++i) {
        const TextSegment& s = segs[i];
        const long long n = (long long)s.rows * s.cols;
        if (s.ids && s.rows == 0) continue;
        if (n == 0) {
            chunks.push_back(Chunk{i, 0, 0, empty_text(s, host_ids[i])});
            continue;
        }
        for (long long g0 = 0; g0 < n; g0 += MB_TEXT_CHUNK_VALUES) {
            const long long m = n - g0 < MB_TEXT_CHUNK_VALUES ? n - g0 : MB_TEXT_CHUNK_VALUES;
            chunks.push_back(Chunk{i, g0, m, {}});
            const size_t b = chunk_bound(s, m);
            bound = b > bound ? b : bound;
        }
    }
    bound = (bound + 255) & ~size_t(255);
    const int max_tiles = MB_TEXT_CHUNK_VALUES / TEXT_TILE;
    // two of everything: chunk k uses slot k % 2
    StreamBuffer text_buf, tile_buf;
    Pinned pinned;
    cudaError_t e = cudaSuccess;
    if (bound) {
        if ((e = text_buf.alloc(2 * bound, io.stream)) != cudaSuccess) return e;
        if ((e = tile_buf.alloc(2 * (max_tiles * sizeof(int) + sizeof(long long)), io.stream)) != cudaSuccess) return e;
        if ((e = cudaMallocHost(&pinned.p, 2 * bound + 2 * sizeof(long long))) != cudaSuccess) return e;
    }
    char* dev_text[2] = {text_buf.as<char>(), text_buf.as<char>() + bound};
    long long* dev_total = tile_buf.as<long long>();                      // [2]
    int* dev_tiles[2] = {reinterpret_cast<int*>(dev_total + 2), reinterpret_cast<int*>(dev_total + 2) + max_tiles};
    char* host_text[2] = {pinned.p, pinned.p + bound};
    long long* host_total = pinned.p ? reinterpret_cast<long long*>(pinned.p + 2 * bound) : nullptr;
    cudaEvent_t const* formatted = io.events;                             // [2]: chunk formatted, its byte count copied
    cudaEvent_t const* copied = io.events + 2;                            // [2]: chunk copied to pinned memory
    long long bytes[2] = {0, 0};
    const int K = (int)chunks.size();
    for (int k = 0; k <= K + 1 && e == cudaSuccess; ++k) {
        if (k < K && chunks[k].n) {
            const Chunk& c = chunks[k];
            const int slot = k & 1;
            const unsigned tiles = (unsigned)((c.n + TEXT_TILE - 1) / TEXT_TILE);
            const TextSegment& sg = segs[c.seg];
            const uint32_t in = (uint32_t)(sg.ids ? sg.cols : sg.rows);
            const ChunkArgs a{c.n, Place{c.g0 / in, (uint32_t)(c.g0 % in)}, in, in > 1 ? ~0ull / in + 1 : 0};
            if ((e = cudaStreamWaitEvent(io.stream, copied[slot], 0)) != cudaSuccess) break;     // chunk k - 2 is out
            text_length_kernel<<<tiles, TEXT_THREADS, 0, io.stream>>>(sg, a, dev_tiles[slot]);
            if ((e = launched()) != cudaSuccess) break;
            text_write_kernel<<<tiles, TEXT_THREADS, 0, io.stream>>>(sg, a, dev_tiles[slot], dev_text[slot], dev_total + slot);
            if ((e = launched()) != cudaSuccess) break;
            if ((e = cudaMemcpyAsync(host_total + slot, dev_total + slot, sizeof(long long), cudaMemcpyDeviceToHost,
                                     io.stream)) != cudaSuccess) break;
            if ((e = cudaEventRecord(formatted[slot], io.stream)) != cudaSuccess) break;
        }
        const int j = k - 1;
        if (j >= 0 && j < K && chunks[j].n) {
            const int slot = j & 1;
            if ((e = cudaEventSynchronize(formatted[slot])) != cudaSuccess) break;
            bytes[slot] = host_total[slot];
            if ((e = cudaStreamWaitEvent(io.copy_stream, formatted[slot], 0)) != cudaSuccess) break;
            if ((e = cudaMemcpyAsync(host_text[slot], dev_text[slot], (size_t)bytes[slot], cudaMemcpyDeviceToHost,
                                     io.copy_stream)) != cudaSuccess) break;
            if ((e = cudaEventRecord(copied[slot], io.copy_stream)) != cudaSuccess) break;
        }
        const int i = k - 2;
        if (i >= 0 && i < K) {
            const char* src;
            size_t len;
            if (chunks[i].n) {
                const int slot = i & 1;
                if ((e = cudaEventSynchronize(copied[slot])) != cudaSuccess) break;
                src = host_text[slot];
                len = (size_t)bytes[slot];
            } else {
                src = chunks[i].host.data();
                len = chunks[i].host.size();
            }
            if (std::fwrite(src, 1, len, io.file) != len) {
                *io_errno = errno ? errno : EIO;
                break;
            }
        }
    }
    // nothing may still read the buffers when they are released
    const cudaError_t e1 = cudaStreamSynchronize(io.copy_stream);
    const cudaError_t e2 = cudaStreamSynchronize(io.stream);
    if (e == cudaSuccess) e = e1 != cudaSuccess ? e1 : e2;
    return e;
}

}  // namespace mb
