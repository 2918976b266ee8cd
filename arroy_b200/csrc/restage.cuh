// restage.cuh — keeping the staged item matrix across an update (arroy_b200_stage_items_delta).
//
// An update keeps most rows of the resident matrix and only changes where they sit: row = rank of the id, so a deleted item
// shifts every later row down by one and an inserted one shifts them up. Both id lists ascend, hence old row -> new row is a
// strictly increasing map over the kept rows, and the move is a stable merge of the matrix onto itself.
//
//   stage_delta_plan   host: which old row every new row keeps (or -1: its vector comes from the host)
//   restage_move_pieces  host: the kept rows that change place, cut into pieces of consecutive rows and grouped into windows
//                      that fit the scratch buffer, in an order that never overwrites a row before it is read
//   restage_upload_pieces  host: the same for the rows that come from the host (host -> scratch -> their rows)
//   restage_copy_rows_kernel   device: one CTA per piece, 16-byte copies; phase 0 matrix -> scratch, phase 1 scratch -> matrix
//
// Why the order is safe. Call a maximal stretch of kept rows whose shift (new row - old row) has one sign a region; rows with
// shift 0 stay where they are and separate regions. Destinations and sources both increase strictly, so the destinations of
// one region lie strictly between the rows of its neighbours: a region never writes a row another region still has to read.
// Inside a region that moves down every destination lies below its source, so going front to back a window only overwrites
// rows that it or an earlier window has read already; a region that moves up is the mirror image, back to front. Inside one
// window every row is read (phase 0) before any is written (phase 1), two launches on one stream.
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

namespace ab {

// out_src[r] = the old row whose vector new row r keeps, -1 when it has to be uploaded: ids that are not in old_ids, and ids
// listed in changed_ids. All three lists ascend strictly. Returns the number of -1 entries.
inline uint64_t stage_delta_plan(const uint32_t* old_ids, uint64_t n_old, const uint32_t* new_ids, uint64_t n_new, const uint32_t* changed_ids, uint64_t n_changed,
                                 int64_t* out_src) {
    uint64_t o = 0, ch = 0, n_upload = 0;
    for (uint64_t r = 0; r < n_new; ++r) {
        const uint32_t id = new_ids[r];
        while (o < n_old && old_ids[o] < id) ++o;
        while (ch < n_changed && changed_ids[ch] < id) ++ch;
        const bool kept = o < n_old && old_ids[o] == id && !(ch < n_changed && changed_ids[ch] == id);
        out_src[r] = kept ? (int64_t)o : -1;
        n_upload += kept ? 0 : 1;
    }
    return n_upload;
}

// consecutive rows that travel together: matrix rows [src, src + len) -> scratch rows [slot, slot + len) -> matrix rows
// [dst, dst + len). For uploaded rows only slot and dst are used.
struct RestagePiece { uint32_t src, dst, len, slot; };
struct RestageWindow { uint64_t piece0, n_pieces; };

struct RestagePieces {
    std::vector<RestagePiece> pieces;
    std::vector<RestageWindow> windows;
    uint64_t rows = 0;
};

namespace restage_detail {
struct Packer {   // fills windows of at most window_rows scratch rows with pieces of at most piece_rows rows
    RestagePieces& out;
    const uint64_t window_rows, piece_rows;
    uint64_t used = 0;
    void add(uint64_t src, uint64_t dst, uint64_t len, bool from_back) {
        out.rows += len;
        while (len) {
            if (out.windows.empty() || used == window_rows) { out.windows.push_back({out.pieces.size(), 0}); used = 0; }
            const uint64_t take = std::min<uint64_t>({len, piece_rows, window_rows - used});
            const uint64_t off = from_back ? len - take : 0;
            out.pieces.push_back({(uint32_t)(src + off), (uint32_t)(dst + off), (uint32_t)take, (uint32_t)used});
            out.windows.back().n_pieces += 1;
            used += take;
            if (!from_back) { src += take; dst += take; }
            len -= take;
        }
    }
};
}  // namespace restage_detail

// The kept rows whose place changes (src[r] >= 0 and src[r] != r), as windows to run in the order given: first every row that
// moves down, front to back, then every row that moves up, back to front (see the head of this file).
inline RestagePieces restage_move_pieces(const int64_t* src, uint64_t n_new, uint64_t window_rows, uint64_t piece_rows) {
    RestagePieces out;
    restage_detail::Packer pk{out, window_rows, piece_rows};
    for (uint64_t r = 0; r < n_new;) {   // down: new row < old row
        if (src[r] <= (int64_t)r) { ++r; continue; }
        uint64_t e = r + 1;
        while (e < n_new && src[e] == src[e - 1] + 1) ++e;
        pk.add((uint64_t)src[r], r, e - r, false);
        r = e;
    }
    for (uint64_t e = n_new; e > 0;) {   // up: new row > old row
        if (src[e - 1] < 0 || src[e - 1] >= (int64_t)(e - 1)) { --e; continue; }
        uint64_t r = e - 1;
        while (r > 0 && src[r - 1] >= 0 && src[r - 1] == src[r] - 1) --r;
        pk.add((uint64_t)src[r], r, e - r, true);
        e = r;
    }
    return out;
}

// The rows to upload (src[r] < 0), in ascending order: upload row k of a window goes to scratch row `slot` first.
inline RestagePieces restage_upload_pieces(const int64_t* src, uint64_t n_new, uint64_t window_rows, uint64_t piece_rows) {
    RestagePieces out;
    restage_detail::Packer pk{out, window_rows, piece_rows};
    for (uint64_t r = 0; r < n_new;) {
        if (src[r] >= 0) { ++r; continue; }
        uint64_t e = r + 1;
        while (e < n_new && src[e] < 0) ++e;
        pk.add(0, r, e - r, false);
        r = e;
    }
    return out;
}

constexpr int RESTAGE_THREADS = 256;

// One CTA per piece (grid-stride), rows as 16-byte words (u4_per_row = row_bytes / 16, any row size the library stages).
// phase 0: matrix rows [src, +len) -> scratch rows [slot, +len); phase 1: scratch rows [slot, +len) -> matrix rows [dst, +len).
__global__ void __launch_bounds__(RESTAGE_THREADS) restage_copy_rows_kernel(uint4* __restrict__ matrix, uint4* __restrict__ scratch, const RestagePiece* __restrict__ pieces,
                                                                            uint64_t n_pieces, uint32_t u4_per_row, int phase) {
    for (uint64_t p = blockIdx.x; p < n_pieces; p += gridDim.x) {
        const RestagePiece pc = pieces[p];
        const uint4* from = phase == 0 ? matrix + (size_t)pc.src * u4_per_row : scratch + (size_t)pc.slot * u4_per_row;
        uint4* to = phase == 0 ? scratch + (size_t)pc.slot * u4_per_row : matrix + (size_t)pc.dst * u4_per_row;
        const uint32_t words = pc.len * u4_per_row;   // <= 64 KB / 16, or one row
        uint32_t i = threadIdx.x;
        for (; i + 3 * RESTAGE_THREADS < words; i += 4 * RESTAGE_THREADS) {   // four loads in flight per thread
            const uint4 a = __ldcs(from + i), b = __ldcs(from + i + RESTAGE_THREADS), c = __ldcs(from + i + 2 * RESTAGE_THREADS), d = __ldcs(from + i + 3 * RESTAGE_THREADS);
            to[i] = a; to[i + RESTAGE_THREADS] = b; to[i + 2 * RESTAGE_THREADS] = c; to[i + 3 * RESTAGE_THREADS] = d;
        }
        for (; i < words; i += RESTAGE_THREADS) to[i] = __ldcs(from + i);
    }
}

}  // namespace ab
