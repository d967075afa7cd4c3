// Where does the next push segment go in the payload ring? Pure host arithmetic, kept apart from
// b9gpu.cu so that the CPU tests (tests/host_shim/ring_place_shim.cpp) run the very function the
// library uses.
//
// Model: live segments sit in FIFO order; the oldest one starts at `oldest`, the next free byte is
// `wp` (256-byte aligned, like every segment start). Either the live bytes are [oldest, wp)
// (unwrapped) or they are [oldest, ring end) + [0, wp) (wrapped, free space is [wp, oldest)).
// wp == oldest is ambiguous from the two positions alone — an exactly full, wrapped ring and a ring
// whose live segments all hold zero bytes look the same — so the caller says whether any live
// segment holds bytes (`live_bytes`): with bytes pending the ring is FULL, never empty.
// (Round 1 decided the tie as "empty" and let the next push DMA over pending payload.)
#pragma once
#include <stdint.h>

constexpr uint64_t B9_SEG_ALIGN = 256;

static inline uint64_t b9_seg_span(uint64_t bytes) { return (bytes + B9_SEG_ALIGN - 1) & ~(B9_SEG_ALIGN - 1); }

// returns 1 and *start when a segment of `bytes` fits, 0 when the ring cannot take it now
static inline int b9_ring_place(uint64_t ring_bytes, int have_segments, uint64_t oldest, uint64_t wp, uint64_t live_bytes,
                                uint64_t bytes, uint64_t* start) {
    const uint64_t need = b9_seg_span(bytes);
    if (need > ring_bytes) return 0;
    if (!have_segments) { *start = 0; return 1; }
    if (live_bytes == 0) {                       // only zero-byte segments are live: positions carry no data
        if (wp + need <= ring_bytes) { *start = wp; return 1; }
        *start = 0; return 1;
    }
    if (wp == oldest) {                          // bytes pending and the positions meet: exactly full
        if (need == 0) { *start = wp; return 1; }
        return 0;
    }
    if (wp > oldest) {                           // live data is [oldest, wp)
        if (wp + need <= ring_bytes) { *start = wp; return 1; }
        if (need <= oldest) { *start = 0; return 1; }   // wrap, leaving the tail gap unused (need == oldest: full afterwards)
        return 0;
    }
    if (wp + need <= oldest) { *start = wp; return 1; }  // wrapped already: free is [wp, oldest)
    return 0;
}

// The free byte ranges of the same model, in the order b9_ring_place tries them: reg[i] = [start, end). Returns their
// number (0, 1 or 2). A segment may fill a range exactly; the next free byte after it is then min(its start +
// b9_seg_span(bytes), the range's end) — the re-push of retried tasks places its segments this way, so that tasks whose
// bytes were exactly the window's fit back into a ring that was exactly full.
static inline int b9_ring_free_ranges(uint64_t ring_bytes, int have_segments, uint64_t oldest, uint64_t wp, uint64_t live_bytes,
                                      uint64_t reg[2][2]) {
    if (!have_segments) { reg[0][0] = 0; reg[0][1] = ring_bytes; return 1; }
    if (live_bytes == 0) { reg[0][0] = 0; reg[0][1] = ring_bytes; return 1; }   // positions carry no data
    if (wp == oldest) return 0;
    if (wp > oldest) {
        int n = 0;
        if (wp < ring_bytes) { reg[n][0] = wp; reg[n][1] = ring_bytes; ++n; }
        if (oldest > 0) { reg[n][0] = 0; reg[n][1] = oldest; ++n; }
        return n;
    }
    reg[0][0] = wp; reg[0][1] = oldest;
    return 1;
}
