// Reuse of a device context's staging regions (client_dev.h): the pinned ring, the device
// scratch and the zeroed counters; and how many blocks one launch stages.  Each region is a
// bump allocator over a fixed buffer, and a launch uses the bytes handed out since the
// previous launch.  When the allocator comes round to bytes again, the launches that used them
// one lap earlier must have completed; only those are waited for, so the launches of the
// current lap keep running.
//
// Positions are byte counts since the context was created: they never wrap, and the offset
// into a region of `size` bytes is pos % size.  No CUDA in here (Event is a plain handle and the
// wait is the caller's), so the arithmetic is unit-tested on the CPU.
#pragma once

#include <cstddef>
#include <cstdint>
#include <deque>
#include <vector>

namespace istore {

template <typename Event, int R>
class StagingFifo {
   public:
    StagingFifo() {
        for (uint64_t& f : first_) f = kNone;
    }
    // Position of `bytes` in region r: the next free bytes, or the start of the next lap when
    // they do not fit before the end of the region.  Before it returns, every launch that may
    // still use those bytes has been passed to wait(ev) and retired, oldest first.
    template <typename Wait>
    uint64_t place(int r, size_t bytes, size_t size, Wait&& wait) {
        uint64_t at = pos_[r];
        if (at % size + bytes > size) at += size - at % size;
        if (at + bytes > size) {
            // The same bytes were handed out last below at + bytes - size.  A launch that used
            // region r and began below that may hold them; launches begin in FIFO order.
            const uint64_t reused_end = at + bytes - size;
            size_t n = 0;
            for (size_t i = 0; i < fifo_.size() && fifo_[i].begin[r] < reused_end; ++i)
                if (fifo_[i].end[r] > fifo_[i].begin[r]) n = i + 1;
            for (; n; --n) {
                wait(fifo_.front().ev);
                retire_front();
            }
        }
        if (first_[r] == kNone) first_[r] = at;
        pos_[r] = at + bytes;
        return at;
    }
    // A launch that uses every byte placed since the previous push; `ev` completes with it.
    void push(Event ev) {
        Launch l{ev, {}, {}};
        for (int r = 0; r < R; ++r) {
            l.begin[r] = first_[r] == kNone ? pos_[r] : first_[r];
            l.end[r] = pos_[r];
            first_[r] = kNone;
        }
        fifo_.push_back(l);
    }
    // Every launch pushed so far has completed.
    void retire_all() {
        while (!fifo_.empty()) retire_front();
    }
    // The event of a retired launch, to be recorded again; false when there is none.
    bool take_free(Event* ev) {
        if (free_.empty()) return false;
        *ev = free_.back();
        free_.pop_back();
        return true;
    }
    size_t in_flight() const { return fifo_.size(); }

   private:
    static constexpr uint64_t kNone = ~uint64_t(0);
    struct Launch {
        Event ev;
        uint64_t begin[R];  // the launch used [begin, end) of each region
        uint64_t end[R];
    };
    void retire_front() {
        free_.push_back(fifo_.front().ev);
        fifo_.pop_front();
    }
    std::deque<Launch> fifo_;
    std::vector<Event> free_;
    uint64_t pos_[R] = {};
    uint64_t first_[R];  // first byte placed since the last push, kNone when there is none
};

// The flag slots of layered reads (client_dev.h: DevCtx::group_flags).  Reader seq = 1, 2, ...
// owns slot seq % Slots.  A slot's flag words only grow and a consumer waits for
// flag >= seq, so a later reader's flags never un-release an earlier reader's wait, and a
// wait enqueued late is still satisfied.  A slot is handed to the next reader once the
// launches of the reader that held it one lap earlier have completed: take() passes only that
// reader to wait(ev).  No CUDA in here (Event is a plain handle), so the ring is unit-tested
// on the CPU.
template <typename Event, int Slots>
class ReaderSlots {
   public:
    // The next reader's sequence number; its slot is free to use when take() returns.
    template <typename Wait>
    uint64_t take(Wait&& wait) {
        const uint64_t seq = ++seq_;
        Slot& s = slots_[seq % Slots];
        if (s.live) {
            wait(s.ev);
            s.live = false;
        }
        return seq;
    }
    // Reader seq's launches complete with ev.  A reader that launched nothing is never waited for.
    void launched(uint64_t seq, Event ev) {
        Slot& s = slots_[seq % Slots];
        s.ev = ev;
        s.live = true;
    }
    // Every reader has completed (the device context was drained).
    void retire_all() {
        for (Slot& s : slots_) s.live = false;
    }
    uint64_t last() const { return seq_; }
    static uint32_t slot_of(uint64_t seq) { return uint32_t(seq % Slots); }

   private:
    struct Slot {
        Event ev{};
        bool live = false;
    };
    Slot slots_[Slots];
    uint64_t seq_ = 0;
};

// One launch's share of a call's keys, taken from the front of the `left` keys still to go:
// at most max_blocks keys, whose staged bytes stay within max_bytes.  A key stages its bytes
// zero padded to a multiple of 8 (an empty key takes 8) plus 16 bytes of offset, length and
// destination.  The batch holds at least one key, so a call always makes progress: a key
// above the bound is staged on its own.  key_len(i) is the length of the i-th key from the front.
struct KeyBatch {
    size_t n = 0;          // keys
    size_t key_bytes = 0;  // their padded bytes
};
template <typename KeyLen>
KeyBatch key_batch(size_t left, size_t max_blocks, size_t max_bytes, KeyLen&& key_len) {
    KeyBatch b;
    size_t staged = 0;
    for (; b.n < left && b.n < max_blocks; ++b.n) {
        const size_t len = key_len(b.n);
        const size_t padded = ((len ? len : 1) + 7) & ~size_t(7);
        staged += padded + 16;
        if (staged > max_bytes && b.n > 0) break;
        b.key_bytes += padded;
    }
    return b;
}

// Gathered blocks of nparts parts: at most 2^30 work items per launch (a chunk is >= 16 KB or
// a whole part), and never fewer than one block.
inline size_t gather_max_blocks(size_t max_blocks, uint32_t nparts, uint32_t part_bytes) {
    const uint64_t items = uint64_t(nparts) * ((uint64_t(part_bytes) + 16383u) / 16384u);
    const uint64_t cap = (1ull << 30) / items;
    return cap == 0 ? 1 : cap < max_blocks ? size_t(cap) : max_blocks;
}

}  // namespace istore
