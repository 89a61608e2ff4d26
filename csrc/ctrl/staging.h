// Reuse of a device context's staging regions (client_dev.h): the pinned ring, the device
// scratch and the zeroed counters.  Each region is a bump allocator over a fixed buffer, and a
// launch uses the bytes handed out since the previous launch.  When the allocator comes round
// to bytes again, the launches that used them one lap earlier must have completed; only those
// are waited for, so the launches of the current lap keep running.
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

}  // namespace istore
