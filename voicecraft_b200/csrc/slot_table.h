// Host bookkeeping of the LM engine's slots (DESIGN.md section 3): one record per slot, the best-of-N groups and the KV
// page allocator, with the rules that decide which pages a slot holds.  No CUDA: the engine keeps every device mirror
// (SlotState / GroupState, sp_tab, the page table, align_masks) and writes them from these records.
#pragma once
#include "../../include/vcb200.h"

#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <utility>
#include <vector>

namespace vcb {

// a group's bits: it was prefilled with sampling parameters of its own; they turn on repetition-aware sampling or a
// length bound (its steps run the sampler instance with those controls); they turn on repetition-aware sampling (its
// steps take no caller noise)
enum : char { GROUP_SP_OWN = 1, GROUP_SP_CTL = 2, GROUP_SP_RAS = 4 };

// One slot's host state; a closed slot's record equals a fresh one
struct SlotRec {
    int group = -1;                   // -1: closed
    std::vector<int> pages;           // the slot's page-table row (a best-of-N member shares its leader's full prompt pages)
    int seq_len = 0;                  // upper bound of SlotState::seq_len: the attention grid, and the position the next
                                      // step writes (page growth)
    int copies = 0;                   // n_copies of the slot's prompt (best-of-N group size)
    int shared = 0;                   // full prompt pages the slot shares with its group (0: none)
    char rng = 0;                     // the slot's group generates its own sampling noise
    char edit = 0;                    // masked spans of the slot's edit prompt (0: a TTS prompt)
    int final_frames = 0;             // final frames vcb_poll_frames last reported for the slot (they only grow)
    std::vector<uint32_t> align;      // the head masks [L] its align_masks row holds (empty: off, or no alignment log)
};

class SlotTable {
public:
    SlotTable() = default;
    // the free list starts as n_pages - 1 .. 0, so pages are taken 0, 1, 2, ...; groups likewise
    SlotTable(int n_pages, int max_slots, int max_pages_per_slot, int page_tokens)
        : page_(page_tokens), max_pages_(max_pages_per_slot), refs_(n_pages, 0), slots_(max_slots),
          members_(max_slots, 0), group_sp_(max_slots, 0) {
        for (int p = n_pages - 1; p >= 0; --p) free_pages_.push_back(p);
        for (int g = max_slots - 1; g >= 0; --g) free_groups_.push_back(g);
    }

    const SlotRec& operator[](int slot) const { return slots_[slot]; }
    SlotRec& operator[](int slot) { return slots_[slot]; }
    bool is_open(int slot) const { return slot >= 0 && slot < static_cast<int>(slots_.size()) && slots_[slot].group >= 0; }
    char sp_bits(int slot) const { return group_sp_[slots_[slot].group]; }
    const std::vector<int>& free_list() const { return free_pages_; }
    size_t groups_left() const { return free_groups_.size(); }
    int page_refs(int page) const { return refs_[page]; }

    // page-list length of a one-copy utterance that writes positions [0, pos]: whole growth chunks, at most
    // max_pages_per_slot
    int grown_pages(int pos) const {
        const int want = pos / page_ + 1;
        return std::min(max_pages_, (want + VCB_KV_GROW_PAGES - 1) / VCB_KV_GROW_PAGES * VCB_KV_GROW_PAGES);
    }
    // pages each slot of a prompt of `total` positions opens with: a one-copy prompt the pages of its positions (steps
    // grow them), a best-of-N member its full reservation
    int open_pages(int total, int copies) const { return copies == 1 ? grown_pages(total - 1) : max_pages_; }
    // pages the prefill of such a prompt takes from the free list: the leader's full prompt pages are counted once
    size_t prompt_pages(int total, int copies) const {
        const size_t per_slot = open_pages(total, copies);
        return per_slot + static_cast<size_t>(copies - 1) * (per_slot - total / page_);
    }

    // Opens a closed slot with record r (its pages and group are ignored) and n_pages pages.  leader < 0: the slot leads
    // a new group with the GROUP_SP_* bits sp; else it joins the leader's group and shares the leader's first r.shared
    // pages.  The caller checked that a group and the pages are free.  Returns the group id.
    int open(int slot, SlotRec r, int n_pages, int leader, char sp) {
        if (leader < 0) {
            r.group = free_groups_.back();
            free_groups_.pop_back();
            group_sp_[r.group] = sp;
        } else {
            r.group = slots_[leader].group;
        }
        ++members_[r.group];
        r.pages.clear();
        if (leader >= 0) r.pages.assign(slots_[leader].pages.begin(), slots_[leader].pages.begin() + r.shared);
        for (int p : r.pages) ++refs_[p];
        slots_[slot] = std::move(r);
        grow_to(slot, n_pages);
        return slots_[slot].group;
    }

    // Closes an open slot: its pages go back once no slot holds them, in page-list order.  Returns its group id when it
    // was the group's last member (the id is free again), else -1.
    int close(int slot) {
        const int g = slots_[slot].group;
        for (int p : slots_[slot].pages)
            if (--refs_[p] == 0) free_pages_.push_back(p);
        slots_[slot] = SlotRec();
        if (--members_[g] > 0) return -1;
        group_sp_[g] = 0;
        free_groups_.push_back(g);
        return g;
    }

    // Page growth of a decode step, planned without touching any state: every listed one-copy slot needs a page for
    // position seq_len (it writes at most there).  Slots take whole chunks when the free list covers them all, else the
    // pages they need.  grow: (slot, new page count).  VCB_ERR_KV_FULL with grow empty when the free list cannot cover
    // even that; need is then the pages the slots lack in all.
    int plan_growth(const int32_t* slots, int n, std::vector<std::pair<int, int>>& grow, size_t& need) const {
        grow.clear();
        need = 0;
        size_t chunked = 0;
        std::vector<int> want;
        for (int i = 0; i < n; ++i) {
            const int s = slots[i];
            const SlotRec& r = slots_[s];
            const int have = static_cast<int>(r.pages.size());
            const int need_s = std::min(max_pages_, r.seq_len / page_ + 1);
            if (r.copies != 1 || need_s <= have ||
                std::any_of(grow.begin(), grow.end(), [s](const std::pair<int, int>& g) { return g.first == s; }))
                continue;
            const int chunk = grown_pages(r.seq_len);
            grow.emplace_back(s, chunk);
            want.push_back(need_s);
            need += need_s - have;
            chunked += chunk - have;
        }
        if (need > free_pages_.size()) {
            grow.clear();
            return VCB_ERR_KV_FULL;
        }
        if (chunked > free_pages_.size())
            for (size_t i = 0; i < grow.size(); ++i) grow[i].second = want[i];
        return 0;
    }

    // takes pages from the back of the free list until the slot holds n_pages (a planned growth, or an open)
    void grow_to(int slot, int n_pages) {
        auto& pg = slots_[slot].pages;
        while (static_cast<int>(pg.size()) < n_pages) {
            pg.push_back(free_pages_.back());
            free_pages_.pop_back();
            ++refs_[pg.back()];
        }
    }

    // a page-table row of `slot` as the device holds it: the slot's pages, then page 0 (never read: attention and the QKV
    // epilogues read positions up to the one a step writes)
    std::vector<int> page_row(int slot) const {
        std::vector<int> row(slots_[slot].pages);
        row.resize(max_pages_, 0);
        return row;
    }

private:
    int page_ = 64, max_pages_ = 0;
    std::vector<int> free_pages_;     // taken from the back
    std::vector<int> refs_;           // slots whose page list holds the page
    std::vector<SlotRec> slots_;
    std::vector<int> free_groups_;
    std::vector<int> members_;        // open slots of each group
    std::vector<char> group_sp_;      // GROUP_SP_* bits of each group (sp_tab holds its parameters)
};

}  // namespace vcb
