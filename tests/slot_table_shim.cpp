// A C face of the LM engine's slot table (voicecraft_b200/csrc/slot_table.h) for test_slot_table.py, which compiles it
// with the host compiler and drives it through ctypes.
#include "../voicecraft_b200/csrc/slot_table.h"

using vcb::SlotRec;
using vcb::SlotTable;

namespace {
SlotTable& T(void* t) { return *static_cast<SlotTable*>(t); }
}  // namespace

extern "C" {

void* st_new(int n_pages, int max_slots, int max_pages_per_slot, int page_tokens) {
    return new SlotTable(n_pages, max_slots, max_pages_per_slot, page_tokens);
}

void st_delete(void* t) { delete static_cast<SlotTable*>(t); }

long long st_prompt_pages(void* t, int total, int copies) { return static_cast<long long>(T(t).prompt_pages(total, copies)); }

int st_open_pages(void* t, int total, int copies) { return T(t).open_pages(total, copies); }

// f: seq_len, copies, shared, rng, edit, final_frames; align: n_align head masks
int st_open(void* t, int slot, int n_pages, int leader, int sp, const int* f, const uint32_t* align, int n_align) {
    SlotRec r;
    r.seq_len = f[0];
    r.copies = f[1];
    r.shared = f[2];
    r.rng = static_cast<char>(f[3]);
    r.edit = static_cast<char>(f[4]);
    r.final_frames = f[5];
    r.align.assign(align, align + n_align);
    return T(t).open(slot, r, n_pages, leader, static_cast<char>(sp));
}

int st_close(void* t, int slot) { return T(t).close(slot); }

// grow: (slot, page count) pairs, *n_grow of them
int st_plan_growth(void* t, const int32_t* slots, int n, int* grow, int* n_grow, long long* need) {
    std::vector<std::pair<int, int>> g;
    size_t nd = 0;
    const int rc = T(t).plan_growth(slots, n, g, nd);
    for (size_t i = 0; i < g.size(); ++i) {
        grow[2 * i] = g[i].first;
        grow[2 * i + 1] = g[i].second;
    }
    *n_grow = static_cast<int>(g.size());
    *need = static_cast<long long>(nd);
    return rc;
}

void st_grow_to(void* t, int slot, int n_pages) { T(t).grow_to(slot, n_pages); }

// the record fields the engine updates in place: seq_len (decode steps), final_frames (vcb_poll_frames)
void st_update(void* t, int slot, int seq_len, int final_frames) {
    T(t)[slot].seq_len = seq_len;
    T(t)[slot].final_frames = final_frames;
}

int st_free_list(void* t, int* out) {
    const std::vector<int>& f = T(t).free_list();
    std::copy(f.begin(), f.end(), out);
    return static_cast<int>(f.size());
}

int st_page_refs(void* t, int page) { return T(t).page_refs(page); }

int st_groups_left(void* t) { return static_cast<int>(T(t).groups_left()); }

int st_sp_bits(void* t, int slot) { return T(t).sp_bits(slot); }

int st_is_open(void* t, int slot) { return T(t).is_open(slot); }

void st_page_row(void* t, int slot, int* out) {
    const std::vector<int> row = T(t).page_row(slot);
    std::copy(row.begin(), row.end(), out);
}

// f: group, page count, seq_len, copies, shared, rng, edit, final_frames, head-mask count; then the pages and masks
void st_rec(void* t, int slot, int* f, int* pages, uint32_t* align) {
    const SlotRec& r = T(t)[slot];
    const int v[] = {r.group, static_cast<int>(r.pages.size()), r.seq_len, r.copies, r.shared, r.rng, r.edit,
                     r.final_frames, static_cast<int>(r.align.size())};
    std::copy(v, v + 9, f);
    std::copy(r.pages.begin(), r.pages.end(), pages);
    std::copy(r.align.begin(), r.align.end(), align);
}

}  // extern "C"
