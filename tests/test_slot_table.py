"""The LM engine's host bookkeeping of slots, best-of-N groups and KV pages (voicecraft_b200/csrc/slot_table.h), compiled
for the host through slot_table_shim.cpp and called the way lm_engine.cu calls it.  Seeded random sequences of prefills
(one-copy prompts and groups, totals on and off page boundaries), decode-step growth (refusals included), releases of
group members in any order, swaps out and back in, and frame polls run against a plain-Python model of the engine's rules
as vcb_prefill, plan_growth / apply_growth, vcb_release and vcb_swap_out / vcb_swap_in wrote them out one by one; and the
Python admission's page count (_Prompt.pages) against the table's prefill reservation."""
import ctypes as C
import os
import random
import subprocess
from types import SimpleNamespace

import pytest

from voicecraft_b200 import _lib
from voicecraft_b200.voicecraft import _Prompt

HERE = os.path.dirname(os.path.abspath(__file__))
PAGE, CHUNK, L = 64, _lib.KV_GROW_PAGES, 3
FRESH = [-1, 0, 0, 0, 0, 0, 0, 0, 0]          # a closed slot's record: group, pages, seq_len, ..., head masks


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("slot_table") / "libslot_table.so")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-O1", "-shared", "-fPIC", "-o", so,
                    os.path.join(HERE, "slot_table_shim.cpp")], check=True)
    lib = C.CDLL(so)
    P, I = C.c_void_p, C.POINTER(C.c_int)
    lib.st_new.restype = P
    for name, args in (("st_delete", [P]), ("st_prompt_pages", [P, C.c_int, C.c_int]),
                       ("st_open_pages", [P, C.c_int, C.c_int]),
                       ("st_open", [P, C.c_int, C.c_int, C.c_int, C.c_int, I, C.POINTER(C.c_uint32), C.c_int]),
                       ("st_close", [P, C.c_int]), ("st_plan_growth", [P, I, C.c_int, I, I, C.POINTER(C.c_longlong)]),
                       ("st_grow_to", [P, C.c_int, C.c_int]), ("st_update", [P, C.c_int, C.c_int, C.c_int]),
                       ("st_free_list", [P, I]), ("st_page_refs", [P, C.c_int]), ("st_groups_left", [P]),
                       ("st_sp_bits", [P, C.c_int]), ("st_is_open", [P, C.c_int]), ("st_page_row", [P, C.c_int, I]),
                       ("st_rec", [P, C.c_int, I, I, C.POINTER(C.c_uint32)])):
        getattr(lib, name).argtypes = args
    lib.st_prompt_pages.restype = C.c_longlong
    return lib


def _ints(v):
    return (C.c_int * max(1, len(v)))(*v)


class Table:
    """the slot table through the shim, in the call sequences of lm_engine.cu"""

    def __init__(self, lib, n_pages, max_slots, max_pages):
        self.lib, self.n_pages, self.max_slots, self.max_pages = lib, n_pages, max_slots, max_pages
        self.t = lib.st_new(n_pages, max_slots, max_pages, PAGE)

    def close_table(self):
        self.lib.st_delete(self.t)

    def free_list(self):
        out = (C.c_int * self.n_pages)()
        return out[:self.lib.st_free_list(self.t, out)]

    def rec(self, slot):
        f, pages, align = (C.c_int * 9)(), (C.c_int * self.max_pages)(), (C.c_uint32 * L)()
        self.lib.st_rec(self.t, slot, f, pages, align)
        return list(f), pages[:f[1]], align[:f[8]]

    def state(self):
        rows = []
        for s in range(self.max_slots):
            row = (C.c_int * self.max_pages)()
            self.lib.st_page_row(self.t, s, row)
            rows.append((self.rec(s), list(row)))
        return (self.free_list(), [self.lib.st_page_refs(self.t, p) for p in range(self.n_pages)], rows,
                self.lib.st_groups_left(self.t))

    def _open(self, slot, n_pages, leader, sp, fields, align):
        return self.lib.st_open(self.t, slot, n_pages, leader, sp, _ints(fields), (C.c_uint32 * max(1, len(align)))(*align),
                                len(align))

    def prefill(self, prompts):
        """vcb_prefill: validate every prompt, then open each group's leader and its members"""
        need = sum(self.lib.st_prompt_pages(self.t, total, n) for _, n, total, *_ in prompts)
        if len(prompts) > self.lib.st_groups_left(self.t) or need > len(self.free_list()):
            return False
        for slot, n, total, sp, rng, edit, align in prompts:
            fields = [total, n, total // PAGE if n > 1 else 0, rng, edit, 0]
            n_pg = self.lib.st_open_pages(self.t, total, n)
            self._open(slot, n_pg, -1, sp, fields, align)
            for c in range(1, n):
                self._open(slot + c, n_pg, slot, 0, fields, align)
        return True

    def step(self, slots):
        """vcb_decode_step: plan the growth; unless refused, take the pages, then every listed slot advances a position"""
        grow, n_grow, need = (C.c_int * (2 * len(slots)))(), C.c_int(), C.c_longlong()
        rc = self.lib.st_plan_growth(self.t, _ints(slots), len(slots), grow, C.byref(n_grow), C.byref(need))
        plan = [(grow[2 * i], grow[2 * i + 1]) for i in range(n_grow.value)]
        if rc:
            return rc, need.value, plan
        for s, n in plan:
            self.lib.st_grow_to(self.t, s, n)
        for s in slots:
            f = self.rec(s)[0]
            self.lib.st_update(self.t, s, f[2] + 1, f[7])
        return rc, None, plan

    def poll(self, slot, frames):
        f = self.rec(slot)[0]
        self.lib.st_update(self.t, slot, f[2], max(f[7], frames))

    def release(self, slot, n):
        """vcb_release: close the open slots of [slot, slot + n); the group ids that came back"""
        back = [self.lib.st_close(self.t, s) for s in range(slot, slot + n) if self.lib.st_is_open(self.t, s)]
        return [g for g in back if g >= 0]

    def swap_out(self, slot):
        """vcb_swap_out: the record without its pages, the written pages and the group's bits; then the release"""
        f, pages, align = self.rec(slot)
        snap = (f[2:8], align, min(len(pages), -(-f[2] // PAGE)), self.lib.st_sp_bits(self.t, slot))
        return snap, self.release(slot, 1)

    def swap_in(self, snap, slot):
        fields, align, n_pages, sp = snap
        if self.lib.st_groups_left(self.t) == 0 or n_pages > len(self.free_list()):
            return False
        self._open(slot, n_pages, -1, sp, fields, align)
        return True


class Parent:
    """the engine's rules as its parallel per-slot containers kept them (vcb_create, vcb_prefill, plan_growth /
    apply_growth, vcb_decode_step, vcb_poll_frames, vcb_release, vcb_swap_out / vcb_swap_in)"""

    def __init__(self, n_pages, max_slots, max_pages):
        self.max_pages = max_pages
        self.free_pages = list(range(n_pages - 1, -1, -1))
        self.page_refs = [0] * n_pages
        self.slot_pages = [[] for _ in range(max_slots)]
        self.slot_group = [-1] * max_slots
        self.free_groups = list(range(max_slots - 1, -1, -1))
        self.group_sp = [0] * max_slots
        self.rec = {}          # open slot -> [h_seq_len, slot_copies, slot_shared, slot_rng, slot_edit, slot_final], masks

    def grown_pages(self, pos):
        return min(self.max_pages, (pos // PAGE + 1 + CHUNK - 1) // CHUNK * CHUNK)

    def take(self, pages):
        pages.append(self.free_pages.pop())
        self.page_refs[pages[-1]] += 1

    def prefill(self, prompts):
        need = 0
        for _, n, total, *_ in prompts:
            need += self.grown_pages(total - 1) if n == 1 else self.max_pages + (n - 1) * (self.max_pages - total // PAGE)
        if len(prompts) > len(self.free_groups) or need > len(self.free_pages):
            return False
        for slot0, n, total, sp, rng, edit, align in prompts:
            gid = self.free_groups.pop()
            self.group_sp[gid] = sp
            shared = total // PAGE
            for c in range(n):
                slot = slot0 + c
                self.slot_group[slot] = gid
                self.rec[slot] = ([total, n, shared if n > 1 else 0, rng, edit, 0], list(align))
                pg = self.slot_pages[slot] = []
                for p in range(self.grown_pages(total - 1) if n == 1 else self.max_pages):
                    if c > 0 and p < shared:
                        pg.append(self.slot_pages[slot0][p])
                        self.page_refs[pg[-1]] += 1
                    else:
                        self.take(pg)
        return True

    def step(self, slots):
        grow, want, need, chunked = [], [], 0, 0
        for s in slots:
            have, seq = len(self.slot_pages[s]), self.rec[s][0][0]
            need_s = min(self.max_pages, seq // PAGE + 1)
            if self.rec[s][0][1] != 1 or need_s <= have or any(g[0] == s for g in grow):
                continue
            chunk = self.grown_pages(seq)
            grow.append([s, chunk])
            want.append(need_s)
            need += need_s - have
            chunked += chunk - have
        if need > len(self.free_pages):
            return _lib.VCB_ERR_KV_FULL, need, []
        self.exact = chunked > len(self.free_pages)
        if self.exact:
            for g, w in zip(grow, want):
                g[1] = w
        for s, n in grow:
            while len(self.slot_pages[s]) < n:
                self.take(self.slot_pages[s])
        for s in slots:
            self.rec[s][0][0] += 1
        return 0, None, [tuple(g) for g in grow]

    def poll(self, slot, frames):
        self.rec[slot][0][5] = max(self.rec[slot][0][5], frames)

    def release(self, slot, n):
        gid = -1
        for s in range(slot, slot + n):
            if s < 0 or s >= len(self.slot_group) or self.slot_group[s] < 0:
                continue
            gid, self.slot_group[s] = self.slot_group[s], -1
            for p in self.slot_pages[s]:
                self.page_refs[p] -= 1
                if self.page_refs[p] == 0:
                    self.free_pages.append(p)
            self.slot_pages[s] = []
            del self.rec[s]
        if gid >= 0 and gid not in self.slot_group:
            self.free_groups.append(gid)
            self.group_sp[gid] = 0
            return [gid]
        return []

    def swap_out(self, slot):
        fields, align = self.rec[slot]
        snap = (list(fields), align, min(len(self.slot_pages[slot]), -(-fields[0] // PAGE)),
                self.group_sp[self.slot_group[slot]])
        return snap, self.release(slot, 1)

    def swap_in(self, snap, slot):
        fields, align, n_pages, sp = snap
        if not self.free_groups or n_pages > len(self.free_pages):
            return False
        gid = self.free_groups.pop()
        self.slot_group[slot] = gid
        self.slot_pages[slot] = []
        for _ in range(n_pages):
            self.take(self.slot_pages[slot])
        self.rec[slot] = (list(fields[:1]) + [1, 0] + list(fields[3:]), align)
        self.group_sp[gid] = sp
        return True


def _check(tab, par):
    free, refs, rows, groups_left = tab.state()
    assert free == par.free_pages and refs == par.page_refs and groups_left == len(par.free_groups)
    assert len(set(free)) == len(free) and all((p in free) != (refs[p] > 0) for p in range(tab.n_pages))
    for s, ((f, pages, align), row) in enumerate(rows):
        assert row == (par.slot_pages[s] + [0] * tab.max_pages)[:tab.max_pages], s
        if par.slot_group[s] < 0:
            assert f == FRESH and pages == [] and align == [], s
            continue
        fields, masks = par.rec[s]
        assert (f[0], pages, f[2:8], align) == (par.slot_group[s], par.slot_pages[s], fields, masks), s
        assert tab.lib.st_sp_bits(tab.t, s) == par.group_sp[par.slot_group[s]], s


def _total(rng, max_pages):
    """prompt positions: on, just before or just after a page boundary, or anywhere"""
    top = PAGE * max_pages
    t = rng.randint(1, max_pages) * PAGE + rng.choice([-1, 0, 1]) if rng.random() < 0.5 else rng.randint(2, top)
    return min(max(t, 2), top)


def _run(lib, seed, seen):
    rng = random.Random(seed)
    max_slots, max_pages = rng.randint(3, 8), rng.randint(1, 9)
    n_pages = max_slots * max_pages if seed % 4 == 0 else rng.randint(max_pages, max_slots * max_pages)
    tab, par = Table(lib, n_pages, max_slots, max_pages), Parent(n_pages, max_slots, max_pages)
    snaps = []
    try:
        for _ in range(400):
            opened = [s for s in range(max_slots) if par.slot_group[s] >= 0]
            op = rng.choices(["prefill", "step", "release", "swap_out", "swap_in", "poll"], [3, 6, 3, 1, 1, 1])[0]
            before, refused = tab.state(), False
            if op == "prefill":
                prompts, claimed = [], set()
                for _ in range(rng.choice([1, 1, 2])):
                    n = rng.choice([1, 1, 2, 3, 4])
                    starts = [s for s in range(max_slots - n + 1)
                              if all(par.slot_group[s + c] < 0 and s + c not in claimed for c in range(n))]
                    if starts:
                        s = rng.choice(starts)
                        claimed.update(range(s, s + n))
                        align = [] if rng.random() < 0.6 else [rng.randint(0, 3) for _ in range(L - 1)] + [1]
                        prompts.append((s, n, _total(rng, max_pages), rng.choice([0, 1, 3, 5, 7]), rng.randint(0, 1),
                                        rng.choice([0, 0, 2]), align))
                if not prompts:
                    continue
                done = par.prefill(prompts)
                assert tab.prefill(prompts) == done
                refused = not done
                seen.add(("prefill", done, max(p[1] for p in prompts) > 1))
            elif op == "step":
                live = [s for s in opened if par.rec[s][0][0] < PAGE * max_pages]
                if not live:
                    continue
                slots = rng.sample(live, rng.randint(1, len(live)))
                if rng.random() < 0.1:
                    slots.append(slots[0])
                want = par.step(slots)
                assert tab.step(slots) == want
                refused = want[0] != 0
                seen.add(("step", "refused" if refused else "exact" if want[2] and par.exact else bool(want[2])))
            elif op == "release" and opened:
                s = rng.choice(opened)
                members = [m for m in opened if par.slot_group[m] == par.slot_group[s]]
                whole = members == list(range(members[0], members[0] + len(members)))    # as _release_slots does
                first, n = (members[0], len(members)) if whole and rng.random() < 0.3 else (s, 1)
                gid = par.slot_group[s]
                back = par.release(first, n)
                assert tab.release(first, n) == back
                assert bool(back) == (gid not in par.slot_group)      # the id comes back with the group's last member
                seen.add(("release", len(members) > 1, bool(back)))
            elif op == "swap_out":
                single = [s for s in opened if par.rec[s][0][1] == 1]
                if not single:
                    continue
                s = rng.choice(single)
                want = par.swap_out(s)
                assert tab.swap_out(s) == want
                snaps.append(want[0])
            elif op == "swap_in" and snaps:
                closed = [s for s in range(max_slots) if par.slot_group[s] < 0]
                if not closed:
                    continue
                snap, s = rng.choice(snaps), rng.choice(closed)
                done = par.swap_in(snap, s)
                assert tab.swap_in(snap, s) == done
                if done:
                    snaps.remove(snap)
                refused = not done
                seen.add(("swap_in", done))
            elif op == "poll" and opened:
                s, frames = rng.choice(opened), rng.randint(0, 40)
                par.poll(s, frames)
                tab.poll(s, frames)
            else:
                continue
            _check(tab, par)
            assert not refused or tab.state() == before, f"a refused {op} changed the table"
    finally:
        tab.close_table()


def test_table_follows_the_parent_rules(lib):
    seen = set()
    for seed in range(32):
        try:
            _run(lib, seed, seen)
        except AssertionError as exc:
            raise AssertionError(f"seed {seed}: {exc}") from exc
    # the sequences reached every rule
    want = {("prefill", True, True), ("prefill", False, False), ("step", "refused"), ("step", "exact"), ("step", True),
            ("release", True, False), ("release", True, True), ("release", False, True), ("swap_in", True),
            ("swap_in", False)}
    assert want <= seen, want - seen


@pytest.mark.parametrize("max_pages", [1, 3, 4, 9, 64])
def test_prompt_pages_is_the_tables_reservation(lib, max_pages):
    t = lib.st_new(8 * max_pages, 8, max_pages, PAGE)
    try:
        for n in range(1, 5):
            for total in range(2, PAGE * max_pages + 1):
                assert _Prompt.pages(SimpleNamespace(total=total), n, max_pages) == lib.st_prompt_pages(t, total, n), \
                    (n, total)
    finally:
        lib.st_delete(t)
