"""Runs whose bytes lie past 2^32: the same blocks as a run the suite already builds, placed elsewhere in the run's data.

The blocks of a run do not depend on where they sit (an upload takes any 16-aligned offsets, with gaps: DESIGN §3.6), so a
moved run must answer exactly as the original does.  Every device reader keeps positions past 2^32 in its own way (the
cursor's base_lo / base_hi and nb_lo / nb_hi, the merge's 40-bit value offsets, k_emit's 64-bit output positions, k_scan's
staging loads, k_index_walk's block pointers), and each of them can truncate to 32 bits without any other symptom.

  relocate(br, layout)   the run's blocks written into an np.zeros buffer of the whole new span; pages no block touches are
                         never allocated, so a 4.3 GB run costs the host only its blocks
  Layout(name, block, entry)
      shift_cross          the whole run moved by one 16-aligned constant so that 2^32 falls strictly inside the value bytes
                           of an entry of `block` (the first one at or after `entry` whose value holds a multiple of 16);
                           block + 1 then starts above 2^32, so the walker's next-block prefetch crosses high word 0 -> 1
      hi2                  the same across 2^33 (high word 1 -> 2)
      start_at             block `block` starts exactly at 2^32
      end_at               a block ends at 2^32 and the next block starts right behind it: exactly, for the first block at
                           or after `block` whose size is a multiple of 16; else `block`'s last byte lies in the 15 bytes
                           below 2^32 (its 16-aligned end is 2^32)
      all_above            the first block at 2^32 + 16 * entry: every offset has a high word of 1
      gap_spans_segments   blocks after `block` moved up by GAP (more than 4 GiB): the merge planner weighs that gap as
                           thousands of segment budgets of nothing

relocate asserts that each layout puts its boundary where its name says (check_layout), so a test fails loudly if a run ever
stops reaching the boundary it is there for."""
from dataclasses import dataclass

import numpy as np

import foreign_blocks as fb
from incubator_pegasus_b200 import BlockRun

G4 = 1 << 32
GAP = G4 + (1 << 20)   # gap_spans_segments: a little more than 4 GiB of nothing
LAYOUTS = ("shift_cross", "start_at", "end_at", "all_above", "hi2", "gap_spans_segments")


@dataclass(frozen=True)
class Layout:
    name: str
    block: int = 0
    entry: int = 0

    def __str__(self):
        return "%s-b%d-e%d" % (self.name, self.block, self.entry)


def block_bytes(br, b):
    o = int(br.blk_off[b])
    return br.data[o:o + int(br.blk_size[b])].tobytes()   # never the whole span: fb.run_blocks copies all of it


def block_entries(br, b):
    st, ents = fb.walk_block(block_bytes(br, b))
    assert st == fb.OK, (b, st)
    return ents


def value_span(e):
    """(start, end) of an entry's value inside its block"""
    start = e.fields[2][0] + e.fields[2][1] + e.ns
    return start, start + e.vl


def _crossing_value(br, b, e, edge):
    """-> (entry index, offset m of the boundary inside the run): the first entry of block b at or after e whose value bytes
    strictly contain a multiple of 16 (edge - m is then a 16-aligned shift)"""
    ents = block_entries(br, b)
    base = int(br.blk_off[b])
    for i in range(e, len(ents)):
        vs, ve = value_span(ents[i])
        m = (base + vs) // 16 * 16 + 16
        if m < base + ve and m <= edge:
            return i, m
    raise AssertionError("no value of block %d from entry %d holds a multiple of 16" % (b, e))


def new_offsets(br, layout):
    """-> (new blk_off, what check_layout needs to know)"""
    off = br.blk_off.astype(np.uint64).copy()
    size = br.blk_size.astype(np.uint64)
    b, name = layout.block, layout.name
    assert 0 <= b < br.n_blocks, (layout, br.n_blocks)
    where = dict(block=b)
    if name in ("shift_cross", "hi2"):
        edge = G4 if name == "shift_cross" else 2 * G4
        i, m = _crossing_value(br, b, layout.entry, edge)
        where.update(entry=i, edge=edge)
        return off + np.uint64(edge - m), where
    if name == "start_at":
        return off + np.uint64(G4 - int(off[b])), where
    if name == "end_at":
        assert b + 1 < br.n_blocks, "end_at needs a block behind the chosen one"
        c = next((c for c in range(b, br.n_blocks - 1) if int(size[c]) % 16 == 0), b)
        where["block"] = c
        out = off + np.uint64(G4 - int(off[c]) - ((int(size[c]) + 15) & ~15))
        out[c + 1:] += np.uint64(G4 - int(out[c + 1]))  # the next block right behind it, whatever gap the run had there
        return out, where
    if name == "all_above":
        return off + np.uint64(G4 + 16 * layout.entry - int(off[0])), where
    if name == "gap_spans_segments":
        assert b + 1 < br.n_blocks
        out = off.copy()
        out[b + 1:] += np.uint64(GAP)
        return out, where
    raise ValueError(name)


def check_layout(moved, layout, where):
    """the boundary lies where the layout's name says"""
    off, size = [int(x) for x in moved.blk_off], [int(x) for x in moved.blk_size]
    b, name = where["block"], layout.name
    assert all(o % 16 == 0 for o in off) and all(a + s <= c for a, s, c in zip(off, size, off[1:])), layout
    if name in ("shift_cross", "hi2"):
        edge = where["edge"]
        e = block_entries(moved, b)[where["entry"]]
        vs, ve = value_span(e)
        assert off[b] + vs < edge < off[b] + ve, (layout, off[b] + vs, off[b] + ve)
        assert off[b] >> 32 == (edge >> 32) - 1 and (b + 1 == len(off) or off[b + 1] >> 32 == edge >> 32), layout
        assert len(block_entries(moved, b)) > 1, "the block that holds the boundary has a single entry"
    elif name == "start_at":
        assert off[b] == G4 and (b == 0 or off[b - 1] + size[b - 1] <= G4 - 1), layout
    elif name == "end_at":
        assert off[b] + ((size[b] + 15) & ~15) == G4 and off[b + 1] == G4, layout
    elif name == "all_above":
        assert all(o >> 32 == 1 for o in off) and off[0] == G4 + 16 * layout.entry, layout
    elif name == "gap_spans_segments":
        assert off[b + 1] - (off[b] + size[b]) > G4 and off[b] + size[b] < G4 < off[b + 1], layout


def relocate(br, layout):
    """the blocks of br at the places `layout` gives them; every other byte zero"""
    off, where = new_offsets(br, layout)
    end = (int(off[-1]) + int(br.blk_size[-1]) + 15) & ~15
    data = np.zeros(end, np.uint8)   # untouched pages stay unallocated
    for o, n, s in zip(br.blk_off.tolist(), off.tolist(), br.blk_size.tolist()):
        data[n:n + s] = br.data[o:o + s]
    moved = BlockRun(data, off, br.blk_size.copy())
    check_layout(moved, layout, where)
    return moved


def compact(br):
    """br with its blocks back to back from offset 0 (what relocate keeps apart from the places)"""
    size = br.blk_size.astype(np.uint64)
    off = np.zeros(br.n_blocks, np.uint64)
    off[1:] = np.cumsum((size[:-1] + np.uint64(15)) & ~np.uint64(15))
    data = np.zeros((int(off[-1]) + int(size[-1]) + 15) & ~15, np.uint8)
    for o, n, s in zip(br.blk_off.tolist(), off.tolist(), br.blk_size.tolist()):
        data[n:n + s] = br.data[o:o + s]
    return BlockRun(data, off, br.blk_size.copy())


def boundary_block(br, edge=G4):
    """the block whose bytes hold position edge, or None"""
    for b, (o, s) in enumerate(zip(br.blk_off.tolist(), br.blk_size.tolist())):
        if o <= edge < o + s:
            return b
    return None
