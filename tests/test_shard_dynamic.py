"""Dynamic resolution in the sharded frame stream (FSR1_SHARD_DYNAMIC, fsr1_shard_frame), the parts that need no GPU: the per-frame
row plan over every render height a dynamic shard can accept, the window capacity it is sized for, and the binding's constants."""
import ctypes
import os
import re

import pytest

import fsr1_b200 as F
from fsr1_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def frame_plan(rw, rh, ow, oh, world):
    """SlabPlan of a frame rendered at rw x rh, with the constants fsr1_shard_frame builds."""
    return F.SlabPlan(rh, oh, world, F.api.easu_con(rw, rh, rw, rh, ow, oh))


def neighbours_only(plan):
    """fsr1_shard_create's rule: every rank's needed rows lie inside [owned(k-1).a, owned(k+1).b)."""
    for r in range(plan.world):
        n0, n1 = plan.needed_in_rows(r)
        lo = plan.owned_in_rows(r - 1)[0] if r > 0 else 0
        hi = plan.owned_in_rows(r + 1)[1] if r + 1 < plan.world else plan.in_h
        if n0 < lo or n1 > hi:
            return False
    return True


def _offsets(plan, r, which, peer_side):
    """offsets into rank r's window of the rows it sends to (which=0) / receives from (which=1) its upper (peer_side=-1) or lower
    (+1) neighbour"""
    w0 = plan.window_rows(r)[0]
    return {y - w0 for peer, a, b in plan.transfers(r)[which] if peer - r == peer_side for y in range(a, b)}


def crossing(p1, p2, r):
    """Rows of rank r's window that a neighbour's push for a frame of plan p2 writes while r's push for the previous frame (plan
    p1) may still read them on the OTHER side: writes from below against the push up, writes from above against the push down.
    (Same-side pairs are ordered: that neighbour waited for r's previous push before it wrote its next frame.)"""
    return ((_offsets(p1, r, 0, -1) & _offsets(p2, r, 1, +1)) | (_offsets(p1, r, 0, +1) & _offsets(p2, r, 1, -1)))


def accepted_heights(iw, ih, ow, oh, world):
    """The render heights a dynamic shard accepts, tallest first: from ih down, those that pass the neighbour-only rule, until the
    first height that would make crossing() non-empty for some rank and some pair of heights accepted so far or this one."""
    up_r, down_r, from_up_w, from_down_w = ([set() for _ in range(world)] for _ in range(4))
    out = []
    for rh in range(ih, world - 1, -1):
        p = frame_plan(iw, rh, ow, oh, world)
        if not neighbours_only(p):
            continue
        new = [(_offsets(p, r, 0, -1), _offsets(p, r, 0, +1), _offsets(p, r, 1, -1), _offsets(p, r, 1, +1)) for r in range(world)]
        if any(((up_r[r] | ur) & (from_down_w[r] | fdw)) or ((down_r[r] | dr) & (from_up_w[r] | fuw))
               for r, (ur, dr, fuw, fdw) in enumerate(new)):
            break
        for r, (ur, dr, fuw, fdw) in enumerate(new):
            up_r[r] |= ur
            down_r[r] |= dr
            from_up_w[r] |= fuw
            from_down_w[r] |= fdw
        out.append(rh)
    return out


def capacity(iw, ih, ow, oh, world):
    """Window rows a dynamic shard gives each slot: the tallest window over every render height it accepts."""
    return max(w1 - w0 for rh in accepted_heights(iw, ih, ow, oh, world) for p in [frame_plan(iw, rh, ow, oh, world)]
               for w0, w1 in map(p.window_rows, range(world)))


RESOURCES = [(1920, 1080, 3840, 2160, 1), (1920, 1080, 3840, 2160, 8), (640, 360, 1280, 720, 2), (640, 360, 1280, 720, 8),
             (2560, 1440, 3840, 2160, 4), (200, 120, 261, 157, 3)]


@pytest.mark.parametrize("iw,ih,ow,oh,world", RESOURCES)
def test_every_render_height_tiles_its_input_and_fits_the_capacity(iw, ih, ow, oh, world):
    cap = capacity(iw, ih, ow, oh, world)
    base = frame_plan(iw, ih, ow, oh, world)
    assert neighbours_only(base)                                        # fsr1_shard_create accepts the resource itself
    assert cap >= max(w1 - w0 for w0, w1 in map(base.window_rows, range(world)))
    accepted = 0
    for rh in range(world, ih + 1):
        p = frame_plan(iw, rh, ow, oh, world)
        owned = [p.owned_in_rows(r) for r in range(world)]
        assert owned[0][0] == 0 and owned[-1][1] == rh                  # the owned rows tile [0, rh)
        assert all(a1 == b0 and a0 < a1 for (a0, a1), (b0, _) in zip(owned, owned[1:] + [(rh, None)]))
        ok = neighbours_only(p)
        for r in range(world):
            _, recvs = p.transfers(r)
            # the rule in other words: an accepted height takes its halo from the direct neighbours only
            assert ok <= all(abs(peer - r) == 1 for peer, _, _ in recvs), (rh, r, recvs)
            if ok:
                w0, w1 = p.window_rows(r)
                assert w1 - w0 <= cap
                n0, n1 = p.needed_in_rows(r)
                got = set(range(*owned[r])) | {y for _, a, b in recvs for y in range(a, b)}
                assert set(range(n0, n1)) <= got                          # every row EASU reads arrives for this frame
        if not ok:
            assert any(abs(peer - r) > 1 for r in range(world) for peer, _, _ in p.transfers(r)[1]), rh
        accepted += ok
    assert accepted >= 1


def test_thin_frames_are_refused_at_eight_ranks():
    """640x360 -> 1280x720 at 8 ranks: a frame a few rows per rank tall needs halo rows from beyond the neighbours, or would let
    a neighbour overwrite rows a push of a taller frame still reads; everything from a few rows per rank up is accepted."""
    refused = [rh for rh in range(8, 361) if not neighbours_only(frame_plan(640, rh, 1280, 720, 8))]
    assert refused and max(refused) < 40 and 8 in refused
    acc = accepted_heights(640, 360, 1280, 720, 8)
    assert acc == [rh for rh in range(360, min(acc) - 1, -1) if rh not in refused]  # every height from the smallest up
    assert 21 not in acc and min(acc) < 48                                # 6 rows per rank are accepted


@pytest.mark.parametrize("world", [3, 4, 8])
def test_no_accepted_height_writes_rows_a_push_of_another_reads(world):
    """A neighbour's push for use q of a slot (plan of q) must never write window rows my push of use q-1 (plan of q-1) may still
    read: it waits for my credit, which covers my EASU's reads only.  Equal heights never meet; some pairs of heights that pass the
    neighbour-only rule do (rank 1 of 8: a 100-row frame, then a 21-row one), and the accepted set has no such pair."""
    iw, ih, ow, oh = 640, 360, 1280, 720
    rule = {rh: p for rh in range(world, ih + 1) for p in [frame_plan(iw, rh, ow, oh, world)] if neighbours_only(p)}
    acc = set(accepted_heights(iw, ih, ow, oh, world))
    assert ih in acc and acc <= set(rule)
    off = {(rh, r): [_offsets(p, r, w, side) for w in (0, 1) for side in (-1, +1)] for rh, p in rule.items() for r in range(world)}
    # crossing(), with the offsets computed once: [send up, send down, from up, from down]
    meeting = {(r, h1, h2) for r in range(world) for h1 in rule for h2 in rule
               if (off[h1, r][0] & off[h2, r][3]) or (off[h1, r][1] & off[h2, r][2])}
    assert (1, 100, 21) not in meeting or crossing(rule[100], rule[21], 1)
    assert not [m for m in meeting if m[1] == m[2]]                     # a static shard never meets it
    assert meeting                                                      # the rule alone would let such frames through
    assert not [m for m in meeting if m[1] in acc and m[2] in acc]
    if world == 8:
        assert (1, 100, 21) in meeting and 21 not in acc


def test_shard_dynamic_matches_the_header():
    text = open(os.path.join(ROOT, "include", "fsr1_b200.h")).read()
    m = re.search(r"#define\s+FSR1_SHARD_DYNAMIC\s+\(1u\s*<<\s*(\d+)\)", text)
    assert m and _lib.SHARD_DYNAMIC == 1 << int(m.group(1)) == 1 << 19
    others = [_lib.SHARD_ONE_STREAM, _lib.SHARD_SKIP_HALO, _lib.SHARD_TRACE]
    assert _lib.SHARD_DYNAMIC not in others
    # no FSR1_FLAG_* kernel flag shares the bit
    flags = [int(v) for v in re.findall(r"FSR1_FLAG_\w+\s*=\s*1u\s*<<\s*(\d+)", text)]
    assert 19 not in flags


def test_frame_refuses_a_null_shard_without_a_gpu():
    L = _lib.lib()
    assert L.fsr1_shard_frame(None, 0, 64, 64, ctypes.c_float(0.25)) == -1


def test_dynamic_needs_the_p2p_data_plane():
    with pytest.raises(ValueError):
        F.ShardedUpscaler(64, 64, 128, 128, 2, 0, halo="nccl", dynamic=True, device="cpu")
