"""CPU checks of the ping-pong consumer schedule of the GEMM (csrc/gemm_tc.cu, PP = true), transliterated from the
kernel: the producer publishes (tile, k-blocks queued before it) into the tile-index ring and closes it with an end
marker in two slots; consumer warpgroup w takes slots w, w + 2, ...; each tile's first stage and phase in the operand
ring come from the published k-block count; the two K loops alternate whole tiles through a pair of order barriers."""
import random


def producer(tiles_kb, pingpong):
    """The producer thread: ring slots (tile, kpos) in publication order, and (FIFO ring position, tile) of every k-block
    it loads."""
    slots, loads, kpos = [], [], 0
    for t, nkb in tiles_kb:
        slots.append((t, kpos))
        for _ in range(nkb):
            loads.append((len(loads), t))
        kpos += nkb
    slots.append((None, kpos))            # end marker: one more fetch / round-robin step, never two
    if pingpong:
        slots.append((None, kpos))        # published again into the next slot
    return slots, loads


def consumer(slots, wg, stages):
    """Consumer warpgroup wg: its tiles with the (stage, phase) of their first k-block, until its end marker."""
    out, it = [], 0
    while True:
        sit = 2 * it + wg
        t, kpos = slots[sit]
        if t is None:
            return out, sit
        out.append((t, kpos % stages, (kpos // stages) & 1, kpos))
        it += 1


def test_each_warpgroup_sees_one_end_marker_and_the_tiles_are_split_in_ring_order():
    rng = random.Random(3)
    for n_tiles in (0, 1, 2, 3, 7, 8, 9, 31, 64):
        for stages in (2, 3, 5, 8):
            tiles_kb = [(t, rng.choice([1, 1, 2, 4, 9, 18])) for t in range(n_tiles)]
            slots, loads = producer(tiles_kb, pingpong=True)
            got = {}
            ends = set()
            for wg in (0, 1):
                mine, end_slot = consumer(slots, wg, stages)
                ends.add(end_slot)
                got[wg] = mine
                assert [t for t, *_ in mine] == [t for i, (t, _) in enumerate(tiles_kb) if i % 2 == wg]
            # the two end markers are the last two slots, one of each parity
            assert ends == {len(slots) - 2, len(slots) - 1}
            # the first k-block of every tile is where the producer put it: stage = position in the FIFO ring mod stages,
            # phase = parity of the ring pass
            first_load = {}
            for pos, t in loads:
                first_load.setdefault(t, pos)
            for wg in (0, 1):
                for t, stage, phase, kpos in got[wg]:
                    pos = first_load[t]
                    assert kpos == pos and stage == pos % stages and phase == (pos // stages) & 1


def test_order_barriers_make_the_k_loops_alternate_whole_tiles():
    """Warpgroup 1's tile `it` waits for completion `it` of order_bar[1] (arrived on by warpgroup 0 after each of its
    tiles); warpgroup 0's tile `it` > 0 waits for completion `it - 1` of order_bar[0] (arrived on by warpgroup 1).  The
    completion waited for is always the tile in the previous ring slot."""
    for slot in range(1, 200):
        wg, it = slot % 2, slot // 2
        if wg == 1:
            arriving_wg, completion = 0, it
        else:
            arriving_wg, completion = 1, it - 1
        assert 2 * completion + arriving_wg == slot - 1


def test_end_marker_costs_no_extra_fetch():
    """The host's fetch accounting (chunks + one end marker per CTA) holds for the ping-pong schedule: the second end
    marker is the first one published again, not a new counter value."""
    for n in (0, 1, 5, 40):
        lockstep, _ = producer([(t, 1) for t in range(n)], pingpong=False)
        pingpong, _ = producer([(t, 1) for t in range(n)], pingpong=True)
        assert sum(1 for t, _ in lockstep if t is None) == 1
        assert pingpong[:-1] == lockstep and pingpong[-1] == pingpong[-2]
