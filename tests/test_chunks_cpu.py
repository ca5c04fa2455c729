"""Chunk plans, index footprint and budgets: host arithmetic of the library, checked without a GPU."""
import pytest

import fastani_b200 as fb

GiB = 1 << 30


def _config3_budget(device_bytes=80 * GiB, n_queries=1000):
    """Index budget of config 3 (1000 x 5 Mbp, k 16, w 24) on a device with device_bytes free: all queries resident."""
    import ctypes as C
    q = C.c_uint64()
    assert fb.load_library().bani_qsketch_bytes_estimate(5_000_000, 24, 3000, C.byref(q)) == 0
    ws = fb.map_working_set(device_bytes)
    return fb.index_budget(device_bytes, n_queries * q.value, ws, 24), ws


def test_config3_plans_into_one_chunk_on_an_80_GB_device():
    """The benchmark's reference list fits one H100 today (70.9 GB peak): a plan that cut it would mean the footprint is
    more pessimistic than the device."""
    budget, ws = _config3_budget()
    assert fb.plan_chunks([5_000_000] * 1000, [1] * 1000, 16, 24, budget) == [(0, 1000)]
    # the budget keeps max(build peak, resident index + working set) within the device, not their sum
    M = 2 * 5_000_000_000 // 25
    peak, resident = fb.index_footprint(M, M, 1000, 5_000_000_000 + 32 * 1000, min(5_000_000_000, 3 * 5_000_000_000 // 25 + 65536))
    assert peak <= budget and resident + ws <= 80 * GiB < peak + ws + resident


def test_species_scale_list_plans_into_chunks_under_budget():
    budget, _ = _config3_budget()
    n = 20_000
    plan = fb.plan_chunks([5_000_000] * n, [1] * n, 16, 24, budget)
    assert len(plan) > 1 and plan[0][0] == 0 and plan[-1][1] == n
    assert all(a < b for a, b in plan) and all(plan[i][1] == plan[i + 1][0] for i in range(len(plan) - 1))
    for a, b in plan:
        pos = (b - a) * (5_000_000 - 15)
        M = 2 * pos // 25
        peak, _ = fb.index_footprint(M, M, b - a, (b - a) * (5_000_000 + 32), min(pos, int(3.0 * pos / 25) + 65536))
        assert peak <= budget
    # every chunk but the last is as long as the budget allows: one more genome would not fit
    sizes = {b - a for a, b in plan[:-1]}
    assert len(sizes) == 1 and plan[-1][1] - plan[-1][0] <= sizes.pop()


def test_mixed_lengths_and_contigs_are_cut_where_the_budget_ends():
    lens = [3_000_000, 8_000_000, 500_000, 12_000_000, 1_000_000] * 40
    conts = [80, 1, 300, 2, 1] * 40
    budget = 600 << 20
    plan = fb.plan_chunks(lens, conts, 16, 24, budget)
    assert plan[0][0] == 0 and plan[-1][1] == len(lens) and len(plan) > 5
    chunked = fb.plan_chunks(lens, conts, 16, 24, budget * 4)
    assert len(chunked) < len(plan)


def test_a_genome_larger_than_the_budget_is_reported_not_planned():
    budget, _ = _config3_budget()
    with pytest.raises(fb.BaniError) as e:
        fb.plan_chunks([5_000_000, 5_000_000, 2_000_000_000_000], [1, 1, 1], 16, 24, budget)
    assert e.value.code == -4 and "genome 2" in str(e.value)
    with pytest.raises(fb.BaniError):
        fb.plan_chunks([5_000_000], [1], 16, 24, 1 << 20)
    assert fb.plan_chunks([], [], 16, 24, budget) == []


def test_footprint_grows_with_every_term():
    base = fb.index_footprint(10_000_000, 5_000_000, 100, 130_000_000, 15_000_000)
    for args in ((20_000_000, 5_000_000, 100, 130_000_000, 15_000_000), (10_000_000, 9_000_000, 100, 130_000_000, 15_000_000),
                 (10_000_000, 5_000_000, 100000, 130_000_000, 15_000_000), (10_000_000, 5_000_000, 100, 900_000_000, 15_000_000)):
        pk, rs = fb.index_footprint(*args)
        assert pk >= base[0] and rs >= base[1] and (pk, rs) != base
    assert fb.index_footprint(10_000_000, 5_000_000, 100, 130_000_000, 200_000_000)[0] > base[0]
    assert base[1] < base[0]
    with pytest.raises(fb.BaniError):
        fb.index_footprint(10, 11, 1, 64, 10)


def test_budget_leaves_room_for_query_sketches_and_working_set():
    ws = fb.map_working_set(80 * GiB)
    assert ws == 12 * (3 << 29) + 20 * GiB + 3 * GiB
    assert fb.map_working_set(80 * GiB, 1000, 1 << 20) == 12000 + (1 << 20) + 3 * GiB
    b0 = fb.index_budget(80 * GiB, 0, ws, 24)
    b1 = fb.index_budget(80 * GiB, 10 * GiB, ws, 24)
    assert 0 < b1 < b0 < 80 * GiB
    assert fb.index_budget(40 * GiB, 0, 45 * GiB, 24) == 0                 # no room for the working set
    assert fb.index_budget(GiB, 2 * GiB, 0, 24) == 0


@pytest.mark.parametrize("text,value", [("0", 0), ("1000", 1000), ("64M", 64 << 20), ("2G", 2 << 30), ("512k", 512 << 10)])
def test_byte_counts_are_read(text, value):
    assert fb.parse_byte_count(text) == value


@pytest.mark.parametrize("text", ["", "abc", "-5", "12x", " 5", "5 ", "1.5G", "4T", "99999999999999999999", "17179869184G"])
def test_bad_budget_values_are_rejected(text):
    with pytest.raises(fb.BaniError) as e:
        fb.parse_byte_count(text)
    assert e.value.code == -1


def test_working_set_is_what_the_run_can_reach():
    """A run of a few genomes reaches about a hundred megabytes of mapping working set, not the caps; config 3 reaches the caps."""
    small = fb.run_working_set(80 * GiB, 2 * 400_000, 2 * 1700, 2, 10_000_000, 2)
    assert small < 256 << 20
    big = fb.run_working_set(80 * GiB, 1000 * 400_000, 1000 * 1667, 1000, 5_000_000_000, 1000)
    assert big >= fb.map_working_set(80 * GiB)


@pytest.mark.parametrize("free_gib", [2, 10, 40, 44, 80])
def test_small_run_keeps_one_index_at_any_free_memory(free_gib):
    """2 x 5 Mbp against 2 queries: one chunk and one block whatever the other tenants of the device hold -- with the
    worst-case caps 40 GB free would leave no budget, 44 GB two chunks -- and a derived budget that cannot hold a genome
    (almost no memory free) plans the run on one index instead of refusing it."""
    chunks, blocks, _ = fb.plan_run(free_gib * GiB, 85_520_000_000, [5_000_000] * 2, [1] * 2, [5_000_000] * 2)
    assert chunks == [(0, 2)] and blocks == [(0, 2)]
    chunks, blocks, ib = fb.plan_run(1 << 20, 85_520_000_000, [5_000_000] * 2, [1] * 2, [5_000_000] * 2)
    assert chunks == [(0, 2)] and blocks == [(0, 2)] and ib == 0


def test_run_plans_of_config3_and_a_species_scale_list():
    q = [5_000_000] * 1000
    chunks, blocks, ib = fb.plan_run(80 * GiB, 85_520_000_000, [5_000_000] * 1000, [1] * 1000, q)
    assert chunks == [(0, 1000)] and blocks == [(0, 1000)]
    chunks, blocks, ib = fb.plan_run(80 * GiB, 85_520_000_000, [5_000_000] * 20000, [1] * 20000, q)
    assert len(chunks) > 1 and blocks == [(0, 1000)] and chunks[-1][1] == 20000
    assert fb.plan_chunks([5_000_000] * 20000, [1] * 20000, 16, 24, ib) == chunks
    # a forced query budget splits the queries into blocks, each leaving the index more room
    chunks2, blocks2, ib2 = fb.plan_run(80 * GiB, 85_520_000_000, [5_000_000] * 20000, [1] * 20000, q, query_budget=400 << 20)
    assert len(blocks2) > 1 and blocks2[-1][1] == 1000 and ib2 > ib and len(chunks2) <= len(chunks)
    # an empty reference list: nothing to chunk
    assert fb.plan_run(80 * GiB, 85_520_000_000, [], [], q)[:2] == ([], [(0, 1000)])


def test_forced_budget_below_a_genome_is_refused():
    with pytest.raises(fb.BaniError) as e:
        fb.plan_run(80 * GiB, 85_520_000_000, [5_000_000, 9_000_000_000], [1, 1], [5_000_000], index_budget=1 << 30)
    assert e.value.code == -4 and "genome 1" in str(e.value)
    chunks, _, ib = fb.plan_run(80 * GiB, 85_520_000_000, [5_000_000] * 40, [1] * 40, [5_000_000], index_budget=300 << 20)
    assert ib == 300 << 20 and len(chunks) > 1
