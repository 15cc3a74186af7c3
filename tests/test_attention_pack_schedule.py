"""CPU: the item / operand-stage schedule of the attention kernel (attention.cuh), restated in Python.

A launch has batch * heads items (crop, head); CTA c of a grid of G takes items c, c + G, c + 2G, ... in order.  Q, K and V of an
item live in one of TWO stages (local item li -> stage li % 2, its (li // 2)-th use: barrier phase (li // 2) & 1).  Thread 0
loads local items 0 and 1 before the loop; after item li has been computed by all three warpgroups (a CTA barrier) it refills
that item's stage with local item li + 2.  (The file keeps its name from the project's earlier packed-pair kernel; the
properties it pins are the same ones.)  Invariants checked here for every CTA of many (batch, heads, grid) shapes -- they are
what makes the kernel's waits terminate and its operands valid:
  * every row of every item is produced exactly once over the launch;
  * every item finds its operands resident, in the stage and barrier phase the kernel computes for it;
  * no load overwrites a stage whose current item is still needed;
  * every load a CTA issues is consumed by that CTA (a CTA must not exit with a TMA load in flight).
Keep `cta_schedule` in step with the index arithmetic of the kernel.
"""
import pytest


def cta_schedule(items: int, grid: int, cta: int):
    """Mirror of attention_wgmma's per-CTA bookkeeping: the global items of this CTA, in the order it computes them."""
    return list(range(cta, items, grid))


def simulate(items: int, grid: int, cta: int):
    """Runs the load / use protocol of one CTA; returns the rows it produces."""
    mine = cta_schedule(items, grid, cta)
    stage = [None, None]                                    # local item resident in each stage
    loads = []
    used = set()
    done = set()

    def load(li):
        assert 0 <= li < len(mine)
        s = li % 2
        if stage[s] is not None:                            # the item being replaced must already be computed
            assert stage[s] in done, (items, grid, cta, li, stage[s])
        assert sum(1 for x in loads if x % 2 == s) == li // 2   # barrier phase (li // 2) & 1 = number of earlier loads of this stage
        stage[s] = li
        loads.append(li)

    # prologue (thread 0): item blockIdx.x and item blockIdx.x + gridDim.x, when they exist
    if cta < items:
        load(0)
    if cta + grid < items:
        load(1)
    produced = []
    for li, item in enumerate(mine):
        assert stage[li % 2] == li, (items, grid, cta, li, stage)
        used.add(li)
        produced += [(item, r) for r in range(192)]          # three warpgroups x 64 query rows
        done.add(li)
        if item + 2 * grid < items:                         # the refill after the CTA barrier
            load(li + 2)
    assert set(loads) == used == set(range(len(mine))), (items, grid, cta, loads, used)    # every load consumed, nothing missing
    return produced


@pytest.mark.parametrize("batch,heads", [(1, 2), (1, 12), (2, 12), (3, 12), (9, 12), (13, 16), (32, 16), (64, 12), (64, 16), (5, 6)])
@pytest.mark.parametrize("sms", [148, 132, 8, 1])
def test_every_row_once_and_operands_resident(batch, heads, sms):
    items = batch * heads
    grid = min(items, sms)                                  # engine.cu: attention_launch
    rows = []
    for cta in range(grid):
        rows += simulate(items, grid, cta)
    assert len(rows) == items * 192 and len(set(rows)) == items * 192


def test_single_step_ranges_start_at_the_item_they_need():
    """CTAs that own exactly one item load that item and nothing else (the prologue's second load must be skipped, or it would
    stay unconsumed); CTAs with two items load both up front and refill nothing.  Swept over grids that produce both cases."""
    counts = set()
    for items, grid in [(12, 12), (8, 7), (10, 9), (14, 13), (16, 11), (6, 5), (20, 19), (22, 17)]:
        for cta in range(grid):
            mine = cta_schedule(items, grid, cta)
            counts.add(len(mine))
            assert mine[0] == cta
            if len(mine) == 1:
                assert cta + grid >= items
            if len(mine) == 2:
                assert mine[1] + 2 * grid >= items            # hence no refill
            simulate(items, grid, cta)
    assert {1, 2} <= counts
