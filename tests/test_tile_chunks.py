"""Chunk planner of tiled sampling (sampler.plan_tile_chunks): which tile-forward units each graph replay holds
when a rank's units exceed the `max_tile_forwards` cap. Host logic only."""
import pytest
import torch

from diffbir_b200.sampler.sampler import (assemble_units, plan_tile_chunks, tile_slots, tiled_run_chunked,
                                          tiles_of_rank)


def _cases():
    for B in (1, 2, 4):
        for world in (1, 2, 3):
            for cap in sorted({B, 2 * B + 1, 7, 64, 128}):
                if cap >= B:
                    yield B, world, cap


@pytest.mark.parametrize("B,world,cap", list(_cases()))
def test_chunk_plan_covers_units_branch_pure_and_capped(B, world, cap):
    for U in range(1, 301):
        for nbr in (1, 2):
            if U % nbr:
                continue
            T = U // nbr
            slots = tile_slots(U, world)
            recv = torch.full((world, slots), -1, dtype=torch.long)
            for rank in range(world):
                mine = tiles_of_rank(U, rank, world)
                per, chunks = plan_tile_chunks(mine, T, B, cap)
                # every local unit in exactly one chunk, chunks in local slot order
                covered = [i for s, n, _ in chunks for i in range(s, s + n)]
                assert covered == list(range(len(mine)))
                assert all(n >= 1 for _, n, _ in chunks)
                assert per == max((n for _, n, _ in chunks), default=0)
                assert per * B <= cap                          # no replay exceeds the cap
                if len(mine) * B <= cap:
                    assert len(chunks) == (1 if mine else 0)  # today's single replay
                else:
                    assert len(chunks) > 1
                    for s, n, br in chunks:                   # branch-pure
                        assert br >= 0 and {u // T for u in mine[s:s + n]} == {br}
                    # each branch's units spread evenly: chunk sizes of a branch differ by the remainder only
                    for br in {c[2] for c in chunks}:
                        sizes = [n for _, n, b in chunks if b == br]
                        assert max(sizes) <= per and len(sizes) == -(-sum(sizes) // (cap // B))
                # each chunk writes its eps to its local slots: the all-gather then yields the reference's unit order
                for s, n, _ in chunks:
                    recv[rank, s:s + n] = torch.tensor(mine[s:s + n])
            assert assemble_units(recv.unsqueeze(-1), U).flatten().tolist() == list(range(U))


def test_chunk_plan_examples():
    # 2048^2 (49 tiles x 2 branches, one image) stays one replay under the default cap
    assert plan_tile_chunks(list(range(98)), 49, 1, 128) == (98, [(0, 98, -1)])
    # 3072^2 (121 tiles x 2 branches): one replay per branch
    assert plan_tile_chunks(list(range(242)), 121, 1, 128) == (121, [(0, 121, 0), (121, 121, 1)])
    # 10 tiles x 2 branches, two images, cap 6: three units per replay, the last chunk of a branch is short
    per, chunks = plan_tile_chunks(list(range(20)), 10, 2, 6)
    assert per == 3 and [n for _, n, _ in chunks] == [3, 3, 3, 1] * 2


def test_chunk_plan_rejects_cap_below_batch():
    with pytest.raises(ValueError):
        plan_tile_chunks(list(range(8)), 4, 4, 3)


def test_tiled_run_chunked_matches_the_plan():
    """The pipeline's question (will this rank's run be chunked?) gets the planner's answer."""
    assert not tiled_run_chunked(49, 2, 1, 128)       # 2048^2: one replay
    assert tiled_run_chunked(121, 2, 1, 128)          # 3072^2: one replay per branch
    assert not tiled_run_chunked(121, 1, 1, 128)      # cfg 1.0: 121 entries fit
    assert tiled_run_chunked(10, 2, 2, 39) and not tiled_run_chunked(10, 2, 2, 40)
