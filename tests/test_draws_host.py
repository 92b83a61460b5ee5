"""CPU tests of flash_vstream_b200/draws.py, the one source of every k-means draw: global `random` is only ever advanced,
an owned source draws what the seeded global generators draw and never touches them, consumed refill counts advance a
source by exactly that many draws, snapshot / rewind, and refills still owed by one model family are applied before the
other family draws."""
import random

import torch

from flash_vstream_b200 import compress_functions as cf
from flash_vstream_b200.draws import GLOBAL, DrawSource


def consumed(n):
    """the k-means kernel's info int32 [4] with n refills consumed, on the host"""
    return torch.tensor([1, n, 1, 0], dtype=torch.int32)


def test_rng_contract_never_rewinds_python_random():
    """the refill candidates come from a private clone of `random`; the global generator is only ever ADVANCED by the
    number of draws the device consumed (0 in the common case), never rewound over what the user did in between"""
    cf.sync_rng()
    random.seed(5)
    GLOBAL.refill_candidates(26, 250, "cpu")[1].consumed_from(consumed(0))               # nothing consumed
    random.seed(7)                                                                        # the user reseeds in between
    cf.sync_rng()
    probe = random.random()
    random.seed(7)
    assert probe == random.random(), "global RNG state was touched although no refill was consumed"
    GLOBAL.refill_candidates(26, 250, "cpu")[1].consumed_from(consumed(2))               # two refills consumed
    random.seed(11)
    cf.sync_rng()
    probe = random.random()
    random.seed(11)
    random.randint(0, 25), random.randint(0, 25)
    assert probe == random.random(), "the global RNG must be advanced by exactly the consumed draws"
    assert not GLOBAL._pending


def test_owned_source_draws_what_the_seeded_global_generators_draw():
    seed = 1234
    torch.manual_seed(99)
    random.seed(99)
    before = (torch.get_rng_state(), random.getstate())
    src = DrawSource(seed, "cpu")
    perms = [src.randperm(n, "cpu") for n in (7, 30)]
    cand, _ = src.refill_candidates(26, 250, "cpu")
    coins = src.randints(0, 1, 9)
    assert torch.equal(torch.get_rng_state(), before[0]) and random.getstate() == before[1], \
        "an owned source must not touch the global generators"
    for draw in (lambda n: torch.randperm(n), lambda n: GLOBAL.randperm(n, "cpu")):
        torch.manual_seed(seed)
        assert all(torch.equal(p, draw(n)) for p, n in zip(perms, (7, 30)))
    random.seed(seed)
    want, _ = GLOBAL.refill_candidates(26, 250, "cpu")
    assert cand.dtype == torch.int32 and torch.equal(cand, want)
    assert cand.tolist() == [random.randint(0, 25) for _ in range(250)]
    random.seed(seed)
    assert coins == [random.randint(0, 1) for _ in range(9)]


def test_lazy_and_eager_consumption_advance_by_the_consumed_count():
    for lazy in (True, False):
        src = DrawSource(3, "cpu")
        _, refills = src.refill_candidates(40, 100, "cpu")
        if lazy:
            refills.consumed_from(consumed(3))         # applied by the next draw
        else:
            src.consume(40, 3)
        ref = random.Random(3)
        for _ in range(3):
            ref.randint(0, 39)
        assert src.randints(0, 1000, 5) == [ref.randint(0, 1000) for _ in range(5)], lazy


def test_snapshot_and_rewind():
    src = DrawSource(8, "cpu")

    def draw():
        return src.randperm(10, "cpu"), src.refill_candidates(12, 20, "cpu")[0], src.randints(0, 9, 4)
    src.randperm(10, "cpu")
    src.refill_candidates(12, 20, "cpu")[1].consumed_from(consumed(2))
    snap = src.snapshot()                              # two refills still owed
    first = draw()                                     # settles them
    src.refill_candidates(12, 20, "cpu")[1].consumed_from(consumed(5))
    src.rewind(snap)                                   # back where it was: the two owed again, the five dropped
    again = draw()
    assert torch.equal(first[0], again[0]) and torch.equal(first[1], again[1]) and first[2] == again[2]

    # the global source: torch's state comes back, `random` is never set and keeps every count it still owes
    torch.manual_seed(4)
    random.seed(6)
    _, refills = GLOBAL.refill_candidates(12, 20, "cpu")
    snap = GLOBAL.snapshot("cpu")
    perm = GLOBAL.randperm(10, "cpu")
    coins = GLOBAL.randints(0, 9, 3)
    refills.consumed_from(consumed(2))
    GLOBAL.rewind(snap)
    assert torch.equal(GLOBAL.randperm(10, "cpu"), perm)
    ref = random.Random(6)
    assert coins == [ref.randint(0, 9) for _ in range(3)]
    ref.randint(0, 11), ref.randint(0, 11)
    GLOBAL.settle()
    assert random.getstate() == ref.getstate()


def test_qwen_draws_start_after_pending_llava_refills():
    """a LLaVA k-means (weighted_kmeans_device) leaves its consumed refill count pending; the Qwen k-means draws its
    candidates (weighted_kmeans_ordered_feature) from the same global `random`, so they start after those refills"""
    from flash_vstream_b200.qwen import compress_functions as qcf
    cf.sync_rng()
    random.seed(9)
    GLOBAL.refill_candidates(26, cf.MAX_ITER * 25, "cpu")[1].consumed_from(consumed(4))
    cand, _ = GLOBAL.refill_candidates(14, qcf.MAX_ITER * 5, "cpu")
    random.seed(9)
    for _ in range(4):
        random.randint(0, 25)
    assert cand.tolist() == [random.randint(0, 13) for _ in range(qcf.MAX_ITER * 5)]
