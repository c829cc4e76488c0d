"""lzgpu_plan_check_slices, lzgpu_plan_correct_slices and lzgpu_plan_salvage_slices at the limits of the multi-slice tables, without a
GPU.  tests/test_gpu_slices_check_edges.py runs these rows on the GPU.

recover_slices_kernel's CHECK, CORRECT and SALVAGE forms hold 192 read entries and CRC streams per combined stripe, a 192-bit mask of
failing read entries and a 64-bit bad_checks word; locate_slices_kernel a 64-bit candidate mask and S[64][128]; correct_slices_kernel
a 64-bit `changed` mask and 4096 + (checks + suspect blocks) * 512 bytes of dynamic shared memory, up to the 69 632 of its attribute.
Each row of CHECK_EDGES and SALVAGE_EDGES reaches one of these limits.  Its literal values are recomputed from the plain-Python rank
models (tests/test_check_slices_plan.py: given_blocks, masks_model; tests/test_recover_slices_geometry.py: shape, with numpy row
reduction where the matrices are 64 wide), and the plans must equal the models:
- A  ec(8,8) + ec(16,32), all 64 parts: 64 checks (bit 63 of bad_checks), 64 candidate parts; its 15-block tail has 63 checks and
     no block of flat part 31;
- B  ec(7,3) + ec(9,4) with parts 0, 1, 2, 3, 5 and 9 lost: L = 63 with exactly 64 checks.  With every part given no L = 63 set
     has 64 checks or fewer (ec(7,1) + ec(9,1) alone has 79), so L = 63 at the check cap needs lost parts;
- C  std + ec(31,1) + ec(2,1), ec(2,1) lost: L = 62, 64 checks, a correctable std part of 62 blocks per combined stripe, so the
     correct kernel takes 4096 + (64 + 62) * 512 = 68 608 bytes;
- D  std + ec(32,31), all 64 parts: 63 checks, a 32-block std suspect;
- E  xor5 + ec(30,28), all 64 parts: 64 checks; in the 18-block tail, flat parts 24..35 (ec(30,28) data parts 18..29) have no
     block at all, so the tail masks leave them out.  A stale part there is stale padding, which nothing checks;
- F  salvage ec(3,3) + ec(16,16) from parts 0..21: reads + image streams = 192 exactly; parts 0..22 make 195 and are refused;
- G  salvage ec(2,30) + ec(3,28) + std with the data parts of both ec slices lost: the std blocks are read entries 146..151 (word 4
     of the failing-entry mask) and the only staged copies; with every part given they are read entries 158..163, only verified,
     and std blocks 2..5 sit in word 5;
- H  salvage ec(7,3) + ec(9,5) from its parity parts: L = 63, position 44 solved, a 62-block tail wholly determined.
At each check row the debug rows have coefficient 1 on their defining blocks, full rank and annihilate a random combined stripe; at
A, C and D every correctable part's left inverse satisfies P_g H_g = I.  One past each cap is refused: 65 checks, 195 streams."""
import numpy as np
import pytest

from lizardfs_b200 import _lib
from lizardfs_b200.engine import Engine, LzGpuError
from tests.test_check_slices_plan import MUL, given_blocks, masks_model
from tests.test_correct_slices_plan import columns
from tests.test_recover_slices_geometry import gf_rank, shape, slices
from tests.test_recover_slices_plan import goalset, lcm_of
from tests.test_salvage_slices_plan import salvage_geometry

ALL = (1 << 64) - 1
RSC_ATTR = 4096 + (64 + 64) * 512      # correct_slices_kernel's shared-memory attribute: 64 checks, 64 suspect blocks


def given_of(names, spec):
    """"all", ("lost", parts) or a list of the given flat parts"""
    n = slices(names)[1]
    if spec == "all":
        return [1] * n
    if isinstance(spec, tuple) and spec[0] == "lost":
        return [0 if g in spec[1] else 1 for g in range(n)]
    return [1 if g in spec else 0 for g in range(n)]


# id, goal set, given, nb values, {stripe shape (valid blocks): (checks, the mask checked = locatable = correctable)},
# {nb: smem_bytes of the CHECK / CORRECT launch}, {valid: correct_slices_kernel's dynamic shared memory} where pinned
CHECK_EDGES = [
    ("A", ("ec(8,8)", "ec(16,32)"), "all", (1024, 1023, 15),
     {16: (64, ALL), 15: (63, 0xffffffff7fffffff)}, {1024: 96256, 1023: 96256, 15: 95232}, {}),
    ("B", ("ec(7,3)", "ec(9,4)"), ("lost", (0, 1, 2, 3, 5, 9)), (126, 125, 40),
     {63: (64, 0x7ffdd0), 62: (63, 0x7ffdd0), 40: (43, 0x7ffdd0)}, {126: 150400, 125: 150400, 40: 124032}, {}),
    ("C", ("std", "ec(31,1)", "ec(2,1)"), list(range(33)), (992, 1007, 61),
     {62: (64, 0x1ffffffff), 15: (16, 0x10000ffff), 61: (63, 0x1ffffffff)}, {992: 149248, 1007: 149248, 61: 148096},
     {62: 68608, 15: 4096 + (16 + 15) * 512}),
    ("D", ("std", "ec(32,31)"), "all", (1024, 1000),
     {32: (63, ALL), 8: (39, 0xfffffffe000001ff)}, {1024: 113536, 1000: 113536}, {32: 4096 + (63 + 32) * 512}),
    ("E", ("xor5", "ec(30,28)"), "all", (1008,),
     {30: (64, ALL), 18: (50, 0xfffffff000ffffff)}, {1008: 112384}, {}),
]
EDGE = {r[0]: r for r in CHECK_EDGES}


def shapes_of(L, nb):
    """the stripe shapes a plan reports: the full one, and the tail (the full one again when L divides nb)"""
    return L, nb % L or L


def check_model(goals, given, valid):
    """(checks, checked, locatable, correctable, blocks of the largest correctable part) of one stripe shape: correctable when the
    columns of the part's blocks in the check matrix have full rank, |B| - (rank(A) - rank(A without B)) = |B|"""
    blocks = given_blocks(goals, given, valid)
    L = lcm_of(goals)
    A = [r for _, _, r in blocks]
    rA = gf_rank(A, L)
    checked, locatable = masks_model(goals, given, valid, rank=gf_rank)
    correctable, most = 0, 0
    for g in sorted({h for h, _, _ in blocks}):
        rest = [r for h, _, r in blocks if h != g]
        n_g = len(A) - len(rest)
        if n_g - (rA - gf_rank(rest, L)) == n_g:
            correctable |= 1 << g
            most = max(most, n_g)
    return len(A) - rA, checked, locatable, correctable, most


_models = {}


def model_of(names, spec, valid):
    key = (names, str(spec), valid)
    if key not in _models:
        _models[key] = check_model(goalset(names), given_of(names, spec), valid)
    return _models[key]


@pytest.mark.parametrize("row", CHECK_EDGES, ids=[r[0] for r in CHECK_EDGES])
def test_check_rows_against_the_rank_model(row):
    rid, names, spec, nbs, lit, smem, rsc = row
    goals = goalset(names)
    given = given_of(names, spec)
    L = lcm_of(goals)
    for nb in nbs:
        p = Engine.plan_correct_slices(goals, nb, given)
        full, tail = shapes_of(L, nb)
        assert (p["ok"], p["L"], p["tail_blocks"], p["smem_bytes"]) == (1, L, nb % L, smem[nb]), (rid, nb)
        for valid, pre in ((full, ""), (tail, "tail_")):
            n_checks, checked, locatable, correctable, most = model_of(names, spec, valid)
            assert (n_checks, checked) == lit[valid][:1] + (lit[valid][1],), (rid, valid)
            assert locatable == correctable == checked, (rid, valid)
            assert (p[pre + "n_checks"], p[pre + "checked"], p[pre + "locatable"], p[pre + "correctable"]) == \
                (n_checks, checked, locatable, correctable), (rid, nb, pre)
            need = 4096 + (n_checks + most) * 512
            assert need <= RSC_ATTR
            if valid in rsc:
                assert need == rsc[valid], (rid, valid)
    # the limits each row is there for
    if rid == "A":
        assert model_of(names, spec, 16)[0] == 64 and len(given) == 64
        assert not any(g == 31 for g, _, _ in given_blocks(goals, given, 15))      # part 31's one block is position 15
    if rid == "B":
        assert L == 63 and model_of(names, spec, 63)[0] == 64
    if rid == "C":
        assert L == 62 and model_of(names, spec, 62)[4] == 62 and 4096 + (64 + 62) * 512 > 48 * 1024
    if rid == "E":
        blocks = {g for g, _, _ in given_blocks(goals, given, 18)}
        assert blocks == set(range(64)) - set(range(24, 36))


@pytest.mark.parametrize("row", CHECK_EDGES, ids=[r[0] for r in CHECK_EDGES])
def test_debug_check_rows_at_the_limit(row):
    rid, names, spec, nbs, lit, _, _ = row
    goals = goalset(names)
    given = given_of(names, spec)
    L = lcm_of(goals)
    rng = np.random.default_rng(len(rid) + L)
    for valid in sorted(lit):
        blocks = given_blocks(goals, given, valid)
        part, stripe, coef = Engine.debug_check_slices_rows(goals, given, valid)
        n_checks = lit[valid][0]
        assert len(part) == n_checks, (rid, valid)
        where = [(g, s) for g, s, _ in blocks]
        defs = [where.index((int(g), int(s))) for g, s in zip(part, stripe)]
        assert defs == sorted(set(defs))
        mask = np.zeros((64, 64), dtype=bool)
        for g, s in where:
            mask[g, s] = True
        for h in range(n_checks):
            assert coef[h, part[h], stripe[h]] == 1
            assert not coef[h][~mask].any()
        rows = [[int(coef[h, g, s]) for g, s in where] for h in range(n_checks)]
        assert gf_rank(rows, len(where)) == n_checks
        # a random combined stripe: every syndrome is zero
        x = rng.integers(0, 256, size=(L, 16), dtype=np.uint8)
        x[valid:] = 0
        val = {}
        for g, s, r in blocks:
            v = np.zeros(16, dtype=np.uint8)
            for q in range(L):
                v ^= MUL[r[q], x[q]]
            val[(g, s)] = v
        for h in range(n_checks):
            syn = np.zeros(16, dtype=np.uint8)
            for g, s in where:
                syn ^= MUL[coef[h, g, s], val[(g, s)]]
            assert not syn.any(), (rid, valid, h)


@pytest.mark.parametrize("rid", ["A", "C", "D"])
def test_left_inverses_at_the_limit(rid):
    _, names, spec, _, lit, _, _ = EDGE[rid]
    goals = goalset(names)
    given = given_of(names, spec)
    for valid in sorted(lit):
        cols, nc = columns(goals, given, valid)
        mask = lit[valid][1]
        assert set(cols) == {g for g in range(64) if (mask >> g) & 1}
        for g, Hg in cols.items():
            blk_s, rows = Engine.debug_correct_slices_rows(goals, given, valid, g)
            assert len(blk_s) == len(Hg) and not rows[:, nc:].any()
            H = np.array(Hg, dtype=np.uint8)   # [block][check]
            prod = np.zeros((len(blk_s), len(blk_s)), dtype=np.uint8)
            for h in range(nc):
                prod ^= MUL[rows[:, h][:, None], H[:, h][None, :]]
            assert np.array_equal(prod, np.eye(len(blk_s), dtype=np.uint8)), (rid, valid, g)
    if rid == "C":
        blk_s, _ = Engine.debug_correct_slices_rows(goals, given, 62, 0)
        assert list(blk_s) == list(range(62))


def test_one_past_the_check_cap():
    """ec(8,9) + ec(16,31) with every part given: 65 checks, refused; its neighbour ec(8,8) + ec(16,31): 63, accepted"""
    for names, n_checks, ok in ((("ec(8,9)", "ec(16,31)"), 65, 0), (("ec(8,8)", "ec(16,31)"), 63, 1)):
        goals = goalset(names)
        given = given_of(names, "all")
        assert len(given) == 64 - ok
        assert check_model(goals, given, 16)[0] == n_checks
        for plan in (Engine.plan_check_slices, Engine.plan_correct_slices):
            p = plan(goals, 1024, given)
            assert (p["n_checks"], p["ok"]) == (n_checks, ok), names
        if ok:
            assert len(Engine.debug_check_slices_rows(goals, given, 16)[0]) == n_checks
        else:
            with pytest.raises(LzGpuError) as ex:
                Engine.debug_check_slices_rows(goals, given, 16)
            assert ex.value.status == _lib.ERR_ARG


def read_entries(names, given, valid):
    """the read entries of a salvage stripe shape with every given part verified, in order: (flat part, stripe of its slice), flat
    part by flat part, each slice stripe that holds a chunk block"""
    lay, _ = slices(names)
    out = []
    for k, m, base, _ in lay:
        for p in range(k + m):
            if given[base + p]:
                out += [(base + p, s) for s in range(lcm_of(goalset(names)) // k) if s * k < valid]
    return out


def known_of(names, given, valid):
    lay, _ = slices(names)
    return sum(1 << q for q in {q for k, m, base, _ in lay for j in range(k) if given[base + j] for q in range(j, valid, k)})


# id, goal set, given, nb values, {nb: (ok, smem_bytes, CRC streams)}, {valid: (known, determined)}
SALVAGE_EDGES = [
    ("F", ("ec(3,3)", "ec(16,16)"), list(range(22)), (1008,), {1008: (1, 77824, 192)}, {48: ((1 << 48) - 1, (1 << 48) - 1)}),
    ("F_over", ("ec(3,3)", "ec(16,16)"), list(range(23)), (1008,), {1008: (0, 78208, 195)}, {48: ((1 << 48) - 1, (1 << 48) - 1)}),
    ("G", ("ec(2,30)", "ec(3,28)", "std"), ("lost", (0, 1, 32, 33, 34)), (1020, 1019, 5),
     {1020: (1, 30464, 146 + 6 + 6), 1019: (1, 30464, 146 + 6 + 6), 5: (1, 30208, 146 + 5 + 5)}, {6: (0x3f, 0x3f), 5: (0x1f, 0x3f)}),
    ("G_all", ("ec(2,30)", "ec(3,28)", "std"), "all", (1020,), {1020: (1, 32000, 158 + 6 + 6)}, {6: (0x3f, 0x3f)}),
    ("H", ("ec(7,3)", "ec(9,5)"), [7, 8, 9, 19, 20, 21, 22, 23], (126, 125, 62),
     {126: (1, 148096, 62 + 63), 125: (1, 148096, 62 + 63), 62: (1, 147968, 62 + 62)},
     {63: (0, 1 << 44), 62: (0, (1 << 63) - 1)}),
]
SALVAGE = {r[0]: r for r in SALVAGE_EDGES}


@pytest.mark.parametrize("row", SALVAGE_EDGES, ids=[r[0] for r in SALVAGE_EDGES])
def test_salvage_rows_against_the_rank_model(row):
    rid, names, spec, nbs, geo, lit = row
    goals = goalset(names)
    given = given_of(names, spec)
    lay, _ = slices(names)
    L = lcm_of(goals)
    for valid, (known, det) in lit.items():
        assert (known_of(names, given, valid), shape(lay, given, valid)["det"]) == (known, det), (rid, valid)
    for nb in nbs:
        p = Engine.plan_salvage_slices(goals, nb, given)
        full, tail = shapes_of(L, nb)
        assert (p["known"], p["determined"]) == lit[full], (rid, nb)
        assert (p["tail_known"], p["tail_determined"]) == lit[tail], (rid, nb)
        want, streams = salvage_geometry(names, nb, given)
        assert {f: p[f] for f in want} == want
        assert (p["ok"], p["smem_bytes"], streams) == geo[nb], (rid, nb)


def test_salvage_stream_cap_and_mask_words():
    # F: 96 reads of ec(3,3), 48 of ec(16,16)'s data parts, 48 image streams
    given = given_of(*SALVAGE["F"][1:3])
    assert len(read_entries(SALVAGE["F"][1], given, 48)) == 144
    # G: the std copy (flat part 63) is read after every ec part's blocks
    names = SALVAGE["G"][1]
    for spec, first in ((SALVAGE["G"][2], 146), ("all", 158)):
        given = given_of(names, spec)
        ent = read_entries(names, given, 6)
        std = [i for i, (g, _) in enumerate(ent) if g == 63]
        assert std == list(range(first, first + 6)) and len(ent) == first + 6
        words = [i // 32 for i in std]
        assert words == ([4] * 6 if first == 146 else [4, 4, 5, 5, 5, 5])
    # with every part given the data parts of ec(2,30) stage every position: the std blocks are only verified
    assert known_of(names, given_of(names, "all"), 6) == 0x3f


def test_salvage_position_44_of_the_parity_row():
    """H: the one solved position of a full stripe, and the unknowns and equations of both shapes"""
    lay, _ = slices(SALVAGE["H"][1])
    given = given_of(SALVAGE["H"][1], SALVAGE["H"][2])
    full, tail = shape(lay, given, 63), shape(lay, given, 62)
    assert (full["U"], full["E"], full["det"]) == (63, 62, 1 << 44)
    assert (tail["U"], tail["E"], tail["det"]) == (62, 62, (1 << 63) - 1)
