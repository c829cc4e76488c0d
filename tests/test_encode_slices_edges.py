"""lzgpu_plan_encode_slices without a GPU, at the limits of the one-pass multi-slice encode's tables (fused_slices_kernel<M>,
csrc/slices_kernel.cuh; slices_plan, csrc/fused_plan.h).

plan_model restates slices_plan in plain Python: L = lcm of the xor/ec slices' k, the largest G whose 4R CRC data rows plus staged
parity rows fit the 512 threads and whose two stages fit 204 800 bytes of shared memory, G capped by ceil(nb / L), as many stages as
fit (at most four), the shared memory of that ring, the CRC rows, the units, and the refusals SINGLE, CAUCHY, WIDE and NO_GEOMETRY.
test_model_matches_the_planner compares all nine plan fields with the library over every multiset of two to four xor2-9 and
Vandermonde ec(k, m) goals whose L is at most 64, at (3 chunks, 1024 blocks), every pair and triple also at 1, 43 and 1000 blocks,
and every set again with a standard slice added where a slot is free.

EDGE holds the goal sets tests/test_gpu_encode_slices_edges.py runs on the GPU.  test_edge_rows_cover_the_planner_space fails when
a value the kernel depends on (features below) occurs in that enumeration and in no EDGE row: 128 stripes per unit, 16 GF items per
thread, 512 CRC streams, shared memory 392 bytes under the cap, parity rows up to warp 15, 12 GF warps beside parity rows, four slices
with parity, the standard slice in every slot.  The API accepts a slice type twice, so 128 stripes per unit (four xor2 / ec(2, m)
slices) are reachable through the C calls although a LizardFS goal never repeats a slice type."""
import ctypes as C
import math

import pytest

from lizardfs_b200 import _lib

FIELDS = ("fused", "refusal", "L", "G", "threads", "stages", "crc_rows", "smem_bytes", "units")
SINGLE, CAUCHY, WIDE, NO_GEOMETRY = (_lib.SLICES_REFUSED_SINGLE, _lib.SLICES_REFUSED_CAUCHY, _lib.SLICES_REFUSED_WIDE,
                                     _lib.SLICES_REFUSED_NO_GEOMETRY)
XOR, EC, STD = 0, 1, 2
THREADS, NPST, MAX_STAGES, SMEM_CAP, STEP = 512, 4, 4, 200 * 1024, 128   # fused_plan.h: kSlicesThreads .. kStepBytes


def parse(name):
    """(kind, k, m) of "xorN", "ec(k,m)" or "std" """
    if name == "std":
        return (STD, 1, 0)
    if name.startswith("xor"):
        return (XOR, int(name[3:]), 1)
    k, m = name[3:-1].split(",")
    return (EC, int(k), int(m))


def name_of(g):
    kind, k, m = g
    return "std" if kind == STD else (f"xor{k}" if kind == XOR else f"ec({k},{m})")


def cauchy(k, m):
    return m >= 5 or (m == 4 and k > 20)


def smem_model(R, prows, nst):
    stage = -(-R * 4 * STEP // 1024) * 1024
    pstage = -(-prows * STEP // 1024) * 1024
    return nst * stage + NPST * pstage + 520 + 8 * (2 * nst + 2 * NPST)


def plan_model(goals, n_chunks, nb):
    """the nine fields of lzgpu_slices_plan for goals = [(kind, k, m)], as a tuple in FIELDS order"""
    striped = [g for g in goals if g[0] != STD]
    Lc = 1
    for _, k, _ in striped:
        Lc = Lc * k // math.gcd(Lc, k)
    refused = lambda why: (0, why, Lc, 0, 0, 0, 0, 0, 0)
    if len(striped) < 2:
        return refused(SINGLE)
    if any(cauchy(k, m) for _, k, m in striped):
        return refused(CAUCHY)
    if Lc > 64:
        return refused(WIDE)
    prows_of = lambda R: sum(R // k * (m - 1) * 4 for _, k, m in striped)
    G = 0
    for g in range(1, 64 // Lc + 1):
        R = g * Lc
        if 4 * R + prows_of(R) > THREADS or smem_model(R, prows_of(R), 2) > SMEM_CAP:
            break
        G = g
    if G == 0:
        return refused(NO_GEOMETRY)
    G = min(G, -(-nb // Lc))
    R = G * Lc
    prows = prows_of(R)
    nst = 2
    while nst < MAX_STAGES and smem_model(R, prows, nst + 1) <= SMEM_CAP:
        nst += 1
    units = -(-nb // R) * n_chunks
    if units > 0x7fffffff:
        return refused(NO_GEOMETRY)
    return (1, 0, Lc, G, THREADS, nst, 4 * R + prows, smem_model(R, prows, nst), units)


_lib_handle = []
_out = _lib.LzSlicesPlan()


def plan_lib(goals, n_chunks, nb):
    """lzgpu_plan_encode_slices for goals = [(kind, k, m)], as a tuple in FIELDS order"""
    if not _lib_handle:
        _lib_handle.append(_lib.load())
    arr = (_lib.LzGoal * len(goals))(*[_lib.LzGoal(*g) for g in goals])
    assert _lib_handle[0].lzgpu_plan_encode_slices(arr, len(goals), n_chunks, nb, C.byref(_out)) == 0
    return tuple(getattr(_out, f) for f in FIELDS)


def kernel_values(goals, plan):
    """what fused_slices_kernel<M> runs for a fused plan: M, R, staged parity rows, stripes per unit, GF items per thread, GF warps,
    first and last warp holding parity rows (slices_kernel.cuh)"""
    Lc, G = plan[2], plan[3]
    R = G * Lc
    striped = [g for g in goals if g[0] != STD]
    M = max(m for _, _, m in striped)
    prows = sum(R // k * (m - 1) * 4 for _, k, m in striped) if M > 1 else 0
    n_stripes = sum(R // k for _, k, _ in striped)
    ips = 4 * (32 // (2 if M >= 3 else 4))                          # items per stripe and step: 8- or 16-byte items
    per_thread = -(-n_stripes // (THREADS // ips))                  # trips of the gs loop
    gf_warps = min(-(-ips * n_stripes // 32), THREADS // 32)
    first_pwarp, last_pwarp = 4 * R // 32, (4 * R + prows - 1) // 32 if prows else 0
    return dict(M=M, R=R, prows=prows, n_stripes=n_stripes, per_thread=per_thread, gf_warps=gf_warps, first_pwarp=first_pwarp,
                last_pwarp=last_pwarp)


def features(goals, plan):
    """the values of a fused plan the kernel's tables, loops and barrier counts depend on"""
    if not plan[0]:
        return set()
    kv = kernel_values(goals, plan)
    M, R, prows = kv["M"], kv["R"], kv["prows"]
    striped = [g for g in goals if g[0] != STD]
    stds = [i for i, g in enumerate(goals) if g[0] == STD]
    ns = kv["n_stripes"]
    f = {("slices", len(goals)), ("std slot", stds[0] if stds else None), ("stages", M, plan[5]),
         ("stripes", "<=32" if ns <= 32 else "33-64" if ns <= 64 else "65-127" if ns < 128 else "128"),
         ("items per thread", "1" if kv["per_thread"] == 1 else "16" if kv["per_thread"] == 16 else "2-15"),
         ("crc rows", "512" if plan[6] == 512 else "<512"), ("smem > 200000", plan[7] > 200000)}
    if M == 1:
        f.add(("M", 1))
    else:
        f |= {("M", M, "largest m first" if striped[0][2] == M else "largest m later"), ("4R % 32 == 0", M, 4 * R % 32 == 0),
              ("parity rows", "one warp" if kv["first_pwarp"] == kv["last_pwarp"] else "to warp 15" if kv["last_pwarp"] == 15 else "other"),
              ("GF warps < 16 beside parity rows", kv["gf_warps"] < 16)}
    if M == 1 or prows == 0:
        f.add(("parity rows", "none"))
    return f


GOALS = [(XOR, k, 1) for k in range(2, 10)] + [(EC, k, m) for k in range(2, 33) for m in range(1, 5) if not (m == 4 and k > 20)]


def goal_sets():
    """every multiset of 2..4 GOALS with L <= 64, in GOALS order"""
    out = []

    def grow(prefix, start, Lc):
        if len(prefix) >= 2:
            out.append(tuple(prefix))
        if len(prefix) == 4:
            return
        for j in range(start, len(GOALS)):
            nl = Lc * GOALS[j][1] // math.gcd(Lc, GOALS[j][1])
            if nl <= 64:
                grow(prefix + [GOALS[j]], j, nl)

    grow([], 0, 1)
    return out


def with_std(gs, i):
    """gs with the standard slice added at slot i % (len(gs) + 1)"""
    pos = i % (len(gs) + 1)
    return gs[:pos] + ((STD, 1, 0),) + gs[pos:]


def enumeration():
    """(goals, n_chunks, nb) of the whole enumeration"""
    for i, gs in enumerate(goal_sets()):
        for cand in (gs, with_std(gs, i)) if len(gs) < 4 else (gs,):
            yield cand, 3, 1024
            if len(gs) < 4:
                for nb in (1, 43, 1000):
                    yield cand, 3, nb


# the rows tests/test_gpu_encode_slices_edges.py runs: id, goals (slot order), chunks, blocks per chunk, the plan in FIELDS order
EDGE = [
    ("A", ("xor2", "xor2", "xor2", "ec(2,3)"), 3, 1024, (1, 0, 2, 32, 512, 2, 512, 197224, 48)),     # 128 stripes, 16 items per thread, 512 streams
    ("B", ("xor2", "xor2", "xor2", "xor2"), 3, 1024, (1, 0, 2, 32, 512, 4, 256, 131720, 48)),        # 128 stripes with M = 1: a 256-row box
    ("C", ("xor2", "ec(2,1)", "ec(2,2)", "std"), 3, 1024, (1, 0, 2, 32, 512, 4, 384, 197256, 48)),   # 96 stripes, the most a real goal has
    ("D", ("xor2", "ec(2,3)"), 3, 1024, (1, 0, 2, 32, 512, 2, 512, 197224, 48)),                     # 512 streams, distinct types, M = 3
    ("E", ("ec(3,4)", "ec(15,3)"), 3, 1000, (1, 0, 15, 4, 512, 2, 512, 201320, 51)),                 # 512 streams with M = 4, L = 15
    ("F", ("ec(2,4)", "ec(21,3)"), 3, 1024, (1, 0, 42, 1, 512, 3, 436, 204408, 75)),                 # 392 bytes under the cap; last unit 16 blocks
    ("F43", ("ec(2,4)", "ec(21,3)"), 3, 43, (1, 0, 42, 1, 512, 3, 436, 204408, 6)),                  # the same with a one-block last unit
    ("G", ("ec(20,4)", "ec(30,3)", "ec(15,2)", "xor5"), 3, 1000, (1, 0, 60, 1, 512, 4, 308, 160392, 51)),  # four slices with parity
    ("H", ("ec(2,3)", "xor2", "ec(2,4)", "ec(2,2)"), 3, 1024, (1, 0, 2, 14, 512, 2, 448, 201320, 111)),  # m = 1 between prow4 ranges
    ("I", ("ec(31,3)", "ec(31,2)", "ec(31,1)", "std"), 3, 1000, (1, 0, 31, 2, 512, 4, 272, 139912, 51)),  # 12 GF warps beside parity rows
    ("J", ("ec(4,4)", "std", "ec(8,4)", "ec(16,4)"), 3, 1024, (1, 0, 16, 3, 512, 2, 444, 180840, 66)),  # std in slot 1, three M = 4 slices
    ("K", ("ec(2,2)", "ec(3,2)", "std"), 3, 1024, (1, 0, 6, 10, 512, 3, 440, 195192, 54)),          # three slices, std in slot 2, M = 2 first
    ("L", ("std", "xor2", "xor3", "ec(8,2)"), 3, 1024, (1, 0, 24, 2, 512, 4, 216, 111240, 66)),      # std in slot 0, parity rows in one warp
    ("M", ("xor2", "xor3", "xor4", "ec(3,3)"), 3, 1024, (1, 0, 12, 5, 512, 3, 400, 174712, 54)),     # M = 3 in three stages
    ("N", ("xor2", "ec(2,2)", "ec(3,2)", "ec(4,2)"), 3, 1024, (1, 0, 12, 5, 512, 2, 500, 197224, 54)),  # M = 2 in two stages
]


def edge_goals(names):
    return [parse(n) for n in names]


def test_model_matches_the_planner():
    n = 0
    for goals, n_chunks, nb in enumeration():
        assert plan_model(goals, n_chunks, nb) == plan_lib(goals, n_chunks, nb), ([name_of(g) for g in goals], n_chunks, nb)
        n += 1
    assert n > 400000


def test_enumeration_counts():
    """the issue's census at 3 chunks of 1024 blocks: 423 316 sets, 374 783 fused and 48 533 refused for want of a geometry"""
    sets = goal_sets()
    plans = [plan_model(gs, 3, 1024) for gs in sets]
    assert len(sets) == 423316
    assert sum(p[0] for p in plans) == 374783
    assert sum(p[1] == NO_GEOMETRY for p in plans) == 48533 == len(sets) - 374783


def test_edge_rows_cover_the_planner_space():
    seen = set()
    for goals, n_chunks, nb in enumeration():
        seen |= features(goals, plan_model(goals, n_chunks, nb))
    table = set()
    for _, names, n_chunks, nb, plan in EDGE:
        table |= features(edge_goals(names), plan)
    assert seen - table == set()


@pytest.mark.parametrize("row", EDGE, ids=lambda r: r[0])
def test_edge_row_plans(row):
    _, names, n_chunks, nb, plan = row
    goals = edge_goals(names)
    assert plan_lib(goals, n_chunks, nb) == plan_model(goals, n_chunks, nb) == plan


def test_edge_rows_reach_the_tables_limits():
    kv = {r[0]: kernel_values(edge_goals(r[1]), r[4]) for r in EDGE}
    assert kv["A"]["n_stripes"] == kv["B"]["n_stripes"] == 128 and kv["A"]["per_thread"] == 16 and kv["B"]["per_thread"] == 8
    assert kv["C"]["n_stripes"] == 96
    assert kv["A"]["last_pwarp"] == kv["D"]["last_pwarp"] == kv["E"]["last_pwarp"] == 15
    assert kv["F"]["R"] == 42 and SMEM_CAP - {r[0]: r[4] for r in EDGE}["F"][7] == 392
    assert kv["G"]["R"] == 60 and 4 * 60 % 32 != 0 and kv["G"]["first_pwarp"] == 7
    assert kv["H"]["prows"] == 336 and kv["I"]["gf_warps"] == 12 and kv["I"]["prows"] > 0


def test_units_refusal():
    """units past 0x7fffffff refuse the set (NO_GEOMETRY) rather than overflow the kernel's unit numbers; planner only"""
    goals = edge_goals(("xor2", "xor2", "xor2", "ec(2,3)"))
    per_chunk = -(-1024 // 64)
    n = 0x7fffffff // per_chunk + 1
    assert plan_lib(goals, n, 1024) == plan_model(goals, n, 1024) == (0, NO_GEOMETRY, 2, 0, 0, 0, 0, 0, 0)
    fused = plan_lib(goals, n - 1, 1024)
    assert fused == plan_model(goals, n - 1, 1024) and fused[0] == 1 and fused[8] == (n - 1) * per_chunk
    # at one block per chunk every chunk is one unit: the largest batch is 0x7fffffff chunks
    assert plan_lib(goals, 0x7fffffff, 1)[0] == 1 and plan_lib(goals, 0x80000000, 1)[1] == NO_GEOMETRY


@pytest.mark.parametrize("names,why", [
    (("ec(8,2)", "std"), SINGLE), (("xor2", "xor2", "ec(21,4)"), CAUCHY), (("ec(3,2)", "ec(2,5)"), CAUCHY),
    (("ec(5,1)", "ec(13,1)"), WIDE), (("xor9", "ec(8,1)"), WIDE), (("ec(2,4)", "ec(25,1)"), NO_GEOMETRY),
    (("ec(32,4)", "ec(16,1)"), CAUCHY), (("xor2", "xor3", "ec(2,3)", "ec(20,4)"), NO_GEOMETRY),
], ids=lambda v: "+".join(v) if isinstance(v, tuple) else str(v))
def test_refusals(names, why):
    goals = edge_goals(names)
    got = plan_lib(goals, 3, 1024)
    assert got == plan_model(goals, 3, 1024) and got[1] == why
