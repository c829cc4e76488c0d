"""The stripe repair and decode (lzgpu_repair_stripes, lzgpu_decode_stripes and their _dev forms) at every instantiation and geometry of
the check pass that records F, the given blocks failing their stored CRCs (fused_check_repair_kernel<R, C> and
fused_check_repair_degraded_kernel<E, R, C>, csrc/check_kernel.cuh); with several working entries per CTA for the two grid-stride
kernels after it (repair_map_kernel and decode_map_kernel, csrc/correct_kernel.cuh); and the decode at every point of its radius.

CASES takes every case of the check geometry table (every data part given) and of the degraded one (data parts lost).  Together they
hold every value of the planner's space with at least k + 1 given parts, which the repair needs: the instantiation (E lost data parts,
R checked rows, rows 0 .. R-1 or not), G, the stage count and the item passes.  test_repair_table_covers_the_planner_space
enumerates that space on the CPU and fails when a value is missing or a literal plan no longer matches.

Every GPU case has three chunks of pb = 2 G + G / 2 stripes (the last unit partial) and nb = k pb - (k - 1) blocks (the last stripe
holds data part 0 alone).  Faults go into chunks 0 and 2; chunk 1 stays clean.  `rot` flips bytes and keeps the stored CRC, so the
block is in F; Batch.corrupt recomputes the CRC (a stale block: only the code sees it).  The faults: rot in a data block at stripe 0;
a stale part at G - 1; rot in given - k blocks at G (data parts, input parity parts and spares, over the four quarters of the block
whose CRCs the check computes in separate streams); rot in quarters 1 and 2 at G + 16 and G + 32 (item passes 1 and 2); rot in
given - k + 1 blocks at 2 G; a wrong stored CRC on a clean stripe; a stale input beside rot; the last byte of data part 0 and a
zero-padded block of another data part at pb - 1; and seeded single faults.  Each case runs both calls, host and _dev (a padded
stride with guard bytes), on the default context, LZGPU_GRID_CAP=2 and LZGPU_DISABLE_FUSED=1.

Expected values come from references, never from the library's kernels: F from zlib.crc32 against the stored CRCs; bad_rows and
suspect_part from the oracle's degraded map (test_gpu_stripe_degraded.expected_map); the status from the rules of include/lzgpu.h,
restated in expected_entry; rebuilt blocks from the oracle's rs_recover; located sets from a brute force over every set of at most
two given parts outside F."""
import itertools
import types
import zlib

import numpy as np
import pytest

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from tests import test_gpu_check_geometry as CG
from tests import test_gpu_stripe_degraded as SD
from tests.test_gpu_check_geometry import expected_geometry, sm_count
from tests.test_gpu_stripe_check import BLOCK, Batch, Dev
from tests.test_gpu_stripe_correct import block, dev_parts, fix_list
from tests.test_gpu_stripe_decode import entries
from tests.test_gpu_stripe_degraded import ROUTES, dev_fix, engine, expected_map, host_result
from tests.test_gpu_stripe_repair import crc_list, given_list, oracle_rebuild, rot, twin

REPAIR = L.Engine.STRIPE_REPAIR_DTYPE
DECODE = L.Engine.STRIPE_DECODE_DTYPE
CALLS = (("repair_stripes", REPAIR), ("decode_stripes", DECODE))
UNRESOLVED = (_lib.FIX_UNEXPLAINED, _lib.FIX_CRC_CONFLICT)
CRC_LEFT = (_lib.FIX_CRC_ONLY, _lib.FIX_CRC_CONFLICT)
gpu = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for e in SD._engines.values():
        e.close()
    SD._engines.clear()


# ---- the planner's space with k + 1 given parts, on the CPU --------------------------------------------------------------------

# (goal, lost data parts, given parity rows, literal plan: test_gpu_stripe_degraded.PLAN_KEYS)
CASES = [(name, (), rows, (1,) + want) for name, rows, want in CG.CASES] + list(SD.CASES)

# (E, R, rows 0 .. R-1): the repair members of kCheckers (E = 0) and kDegradedCheckers (csrc/fused.cu)
REPAIR_INSTANTIATIONS = {(0, 1, 1), (0, 2, 1), (0, 3, 1), (0, 4, 1), (0, 1, 0), (0, 2, 0), (0, 3, 0),
                         (1, 2, 1), (1, 3, 1), (1, 4, 1), (2, 3, 1), (2, 4, 1), (3, 4, 1), (1, 2, 0), (1, 3, 0), (2, 3, 0)}


def plan_of(g, lost, rows):
    return L.Engine.plan_check_degraded(g, SD.flags(g, set(lost) | {g.k + r for r in range(g.m) if r not in rows}))


def features(e, p):
    return {("instantiation", e, p["rows"], p["consecutive"]), ("G", p["G"]), ("stages", p["stages"]), ("item passes", p["item_passes"])}


def repair_space():
    """{(goal, lost data count, given parity rows): plan} for every Vandermonde goal, 0 .. 3 lost data parts and every set of given
    parity parts that leaves at least k + 1 given parts"""
    space = {(name, 0, rows): p for (name, rows), p in CG.planner_space().items()}
    space.update(SD.degraded_space())
    return space


def test_repair_table_covers_the_planner_space():
    space = repair_space()
    feats = set()
    for (name, e, rows), p in space.items():
        g = L.SliceType(name)
        assert g.k - e + len(rows) >= g.k + 1 and p["fused"] == 1, (name, e, rows, p)
        feats |= features(e, p)
    assert {f[1:] for f in feats if f[0] == "instantiation"} == REPAIR_INSTANTIATIONS
    assert {f[1] for f in feats if f[0] == "item passes"} == {1, 2, 3}
    table = set()
    for name, lost, rows, want in CASES:
        g = L.SliceType(name)
        p = plan_of(g, lost, rows)
        assert SD.literal(p) == want, (name, lost, rows, SD.literal(p))
        assert p == space[(name, len(lost), rows)]
        table |= features(len(lost), p)
    assert not feats - table, sorted(feats - table, key=str)


# ---- the expected result, on the CPU -----------------------------------------------------------------------------------------------

def mask(parts):
    return sum(1 << p for p in parts)


def crc_of(blk):
    return zlib.crc32(blk.tobytes())


def stripe_view(b, parts, c, s):
    """stripe s of chunk c as a one-chunk batch of one stripe (a short stripe is zero-padded, so its syndromes are the same)"""
    return types.SimpleNamespace(k=b.k, m=b.m, n=1, pb=1, parts=[block(parts, i, c, s).reshape(1, BLOCK) for i in range(b.k + b.m)])


def consistent(oracle, b, parts, c, s, kept, cols):
    """the blocks of the parts `kept` (ascending, at least k) agree with one codeword at the byte columns `cols`: the parts after the
    first k equal their rebuild from the first k"""
    inputs, rest = kept[:b.k], kept[b.k:]
    if not rest or not len(cols):
        return True
    n = b.k + b.m
    ins = [np.ascontiguousarray(block(parts, i, c, s)[cols]) if i in inputs else None for i in range(n)]
    out = oracle.rs_recover(b.k, b.m, ins, [0 if i in inputs else 1 for i in range(n)], [int(i in rest) for i in range(n)], len(cols))
    return all((out[p] == block(parts, p, c, s)[cols]).all() for p in rest)


def brute_force(oracle, b, parts, pristine, c, s, given, failed):
    """E for the smallest e, 1 <= e <= 2 with 2 e + |F| <= spares, for which exactly one set E of e given parts outside F leaves a
    codeword; None when there is none.  Only the byte columns where a kept block differs from the pristine one are compared: the
    pristine stripe is a codeword, so every other column agrees for every set."""
    kept = [p for p in sorted(given) if p not in failed]
    spare = len(given) - b.k
    cols = np.nonzero(np.any([block(parts, p, c, s) != block(pristine, p, c, s) for p in kept], axis=0))[0]
    if consistent(oracle, b, parts, c, s, kept, cols):
        return None
    for e in (1, 2):
        if 2 * e + len(failed) > spare:
            break
        sets = [E for E in itertools.combinations(kept, e) if consistent(oracle, b, parts, c, s, [p for p in kept if p not in E], cols)]
        assert len(sets) <= 1, ("two sets within the radius explain the stripe", c, s, sets)
        if sets:
            return sets[0]
    return None


def expected_entry(oracle, b, pristine, given, c, s, decode):
    """(the entry as a tuple, {part: block written}) of stripe s of chunk c, by the rules of lzgpu_repair_stripes and (decode)
    lzgpu_decode_stripes in include/lzgpu.h"""
    g = sorted(given)
    spare = len(g) - b.k
    failed = [p for p in g if crc_of(block(b.parts, p, c, s)) != int(b.crc[p][c, s])]
    state = expected_map(oracle, stripe_view(b, b.parts, c, s), g)[0, 0]
    bad_rows, suspect = int(state["bad_rows"]), int(state["suspect_part"])
    crc, written = 0, {}
    if not failed:                                        # 1: the degraded correction (its CRC gate passes: no block fails)
        if not bad_rows:
            status = _lib.FIX_CLEAN
        elif suspect < 0:
            status = _lib.FIX_UNEXPLAINED
        else:
            written = oracle_rebuild(oracle, b, b.parts, c, s, {suspect}, given)
            status, crc = _lib.FIX_CORRECTED, crc_of(written[suspect])
    elif not bad_rows:                                    # 2
        status = _lib.FIX_CRC_ONLY
    elif len(failed) > spare:                             # 4
        status = _lib.FIX_CRC_CONFLICT
    else:                                                 # 3: F rebuilt from the first k given parts outside F, gated by F's CRCs
        out = oracle_rebuild(oracle, b, b.parts, c, s, set(failed), given)
        if all(crc_of(out[p]) == int(b.crc[p][c, s]) for p in failed):
            status, written = _lib.FIX_REBUILT, out
        else:
            status = _lib.FIX_CRC_CONFLICT
    if not decode:
        return (bad_rows, suspect, status, crc, mask(failed)), written
    located, lcrc = 0, [0, 0]
    if status in UNRESOLVED:                              # decode rule 2: the code punctured by F locates E
        E = brute_force(oracle, b, b.parts, pristine, c, s, given, failed)
        if E:
            out = oracle_rebuild(oracle, b, b.parts, c, s, set(failed) | set(E), given)
            if all(crc_of(out[p]) == int(b.crc[p][c, s]) for p in failed):
                status, crc, written, located = _lib.FIX_DECODED, 0, out, mask(E)
                lcrc = [crc_of(out[p]) for p in sorted(E)] + [0] * (2 - len(E))
    return (bad_rows, suspect, status, crc, mask(failed), located, lcrc[0], lcrc[1]), written


def touched(b, pristine, c, s):
    """stripe s of chunk c differs from the pristine batch in a block or a stored CRC"""
    return any(int(b.crc[p][c, s]) != int(pristine.crc[p][c, s]) or (block(b.parts, p, c, s) != block(pristine.parts, p, c, s)).any()
               for p in range(b.k + b.m))


def expected(oracle, b, pristine, given, decode, work=None):
    """(entries [n][pb] as tuples, the given parts after the call); work: the stripes that differ from the pristine batch (default:
    found by comparison); every other stripe is the pristine codeword with valid CRCs, so CLEAN"""
    work = [(c, s) for c in range(b.n) for s in range(b.pb) if touched(b, pristine, c, s)] if work is None else work
    clean = (0, -1, _lib.FIX_CLEAN, 0, 0) + ((0, 0, 0) if decode else ())
    ents = [[clean] * b.pb for _ in range(b.n)]
    written = {}
    for c, s in work:
        ents[c][s], w = expected_entry(oracle, b, pristine.parts, given, c, s, decode)
        written.update({(c, s, p): blk for p, blk in w.items()})
    assert all(p in given for _, _, p in written)
    return ents, written


def resolved(oracle, b, given, ents, written):
    """with each entry's new CRCs stored (CORRECTED: crc; DECODED: located_crc), every given block of a stripe matches its stored CRC
    unless the stripe is CRC_ONLY or CRC_CONFLICT, and the oracle's map of the result is clean unless the stripe is UNEXPLAINED or
    CRC_CONFLICT"""
    for c, row in enumerate(ents):
        for s, e in enumerate(row):
            if e[2] == _lib.FIX_CLEAN and not any((c, s, p) in written for p in given):
                continue
            view = stripe_view(b, b.parts, c, s)
            view.parts = [v.copy() for v in view.parts]
            crcs = {p: int(b.crc[p][c, s]) for p in given}
            for p in given:
                if (c, s, p) in written:
                    view.parts[p][0] = written[(c, s, p)]
            if e[2] == _lib.FIX_CORRECTED:
                crcs[e[1]] = e[3]
            if len(e) > 5:
                for p, v in zip(sorted(p for p in given if e[5] >> p & 1), e[6:]):
                    crcs[p] = v
            ok = {p: crc_of(view.parts[p][0]) == crcs[p] for p in given}
            assert all(ok.values()) or e[2] in CRC_LEFT, (c, s, e, ok)
            bad = int(expected_map(oracle, view, sorted(given))[0, 0]["bad_rows"])
            assert bad == 0 or e[2] in UNRESOLVED, (c, s, e)


def apply(parts, written):
    out = [p.copy() for p in parts]
    for (cc, s, p), blk in written.items():
        block(out, p, cc, s)[:] = blk
    return out


# ---- the faults of a case ----------------------------------------------------------------------------------------------------------

def classes(b, given):
    """(given data parts, input parity parts, spares): the inputs are the first k given parts"""
    inputs, spares = SD.roles(b, sorted(given))
    return [p for p in inputs if p < b.k], [p for p in inputs if p >= b.k], spares


def spread(b, given, n, start=0, skip=()):
    """n given parts outside skip, taken in turn from the data parts, the input parity parts and the spares (from class `start`)"""
    cls = [c for c in ([p for p in c if p not in skip] for c in classes(b, given)) if c]
    cls = cls[start % len(cls):] + cls[:start % len(cls)]
    order = [c[r] for r in range(max(map(len, cls))) for c in cls if r < len(c)]
    assert len(order) >= n, (n, order)
    return order[:n]


def inject(b, given, G, seed):
    """the faults of the module docstring; returns {(chunk, stripe): kind}"""
    k, pb = b.k, b.pb
    spare = len(given) - k
    used = {}

    def slot(s, kind, prefer=0):
        for c in (prefer, 2 - prefer):
            if (c, s) not in used:
                used[(c, s)] = kind
                return c
        raise AssertionError(("no free chunk for stripe", s))

    data = [p for p in sorted(given) if p < k]
    inputs, _ = SD.roles(b, sorted(given))
    rot(b, slot(0, "rot data"), data[len(data) // 2], 0, offset=16384 + 11)
    b.corrupt(slot(G - 1, "stale"), inputs[-1], G - 1, offset=40000)
    c = slot(G, "rot given - k")
    for i, p in enumerate(spread(b, given, spare)):
        rot(b, c, p, G, offset=16384 * (i % 4) + 97 * i)
    for q, s in ((1, G + 16), (2, G + 32)):
        if s < pb:
            rot(b, slot(s, f"rot quarter {q}", prefer=2), spread(b, given, q + 1)[q], s, offset=16384 * q + 5)
    c = slot(2 * G, "rot given - k + 1")
    for i, p in enumerate(spread(b, given, spare + 1, start=1)):
        rot(b, c, p, 2 * G, offset=16384 * ((i + 2) % 4) + 31 * i)
    # the short last stripe: the last byte of data part 0, and a zero-padded block of another data part
    padded = [p for p in data if p > 0][:1]
    last = ([0] if 0 in given else []) + padded
    c = slot(pb - 1, "short stripe", prefer=2)
    for i, p in enumerate(last):
        if i and spare < 2:
            c = slot(pb - 1, "short stripe", prefer=c)
        rot(b, c, p, pb - 1, offset=BLOCK - 1 if p == 0 else 20000, length=1 if p == 0 else 3)
    rng = np.random.default_rng(seed)
    free = [(c, s) for c in (0, 2) for s in range(pb) if (c, s) not in used]
    order = [free[i] for i in rng.permutation(len(free))]
    c, s = order.pop()
    used[(c, s)] = "wrong stored CRC"
    b.crc[sorted(given)[-1]][c, s] ^= 0x10
    c, s = order.pop()
    used[(c, s)] = "stale input beside rot"
    r = spread(b, given, 1, start=2)[0]
    rot(b, c, r, s, offset=777)
    b.corrupt(c, [p for p in sorted(given) if p != r][:k][-1], s, offset=50000)
    for c, s in order[:4]:
        p, offset = int(rng.choice(sorted(given))), int(rng.integers(0, BLOCK - 8))
        used[(c, s)] = "rot" if rng.integers(2) else "stale"
        if used[(c, s)] == "rot":
            rot(b, c, p, s, offset=offset)
        else:
            b.corrupt(c, p, s, offset=offset)
    return used


# ---- GPU runs ------------------------------------------------------------------------------------------------------------------------

def rows_of(fix, dtype):
    return entries(fix) if dtype is DECODE else fix_list(fix)


def check_launch(eng, ctx, plan, b, given, fn):
    """fn() on context ctx; lzgpu_debug_last_geometry afterwards is the plan's check launch (none on the generic route)"""
    before = eng.last_geometry()
    out = fn()
    want, got = expected_geometry(ctx, plan, b), eng.last_geometry()
    if want is None:
        assert got["kernel"] not in (_lib.KERNEL_CHECK, _lib.KERNEL_CHECK_DEGRADED) or got == before, (ctx, got)
    else:
        if any(j not in given for j in range(b.k)):
            want["kernel"] = _lib.KERNEL_CHECK_DEGRADED
        assert got == want, (ctx, got, want)
    return out


def outside_untouched(b, bufs, dev, lead):
    for i in range(b.k + b.m):                            # the stride gaps and the bytes past the last chunk
        outside = np.ones(len(bufs[i]), dtype=bool)
        for c in range(b.n):
            outside[lead + c * dev.stride: lead + c * dev.stride + b.pb * BLOCK] = False
        host_init = np.random.default_rng(7).integers(0, 256, len(bufs[i]), dtype=np.uint8)
        assert (bufs[i][outside] == host_init[outside]).all(), i


def expected_case(oracle, b, pristine, given, kinds):
    """{call: (entries, parts after)} of both calls, after checking them against the statuses the faults of inject() are meant to
    reach and the pristine bytes"""
    out = {}
    spare = len(given) - b.k
    for call, dtype in CALLS:
        ents, written = expected(oracle, b, pristine, given, dtype is DECODE)
        resolved(oracle, b, given, ents, written)
        out[call] = (ents, apply(b.parts, written))
    rep, dec = out["repair_stripes"][0], out["decode_stripes"][0]
    want = {"rot data": _lib.FIX_REBUILT, "rot given - k": _lib.FIX_REBUILT, "rot quarter 1": _lib.FIX_REBUILT,
            "rot quarter 2": _lib.FIX_REBUILT, "short stripe": _lib.FIX_REBUILT,
            "stale": _lib.FIX_CORRECTED if spare >= 2 else _lib.FIX_UNEXPLAINED, "rot given - k + 1": _lib.FIX_CRC_CONFLICT,
            "stale input beside rot": _lib.FIX_CRC_CONFLICT, "wrong stored CRC": _lib.FIX_CRC_ONLY}
    for (c, s), kind in kinds.items():
        assert c != 1 and rep[c][s][2] == want.get(kind, rep[c][s][2]), (c, s, kind, rep[c][s])
        if kind == "stale input beside rot":
            assert dec[c][s][2] == (_lib.FIX_DECODED if spare >= 3 else _lib.FIX_CRC_CONFLICT), (c, s, dec[c][s])
    for call, (ents, after) in out.items():               # every stripe written is back to the pristine bytes
        for c, s in kinds:
            if ents[c][s][2] in (_lib.FIX_REBUILT, _lib.FIX_CORRECTED, _lib.FIX_DECODED):
                assert all((block(after, p, c, s) == block(pristine.parts, p, c, s)).all() for p in given), (call, c, s)
    return out


def prepare_case(oracle, case):
    """(pristine, b, given, plan, kinds) of CASES[case], the faults injected"""
    name, lost, rows, want = CASES[case]
    g = L.SliceType(name)
    plan = plan_of(g, lost, rows)
    assert SD.literal(plan) == want
    pb, nb = CG.shape_of(g, plan["G"])
    given = {i for i in range(g.k) if i not in lost} | {g.k + r for r in rows}
    pristine, b = twin(oracle, name, 3, nb, seed=300 + case)
    kinds = inject(b, given, plan["G"], seed=case)
    return pristine, b, given, plan, kinds


def run_case(oracle, b, given, plan, want, contexts=CG.CONTEXTS, dev_pad=65536 + 48, lead=16):
    """both calls, host and _dev, on every context, against want = expected_case()"""
    for call, dtype in CALLS:
        ents, want_parts = want[call]
        crc_left = any(e[2] in CRC_LEFT for row in ents for e in row)
        for ctx, env in contexts.items():
            eng = engine(**env)
            after = [p.copy() for p in b.parts]
            fix, where = check_launch(eng, ctx, plan, b, given, lambda: host_result(
                lambda: getattr(eng, call)(b.goal, b.nb, given_list(b, given, after), crc_list(b, given)), "fix"))
            assert rows_of(fix, dtype) == ents, (ctx, call)
            assert (where is not None) == crc_left, (ctx, call, where)
            assert all((after[i] == want_parts[i]).all() for i in range(b.k + b.m)), (ctx, call)
            del after
            dev = Dev(b, dev_pad, lead)
            fix = check_launch(eng, ctx, plan, b, given, lambda: dev_fix(eng, call + "_dev", b, dev, given, dtype=dtype))
            assert rows_of(fix, dtype) == ents, (ctx, call, "_dev")
            parts, bufs = dev_parts(b, dev, lead)
            assert all((parts[i] == want_parts[i]).all() for i in range(b.k + b.m)), (ctx, call, "_dev")
            outside_untouched(b, bufs, dev, lead)
            del dev, parts, bufs
            assert eng.status_slots()[1] == 0


@gpu
@pytest.mark.parametrize("case", range(len(CASES)),
                         ids=[f"{c[0]}-lost{'.'.join(map(str, c[1]))}-rows{''.join(map(str, c[2]))}" for c in CASES])
def test_geometry_case(oracle, case):
    pristine, b, given, plan, kinds = prepare_case(oracle, case)
    run_case(oracle, b, given, plan, expected_case(oracle, b, pristine, given, kinds))


# ---- the decode's radius -----------------------------------------------------------------------------------------------------------

# (goal, lost parts): spares s = given - k from 3 to 8; a lost data part makes a parity part an input.  The Cauchy goals (m >= 5)
# take the generic check route.
RADIUS = [("ec(8,3)", ()), ("ec(8,4)", (2,)), ("ec(8,4)", ()), ("ec(6,5)", (1,)), ("ec(6,5)", ()), ("ec(4,6)", (0,)),
          ("ec(4,6)", ()), ("ec(10,8)", (3,)), ("ec(10,8)", ())]


def radius_patterns(spare):
    """(|F|, e, inside): every |F| and e, 1 <= e <= 2, with 2 e + |F| <= s, and the patterns with 2 e + |F| = s + 1"""
    inside = [(nf, e, True) for e in (1, 2) for nf in range(spare - 2 * e + 1)]
    return inside + [(spare - 1, 1, False)] + [(spare - 3, 2, False)] * (spare >= 3)


def radius_case(oracle, name, lost):
    """(b, given, {call: (entries, parts after)}): one stripe per pattern and placement, F (rot) and E (stale) taken in turn from the
    data parts, the input parity parts and the spares, one part of E always an input of F's rebuild (else the repair rebuilds F
    and the stale part survives, as documented).  Inside the radius the decode must locate E and restore the pristine bytes;
    beyond it, where it locates nothing, the repair's entry and bytes stand."""
    g = L.SliceType(name)
    given = {i for i in range(g.k + g.m) if i not in lost}
    spare = len(given) - g.k
    pats = [(nf, e, inside, j) for nf, e, inside in radius_patterns(spare) for j in range(3)]
    pristine, b = twin(oracle, name, 1, g.k * len(pats), seed=400 + g.k * 16 + spare)
    placed = []
    for s, (nf, e, inside, j) in enumerate(pats):
        F = spread(b, given, nf, start=j)
        ins = [p for p in sorted(given) if p not in F][:g.k]
        cand = spread(b, given, len(given) - nf, start=j + 1, skip=F)
        first = next(p for p in cand if p in ins) if nf else cand[0]
        E = [first] + [p for p in cand if p != first][:e - 1]
        for i, p in enumerate(F):
            rot(b, 0, p, s, offset=16384 * (i % 4) + 300 * i + 7)
        for i, p in enumerate(E):
            b.corrupt(0, p, s, offset=[100, 102 if j else 60000][i] + 16384 * j)   # overlapping bytes, or disjoint ones
        placed.append((F, E))
    given_l = sorted(given)
    want = {}
    for call, dtype in CALLS:
        ents, written = expected(oracle, b, pristine, given, dtype is DECODE)
        resolved(oracle, b, given, ents, written)
        want[call] = (ents, apply(b.parts, written))
    rep, rep_parts = want["repair_stripes"]
    dec, dec_parts = want["decode_stripes"]
    for s, ((nf, e, inside, j), (F, E)) in enumerate(zip(pats, placed)):
        d = dec[0][s]
        assert d[4] == mask(F), (s, d)
        if inside:
            assert d[2] == (_lib.FIX_CORRECTED if (nf, e) == (0, 1) else _lib.FIX_DECODED), (s, nf, e, F, E, d)
            if d[2] == _lib.FIX_DECODED:
                assert d[5] == mask(E) and list(d[6:]) == [crc_of(block(pristine.parts, p, 0, s)) for p in sorted(E)] + [0] * (2 - e)
            else:
                assert d[1] == E[0] and d[3] == crc_of(block(pristine.parts, E[0], 0, s))
            assert all((block(dec_parts, p, 0, s) == block(pristine.parts, p, 0, s)).all() for p in given_l), (s, nf, e)
        elif d[2] != _lib.FIX_DECODED:                    # beyond: the repair's entry and bytes
            assert d[:5] == rep[0][s] and d[5:] == (0, 0, 0), (s, d, rep[0][s])
            assert all((block(dec_parts, p, 0, s) == block(rep_parts, p, 0, s)).all() for p in given_l), s
    return b, given, want


@gpu
@pytest.mark.parametrize("name,lost", RADIUS, ids=[f"{n}-lost{'.'.join(map(str, l))}" for n, l in RADIUS])
def test_decode_radius(oracle, name, lost):
    b, given, want = radius_case(oracle, name, lost)
    for call, dtype in CALLS:
        ents, want_parts = want[call]
        for env in ROUTES.values():
            eng = engine(**env)
            after = [p.copy() for p in b.parts]
            fix, _ = host_result(lambda: getattr(eng, call)(b.goal, b.nb, given_list(b, given, after), crc_list(b, given)), "fix")
            assert rows_of(fix, dtype) == ents, (call, env)
            assert all((after[i] == want_parts[i]).all() for i in range(b.k + b.m)), (call, env)


# ---- several working entries per CTA -------------------------------------------------------------------------------------------

# the entries i, i + grid, i + 2 grid, ... of a CTA i, in this order (rotated per CTA), and the statuses of the repair and the decode
SEQUENCES = {
    4: [("rot s", _lib.FIX_REBUILT, _lib.FIX_REBUILT), ("stale 1", _lib.FIX_CORRECTED, _lib.FIX_CORRECTED),
        ("rot 1", _lib.FIX_REBUILT, _lib.FIX_REBUILT), ("stale 2", _lib.FIX_UNEXPLAINED, _lib.FIX_DECODED),
        ("rot s - 2, stale input", _lib.FIX_CRC_CONFLICT, _lib.FIX_DECODED), ("rot s + 1", _lib.FIX_CRC_CONFLICT, _lib.FIX_CRC_CONFLICT),
        ("wrong stored CRC", _lib.FIX_CRC_ONLY, _lib.FIX_CRC_ONLY), ("clean", _lib.FIX_CLEAN, _lib.FIX_CLEAN)],
    3: [("rot s", _lib.FIX_REBUILT, _lib.FIX_REBUILT), ("stale 1", _lib.FIX_CORRECTED, _lib.FIX_CORRECTED),
        ("rot 1", _lib.FIX_REBUILT, _lib.FIX_REBUILT), ("rot s - 2, stale input", _lib.FIX_CRC_CONFLICT, _lib.FIX_DECODED),
        ("rot s + 1", _lib.FIX_CRC_CONFLICT, _lib.FIX_CRC_CONFLICT), ("clean", _lib.FIX_CLEAN, _lib.FIX_CLEAN)],
}


def put(b, given, kind, c, s, q):
    """the faults of `kind` in stripe s of chunk c; q varies the parts and the bytes"""
    spare = len(given) - b.k
    g = sorted(given)
    off = 16384 * (q % 4) + 113 * q
    if kind == "rot s":
        for i, p in enumerate(spread(b, given, spare, start=q)):
            rot(b, c, p, s, offset=(off + 16384 * i) % (BLOCK - 8))
    elif kind == "stale 1":
        b.corrupt(c, g[(3 + 5 * q) % len(g)], s, offset=off)
    elif kind == "rot 1":
        rot(b, c, g[(7 * q + 1) % len(g)], s, offset=off)
    elif kind == "stale 2":
        for i, p in enumerate(spread(b, given, 2, start=q)):
            b.corrupt(c, p, s, offset=(off + 20000 * i) % (BLOCK - 8))
    elif kind == "rot s - 2, stale input":
        F = spread(b, given, spare - 2, start=q + 1)
        for p in F:
            rot(b, c, p, s, offset=off)
        b.corrupt(c, [p for p in g if p not in F][:b.k][(q * 3) % b.k], s, offset=(off + 999) % (BLOCK - 8))
    elif kind == "rot s + 1":
        for i, p in enumerate(spread(b, given, spare + 1, start=q)):
            rot(b, c, p, s, offset=(off + 5000 * i) % (BLOCK - 8))
    elif kind == "wrong stored CRC":
        b.crc[g[q % len(g)]][c, s] ^= 0x400
    else:
        assert kind == "clean"


class Tiled(Batch):
    """n copies of one encoded 64 MiB chunk: parts and stored CRCs (the copies are codewords as the chunk is)"""

    def __init__(self, one, n):
        self.goal, self.k, self.m, self.kind = one.goal, one.k, one.m, one.kind
        self.n, self.nb, self.pb = n, one.nb, one.pb
        self.parts = [np.tile(p, (n, 1)) for p in one.parts]
        self.crc = [np.tile(c, (n, 1)) for c in one.crc]
        self.faulty = set()


@gpu
@pytest.mark.parametrize("lost", [(), (2,)], ids=["all-given", "lost2"])
def test_several_working_entries_per_cta(oracle, lost):
    """ec(8,4) over more than 6 x grid stripes, grid = min(entries, 2 x SMs) the CTAs of repair_map_kernel and decode_map_kernel
    (csrc/engine.cu, grid_for(..., 2)), each stepping over the entries by the grid.  Several CTAs get a sequence of working entries
    whose set X of rebuilt blocks changes size, from a different start each (so the first entry with work is not always the CTA's
    first); the shared arrays, the per-CTA setup and the per-entry counters must not carry over.  The _dev calls on the default
    context and the generic route; every entry and every byte against expected()."""
    import torch
    b, given, plan, want = cta_case(oracle, lost, sm_count())
    k, m, pb = b.k, b.m, b.pb
    for call, dtype in CALLS:
        ents, written = want[call]
        for ctx in ("default", "generic"):
            eng = engine(**CG.CONTEXTS[ctx])
            bufs = [torch.from_numpy(p).cuda() for p in b.parts]
            crcs = [torch.from_numpy(c.view(np.int32)).cuda() for c in b.crc]
            dev = types.SimpleNamespace(ptrs=[t.data_ptr() for t in bufs], crcs=[t.data_ptr() for t in crcs], stride=pb * BLOCK)
            fix = check_launch(eng, ctx, plan, b, given, lambda: dev_fix(eng, call + "_dev", b, dev, given, dtype=dtype))
            assert rows_of(fix, dtype) == ents, (call, ctx)
            for i in range(k + m):                        # part by part: the written blocks, then every other byte
                got = bufs[i].cpu().numpy()
                for (c, s, p), blk in written.items():
                    if p == i:
                        assert (block([got], 0, c, s) == blk).all(), (call, ctx, c, s, p)
                        block([got], 0, c, s)[:] = block(b.parts, p, c, s)
                assert (got == b.parts[i]).all(), (call, ctx, i)
                del got
            del bufs, crcs, dev
            torch.cuda.empty_cache()
            assert eng.status_slots()[1] == 0


def cta_case(oracle, lost, sms):
    """(b, given, plan, {call: (entries, blocks written)}) of test_several_working_entries_per_cta on a device with `sms` SMs"""
    k, m, pb = 8, 4, 128
    given = {i for i in range(k + m) if i not in lost}
    seq = SEQUENCES[len(given) - k]
    grid = 2 * sms
    n = -(-(max(len(seq), 7) * grid + 1) // pb)
    assert n * pb > 6 * grid and min(n * pb, 2 * sms) == grid
    one = Batch(oracle, "ec(8,4)", 1, k * pb, seed=500 + len(lost), tail=0)
    pristine = types.SimpleNamespace(parts=[np.broadcast_to(p, (n, pb * BLOCK)) for p in one.parts],
                                     crc=[np.broadcast_to(c, (n, pb)) for c in one.crc])
    b = Tiled(one, n)
    ctas = [0, 1, grid // 3, grid - 1]
    kinds = {}
    for q, i in enumerate(ctas):
        for j in range(len(seq)):
            e = i + j * grid
            kinds[e] = seq[(j + q) % len(seq)]
            put(b, given, kinds[e][0], e // pb, e % pb, q)
    plan = L.Engine.plan_check_degraded(b.goal, SD.flags(b.goal, set(lost)))
    want = {}
    for call, dtype in CALLS:
        work = [(e // pb, e % pb) for e in sorted(kinds)]
        ents, written = expected(oracle, b, pristine, given, dtype is DECODE, work=work)
        resolved(oracle, b, given, ents, written)
        for e, (kind, rep_status, dec_status) in kinds.items():
            assert ents[e // pb][e % pb][2] == (dec_status if dtype is DECODE else rep_status), (call, e, kind)
        for (c, s, p), blk in written.items():
            assert (blk == block(pristine.parts, p, c, s)).all(), (call, c, s, p)
        want[call] = (ents, written)
    return b, given, plan, want
