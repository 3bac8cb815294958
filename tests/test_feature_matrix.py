"""The attention features where they meet: a pairwise covering array of cases over both kernel families.

Every feature has a suite of its own (tests/test_causal.py, test_kv_group.py, test_varlen.py, test_paged_kv.py) that
holds the other features at their defaults.  This module runs them together: each case picks one value per axis of
AXES, and the cases cover every admissible pair of values (a greedy all-pairs construction, deterministic), plus the
TRIPLES below, whose paths pairs alone may miss.

Each case runs through the suites' own runners (fixed length: tests.test_kv_group.run, packed: tests.test_varlen.
run_packed, paged: tests.test_paged_kv.PagedRun) and is checked against the float64 reference assembled as
tests.test_varlen.reference does it.  The backward kernels recompute P from the L they stored, dQ computes D in FP32
from the stored O and dO, and dK / dV read the stored D; so the gradients are checked against a float64 backward that
takes those stored values, and the stored L and D are checked on their own, with the rounding of their storage format
(FP16 L, BF16 D under lowPrecisionIntermediates) on top.  This keeps one set of gradient bounds for FP32 and 16-bit
intermediates alike.  Every case also checks the rows that see no key (L = +inf, O = D = dQ = 0), finite outputs
elsewhere, untouched sentinels, and a second run that is bitwise identical."""
import itertools

import numpy as np
import pytest

import mfa_b200 as mfa
import oracle
from tests.test_varlen import LOG2E, _offsets, reference

KT, Op, P = mfa.AttentionKernelType, mfa.AttentionOperand, mfa.GEMMOperandPrecision

AXES = {
    "entry": ("fixed", "packed", "paged"),                 # encode(), sequences=, paged= (forward only)
    "operands": ("bf16", "fp16", "reference", "fp32"),    # reference: FP16 Q/K/V + BF16 dO
    "D": (36, 64, 72, 128, 196, 256, 320),                # 36, 196: staged (D % 8 != 0); 16-bit 320: SIMT family
    "causal": (False, True),
    "G": (1, 3, 4),                                        # query heads per K/V head (2 K/V heads)
    "mid": ("fp32", "low"),                                # low: FP16 L + BF16 D (lowPrecisionIntermediates)
    "split": ("default", "off", "forced"),                 # fixed-length tensor-core calls: the plan, (0, 1), (1, 8)
    "transpose": ("none", "aligned", "unaligned"),         # fixed only; unaligned routes 16-bit operands to SIMT
    "scores": ("standard", "sharp", "sink"),
    "shape": ("short", "tall", "tiny"),                    # R < C, R > C, 1 to 8 rows or keys
    "page": (None, 16, 64, 256),                           # paged only
}

# Paths the pairs alone may miss (partial cases; each must be contained in at least one case)
TRIPLES = [
    # FP16 L = +inf of the rows of a sequence without keys, read back by the packed dK/dV kernel
    {"entry": "packed", "mid": "low", "causal": True, "shape": "tall", "operands": "fp32"},
    {"entry": "paged", "mid": "low", "page": 16},
    {"entry": "fixed", "split": "forced", "G": 4, "causal": True, "mid": "low"},
    # 16-bit D = 320 packed: the SIMT family in all three kernels, dK/dV over two head slices
    {"operands": "bf16", "D": 320, "entry": "packed", "G": 4},
    # every split range but the first has a merge weight near 0
    {"scores": "sink", "split": "forced"},
    # the largest |L| in FP16, with dO converted to FP16 on chip
    {"scores": "sharp", "mid": "low", "operands": "reference"},
]

TRANSPOSE_MASK = {"none": (False,) * 4, "aligned": (True,) * 4, "unaligned": (False, True, True, False)}

# fixed-length (R, C): every length a multiple of 8 for aligned transposes, none of them for unaligned ones
FIXED_SHAPES = {"short": ((136, 296), (100, 300)), "tall": ((296, 200), (300, 199)), "tiny": ((8, 296), (5, 300))}
# packed / paged (query lengths, key lengths)
LENGTHS = {
    "short": ([1, 63, 0, 129, 65, 40], [5, 64, 30, 300, 65, 41]),    # an empty query sequence, Rs <= Cs
    "tall": ([129, 65, 1, 64, 200], [63, 0, 1, 65, 100]),           # an empty key sequence, Rs > Cs
    "tiny": ([1, 8, 0, 3, 5], [7, 1, 4, 0, 8]),
}


def family(case):
    """The kernel family a (complete) case is written for: every kernel type of it runs there."""
    if case["operands"] == "fp32" or case["D"] > 256:
        return mfa.Backend.simtFP32
    if case["transpose"] == "unaligned" or (case["transpose"] == "aligned" and case["D"] % 8 != 0):
        return mfa.Backend.simtFP32    # (transposed operands are staged only with D % 8 == 0)
    return mfa.Backend.tcgen05


def admissible(case):
    """The constraints, on a partial case (axes not yet chosen are unconstrained)."""
    get = case.get
    if get("entry") not in (None, "fixed"):
        if get("transpose") not in (None, "none") or get("split") not in (None, "default"):
            return False
    if get("entry") is not None and get("page", 0) != 0 and (get("entry") == "paged") != (get("page") is not None):
        return False
    if get("entry") == "paged" and get("operands") not in (None, "fp32") and get("D") in (36, 196):
        return False           # the tensor-core paged forward needs D % 8 == 0
    if get("split") not in (None, "default"):
        if get("operands") == "fp32" or get("D") == 320 or get("transpose") == "unaligned":
            return False
        if get("transpose") == "aligned" and get("D") in (36, 196):
            return False
    return True


def _complete(case, order):
    """The first admissible completion of `case` over the axes in `order`, or None."""
    if not order:
        return dict(case)
    axis, rest = order[0], order[1:]
    if axis in case:
        return _complete(case, rest)
    for value in AXES[axis]:
        trial = dict(case, **{axis: value})
        if admissible(trial):
            done = _complete(trial, rest)
            if done is not None:
                return done
    return None


def _pairs_of(case):
    names = [a for a in AXES if a in case]
    return {((a, case[a]), (b, case[b])) for a, b in itertools.combinations(names, 2)}


def admissible_pairs():
    order = list(AXES)
    out = set()
    for a, b in itertools.combinations(order, 2):
        for x in AXES[a]:
            for y in AXES[b]:
                if _complete({a: x, b: y}, order) is not None:
                    out.add(((a, x), (b, y)))
    return out


def generate_cases():
    """TRIPLES first, then one case per still uncovered pair, each completed greedily: every further axis takes the
    admissible value that covers the most uncovered pairs (ties: the value least used so far, then AXES order)."""
    order = list(AXES)
    uncovered = admissible_pairs()
    used = {(a, v): 0 for a in AXES for v in AXES[a]}
    cases = []

    def grow(seed):
        case = dict(seed)
        for axis in order:
            if axis in case:
                continue
            best = None
            for value in AXES[axis]:
                trial = dict(case, **{axis: value})
                if not admissible(trial) or _complete(trial, order) is None:
                    continue
                gain = len(_pairs_of(trial) & uncovered) - len(_pairs_of(case) & uncovered)
                key = (gain, -used[(axis, value)])
                if best is None or key > best[0]:
                    best = (key, trial)
            case = best[1]
        for a, v in case.items():
            used[(a, v)] += 1
        uncovered.difference_update(_pairs_of(case))
        cases.append(case)

    for triple in TRIPLES:
        grow(triple)
    while uncovered:
        (a, x), (b, y) = min(uncovered, key=lambda p: (order.index(p[0][0]), order.index(p[1][0]), str(p)))
        grow({a: x, b: y})
    return cases


CASES = generate_cases()


def case_id(case):
    return "-".join([case["entry"], case["operands"], f"D{case['D']}", "causal" if case["causal"] else "full",
                     f"G{case['G']}", f"{case['mid']}L", f"split-{case['split']}", f"T-{case['transpose']}",
                     case["scores"], case["shape"]] + ([f"P{case['page']}"] if case["page"] else []))


# ------------------------------------------------------------------------------------------------ the calls
def _layout(case):
    """(qo, ko, rows, columns): sequence offsets and the buffers' rows (packed / paged: sentinel rows past the table)"""
    if case["entry"] == "fixed":
        R, C = FIXED_SHAPES[case["shape"]][case["transpose"] != "aligned"]
        return [0, R], [0, C], R, C
    rq, rk = LENGTHS[case["shape"]]
    qo, ko = _offsets(rq), _offsets(rk)
    return qo, ko, qo[-1] + 9, ko[-1] + 5


def descriptor(case):
    from tests.test_kv_group import _descriptor
    qo, ko, T, Tk = _layout(case)
    return _descriptor(T, Tk, case["D"], case["operands"], batch=2 * case["G"], causal=case["causal"],
                       transpose=TRANSPOSE_MASK[case["transpose"]], lowMid=case["mid"] == "low")


def _split_edit(case):
    policy = {"default": None, "off": (0, 1), "forced": (1, 8)}[case["split"]]
    if policy is None:
        return None

    def edit(kd):
        kd.splitPolicy = policy
    return edit


def _constants(case, desc):
    from tests.test_varlen import _constants as packed_constants
    qo, ko, T, Tk = _layout(case)
    H = desc.batchCount
    if case["entry"] == "paged":
        return packed_constants(T, 64 * case["page"], H, case["G"])
    return packed_constants(T, Tk, H, case["G"])


def _table(case):
    """The host-side table of a packed / paged call (pointers are not dereferenced by gridSize / launchCount)"""
    qo, ko, _, _ = _layout(case)
    if case["entry"] == "packed":
        return {"sequences": mfa.SequenceTable(len(qo) - 1, max(np.diff(qo)), max(np.diff(ko)), 16, 16)}
    if case["entry"] == "paged":
        return {"paged": mfa.PagedKV(len(qo) - 1, max(np.diff(qo)), 16, 16, 16, 4, case["page"])}
    return {}


def kernel_types(case):
    return (KT.forward,) if case["entry"] == "paged" else tuple(KT)


def inputs(case, desc):
    """Q, dO [H][T][D], K, V [H / G][Tk][D], rounded to the operands' memory formats.  sharp: Q and K x 3.  sink: the
    queries of each (K/V head, sequence) share a direction w (4 w added), key 0 is a multiple of their mean direction
    that puts about 1 - e^-2 / 9 (> 0.98) of a mean row's mass on it, and its value row gets +8."""
    qo, ko, T, Tk = _layout(case)
    D, G = case["D"], case["G"]
    H = desc.batchCount
    rng = np.random.default_rng(CASES.index(case) if case in CASES else 0)
    x = {Op.Q: rng.standard_normal((H, T, D)), Op.K: rng.standard_normal((H // G, Tk, D)),
         Op.V: rng.standard_normal((H // G, Tk, D)), Op.dO: rng.standard_normal((H, T, D))}
    if case["scores"] == "sharp":
        x[Op.Q] *= 3.0
        x[Op.K] *= 3.0
    elif case["scores"] == "sink":
        for g in range(H // G):
            for s in range(len(qo) - 1):
                q, k0 = slice(qo[s], qo[s + 1]), ko[s]
                if qo[s + 1] == qo[s] or ko[s + 1] == k0:
                    continue
                w = rng.standard_normal(D)
                x[Op.Q][g * G:(g + 1) * G, q] += 4.0 * w / np.linalg.norm(w)
                mean = x[Op.Q][g * G:(g + 1) * G, q].reshape(-1, D).mean(axis=0)
                u = mean / np.linalg.norm(mean)
                proj = float((x[Op.Q][g * G:(g + 1) * G, q] @ u).mean())
                x[Op.K][g, k0] = (np.log(9.0 * (ko[s + 1] - k0)) + 2.0) * np.sqrt(D) / proj * u
                x[Op.V][g, k0] += 8.0
    prec = desc.memoryPrecisions
    return {op: oracle.roundtrip(a.astype(np.float32), int(prec[op])) for op, a in x.items()}


def run_case(case, desc, x):
    """Raw outputs {name: float32 [heads][rows](...)} over the sequences' rows (L in log2 units, D pre-scaled);
    sentinels and tails are checked by the runners and here."""
    qo, ko, T, Tk = _layout(case)
    G = case["G"]
    if case["entry"] == "fixed":
        from tests.test_kv_group import run
        return run(desc, G, x, edit=_split_edit(case), raw=True)
    if case["entry"] == "packed":
        from tests.test_varlen import _check_sentinels, run_packed
        out = run_packed(desc, G, x, qo, ko)
        _check_sentinels(out, qo, ko)
        return {n: a[:, :qo[-1]] if n in ("O", "L", "D", "dQ") else a[:, :ko[-1]] for n, a in out.items()}
    from tests.test_paged_kv import PagedRun, _check_sentinels, build_pool
    lengths = np.diff(ko)
    Kp, Vp, table = build_pool(x[Op.K], x[Op.V], ko, case["page"], np.random.default_rng(case["page"]))
    paged = PagedRun(desc, G, x[Op.Q], Kp, Vp, qo, lengths, table)
    paged.encode()
    out = paged.results()
    _check_sentinels(out, qo)
    return {n: a[:, :qo[-1]] for n, a in out.items()}


# ------------------------------------------------------------------------------------------------ reference and bounds
def backward_from_stored(x, G, qo, ko, causal, O, L, Dkv):
    """float64 dQ, dK, dV with the kernels' statistics: P = exp2(S log2(e) - L) from the stored L (log2 units), D of
    dQ = rowsum(dO * O) from the stored O, D of dK / dV the stored D (oracle units)."""
    Q, K, V, dO = (np.asarray(x[op], np.float64)[:, :n] for op, n in ((Op.Q, qo[-1]), (Op.K, ko[-1]),
                                                                        (Op.V, ko[-1]), (Op.dO, qo[-1])))
    H, _, D = Q.shape
    scale = 1.0 / np.sqrt(D)
    out = {"dQ": np.zeros_like(Q), "dK": np.zeros_like(K), "dV": np.zeros_like(V)}
    for s in range(len(qo) - 1):
        q, k = slice(qo[s], qo[s + 1]), slice(ko[s], ko[s + 1])
        Rs, Cs = qo[s + 1] - qo[s], ko[s + 1] - ko[s]
        if Rs == 0 or Cs == 0:
            continue
        seen = np.arange(Cs)[None, :] <= np.arange(Rs)[:, None] + (Cs - Rs) if causal else np.ones((Rs, Cs), bool)
        for h in range(H):
            g = h // G
            S = Q[h, q] @ K[g, k].T * scale
            with np.errstate(invalid="ignore", over="ignore"):
                Pm = np.where(seen, np.exp2(S * np.log2(np.e) - np.asarray(L[h, q], np.float64)[:, None]), 0.0)
            dP = dO[h, q] @ V[g, k].T
            Dq = (dO[h, q] * np.asarray(O[h, q], np.float64)).sum(axis=1)
            out["dQ"][h, q] = (Pm * (dP - Dq[:, None]) * scale) @ K[g, k]
            dS = Pm * (dP - np.asarray(Dkv[h, q], np.float64)[:, None]) * scale
            out["dK"][g, k] += dS.T @ Q[h, q]
            out["dV"][g, k] += Pm.T @ dO[h, q]
    return out


def storage_error(values, prec):
    """The largest rounding error of storing `values` in `prec`: half an ulp (FP16 and FP32 round to nearest), one ulp
    for BF16 (stores truncate)."""
    mantissa = {P.FP32: 23, P.FP16: 10, P.BF16: 7}[prec]
    v = np.abs(np.asarray(values, np.float64)) * (1 + 2.0 ** -8)
    ulp = 2.0 ** (np.floor(np.log2(np.maximum(v, 2.0 ** -126))) - mantissa)
    if prec == P.FP16:
        ulp = np.maximum(ulp, 2.0 ** -24)
    return ulp if prec == P.BF16 else ulp / 2


def bounds(case, name, ref, small):
    """(max-abs bound, relative-RMS bound or None) of output `name` against its float64 reference: the bars the suites
    state.  The SIMT family computes in FP32 whatever the operands; the tensor-core family rounds P and dS to its
    16-bit operand type."""
    G = case["G"]
    peak = float(np.abs(ref).max()) if ref.size else 0.0
    group = np.sqrt(G) if name in ("dK", "dV") else 1.0
    if family(case) == mfa.Backend.simtFP32:
        return 2e-5 * max(1.0, peak) * group, None
    bf16 = case["operands"] == "bf16"
    if name == "O":
        return None, 2e-3 if bf16 else 3e-4     # (element-wise: eps_P * max|V|, in check_outputs)
    rel = (2.5e-3 if bf16 else 3e-4) * (1.5 if small else 1.0)
    return 5e-2 * group, rel


def _check_within(expected, actual, bound, name):
    """attention_harness.check with an element-wise bound (recorded as its largest value)."""
    from tests.attention_harness import record
    record(name, expected, actual, float(np.max(bound)) if np.size(bound) else 0.0)
    err = np.abs(np.asarray(expected, np.float64) - np.asarray(actual, np.float64))
    bad = ~(err <= bound)
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError(f"{int(bad.sum())} elements of {name} exceed their bound: {name}{i}: expected "
                             f"{expected[i]!r} actual {actual[i]!r} bound {np.broadcast_to(bound, err.shape)[i]!r}")


def _rel_rms(got, ref):
    from tests.test_tcgen05_backward import _rel_rms
    return _rel_rms(got, ref)


def check_outputs(case, desc, x, out):
    from tests.attention_harness import check
    qo, ko, _, _ = _layout(case)
    D = case["D"]
    T, Tk = qo[-1], ko[-1]
    prec = desc.memoryPrecisions
    ref = {n: a[:, :T] if n in ("O", "L", "D", "dQ") else a[:, :Tk]
           for n, a in reference(x, case["G"], qo, ko, case["causal"]).items()}
    rq, rk = np.diff(qo), np.diff(ko)
    small = min(int(rq[rq > 0].min()), int(rk[rk > 0].min()), D) < 16
    empty = np.isposinf(ref["L"])                        # rows that see no key

    # rows that see no key: L = +inf exactly (also as FP16), O = 0; every other output finite
    assert (np.isposinf(out["L"]) == empty).all(), "L = +inf exactly on the rows that see no key"
    assert (out["O"][empty] == 0).all(), "O = 0 on the rows that see no key"
    for name, a in out.items():
        assert np.isfinite(a[~empty] if name in ("O", "L", "D", "dQ") else a).all(), name

    # O against the float64 reference
    tol, rel = bounds(case, "O", ref["O"], small)
    if tol is None:
        tol = (2.0 ** -8 if case["operands"] == "bf16" else 2.0 ** -10) * float(np.abs(x[Op.V]).max()) + 1e-5
    check(ref["O"], out["O"], tol, "O")
    if rel is not None:
        assert _rel_rms(out["O"], ref["O"]) <= rel, f"O: relative RMS {_rel_rms(out['O'], ref['O']):.3e} > {rel}"

    # the stored L: the float64 L within the kernel's bound plus its storage format's rounding
    L_nat = np.where(empty, 0.0, out["L"] / LOG2E)
    ref_L = np.where(empty, 0.0, ref["L"])
    base = 2e-5 * max(1.0, float(np.abs(ref_L).max())) if family(case) == mfa.Backend.simtFP32 else 1e-3
    _check_within(ref_L, L_nat, base + storage_error(ref_L * LOG2E, prec[Op.L]) / LOG2E, "L")
    if case["entry"] == "paged":
        return

    # the stored D: rowsum(dO * O) of the stored O in FP32, then rounded to its storage format (oracle units)
    dO64 = np.asarray(x[Op.dO][:, :T], np.float64)
    D_of_O = (dO64 * out["O"]).sum(axis=-1)
    D_got = out["D"].astype(np.float64) * np.sqrt(D)
    assert (D_got[empty] == 0).all() and (out["dQ"][empty] == 0).all(), "D = dQ = 0 on the rows that see no key"
    magnitude = max(1.0, float(np.abs(dO64 * out["O"]).sum(axis=-1).max()))
    _check_within(D_of_O, D_got, 2e-5 * magnitude + storage_error(D_of_O / np.sqrt(D), prec[Op.D]) * np.sqrt(D),
                  "D")

    # gradients against the float64 backward on the stored statistics
    grads = backward_from_stored(x, case["G"], qo, ko, case["causal"], out["O"], out["L"], D_got)
    for name in ("dQ", "dK", "dV"):
        tol, rel = bounds(case, name, grads[name], small)
        check(grads[name], out[name], tol, name)
        if rel is not None and np.abs(grads[name]).max() > 0:
            got_rel = _rel_rms(out[name], grads[name])
            assert got_rel <= rel, f"{name}: relative RMS {got_rel:.3e} > {rel}"


# ------------------------------------------------------------------------------------------------ CPU: the matrix
def test_every_admissible_pair_and_triple_is_covered():
    pairs = set().union(*(_pairs_of(c) for c in CASES))
    missing = admissible_pairs() - pairs
    assert not missing, sorted(missing)[:10]
    for triple in TRIPLES:
        assert any(all(c[a] == v for a, v in triple.items()) for c in CASES), triple
    assert all(admissible(c) and set(c) == set(AXES) for c in CASES)
    assert 40 <= len(CASES) <= 70, len(CASES)
    assert len({case_id(c) for c in CASES}) == len(CASES)
    assert generate_cases() == CASES     # deterministic


def test_the_constraints():
    assert not admissible({"entry": "paged", "operands": "bf16", "D": 196})
    assert admissible({"entry": "paged", "operands": "fp32", "D": 196, "page": 64})
    assert not admissible({"entry": "packed", "transpose": "aligned"})
    assert not admissible({"entry": "packed", "page": 16}) and not admissible({"entry": "paged", "page": None})
    assert not admissible({"split": "forced", "operands": "fp32"})
    assert not admissible({"split": "off", "transpose": "aligned", "D": 36})
    assert not admissible({"split": "forced", "D": 320})
    # the sizes the float64 reference runs at stay small
    for c in CASES:
        qo, ko, T, Tk = _layout(c)
        assert 2 * c["G"] <= 8 and max(np.diff(qo)) <= 700 and max(np.diff(ko)) <= 700


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_case_reaches_its_kernel_family_and_plan(case):
    """Each kernel type runs on the family the case was written for, and launches exactly the kernel, + the split merge
    of a forced split whose traversal has two blocks or more, + one staging copy per staged operand."""
    desc = descriptor(case)
    _, _, R, C = _layout(case)     # (splits are forced on fixed-length calls only)
    c = _constants(case, desc)
    edit = _split_edit(case)
    transposed = desc.transposeState
    for t in kernel_types(case):
        kd = desc.kernelDescriptor(t)
        assert kd.backend == family(case), (t, kd.backend)
        if edit is not None:
            edit(kd)
        kernel = mfa.AttentionKernel(kd)
        staged = 0
        if family(case) == mfa.Backend.tcgen05:
            operands = {KT.forward: (Op.Q, Op.K, Op.V, Op.O), KT.backwardQuery: (Op.Q, Op.K, Op.V, Op.O, Op.dO, Op.dQ),
                        KT.backwardKeyValue: (Op.Q, Op.K, Op.V, Op.dO, Op.dV, Op.dK)}[t]
            follows = {Op.Q: 0, Op.dQ: 0, Op.K: 1, Op.dK: 1, Op.V: 2, Op.dV: 2, Op.O: 3, Op.dO: 3}
            staged = sum(1 for op in operands if case["D"] % 8 != 0 or transposed[follows[op]])
        launches = kernel.launchCount(c, **_table(case))
        if case["split"] == "default":     # (the parameter table's plan may split a fixed-length call)
            assert launches - staged in ((1, 2) if case["entry"] == "fixed" and family(case) == mfa.Backend.tcgen05
                                         else (1,)), (t, launches, staged)
            continue
        split = 0
        if case["split"] == "forced":
            traversal = C if t != KT.backwardKeyValue else R
            split = int(-(-traversal // kernel.blockDimensions[1]) >= 2)
        assert launches == 1 + split + staged, (t, launches, split, staged)


def test_the_stored_statistics_reference():
    """backward_from_stored with the float64 L and D is the float64 backward; storage_error bounds the formats."""
    rng = np.random.default_rng(0)
    rq, rk = [5, 0, 9, 4], [7, 3, 0, 2]
    qo, ko = _offsets(rq), _offsets(rk)
    x = {Op.Q: rng.standard_normal((4, qo[-1], 8)), Op.K: rng.standard_normal((2, ko[-1], 8)),
         Op.V: rng.standard_normal((2, ko[-1], 8)), Op.dO: rng.standard_normal((4, qo[-1], 8))}
    ref = reference(x, 2, qo, ko, True)
    got = backward_from_stored(x, 2, qo, ko, True, ref["O"], ref["L"] * np.log2(np.e), ref["D"])
    for name in ("dQ", "dK", "dV"):
        assert np.abs(got[name] - ref[name]).max() <= 1e-12, name
    v = rng.uniform(-70, 70, 1000).astype(np.float32)
    for prec in (P.FP16, P.BF16, P.FP32):
        assert (np.abs(oracle.roundtrip(v, int(prec)) - v) <= storage_error(v, prec)).all(), prec


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_feature_matrix(case):
    desc = descriptor(case)
    x = inputs(case, desc)
    out = run_case(case, desc, x)
    again = run_case(case, desc, x)
    for name, a in out.items():
        assert again[name].tobytes() == a.tobytes(), f"{name}: a second run differs"
    check_outputs(case, desc, x, out)
