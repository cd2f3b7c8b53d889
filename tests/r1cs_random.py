"""Seeded generator of satisfiable random R1CS instances of general shape (test helper, not a test).

`DummyCircuit` and the reference's test `Circuit` have one entry per row in each matrix, three distinct columns and one or
two public inputs.  The instances made here have what real circuits have instead: any number of public inputs (zero
included, which formats to |X| = 1), several terms per linear combination, rows with an empty A or B, columns spread
over the whole witness or concentrated on a few hot ones, and coefficients 1, p - 1, small or random.

Construction (satisfiable by design):
- the public inputs and the `free` witnesses are random field elements;
- every live row draws its A and B terms from the free variables (One, the public inputs, the free witnesses);
- its C row holds optional free terms plus one dedicated output witness whose value makes the row hold;
- `echo` extra rows repeat a live row j as (k1 A_j) * (k2 B_j) = (k1 k2 C_j): more constraints than variables (a tall
  system) without new witnesses.
Witness columns are a random permutation of (free witnesses, outputs), and the terms of each row are emitted in random
column order: the ABI does not ask for sorted rows.

Matrices are emitted in the shape `b2m_index_create` takes (include/b2m.h: as `ConstraintSystem::to_matrices()` yields
them, whose rows ark-relations' `make_row` builds): no explicit zero coefficient (`make_row` drops them) and no
(row, column) twice in one matrix (a `LinearCombination` is compacted before it becomes a row).  Inputs outside that
shape are not something a real caller can produce, so parity on them would test nothing the reference defines.  Padding and squaring follow `marlin_b200.r1cs.from_rows`: the formatted input (One + public
inputs) is padded with zeros to a power of two, which moves every witness column up, and the matrices are made square
with empty rows (more variables) or witnesses equal to one (more constraints).

Field arithmetic runs on numpy object arrays of Python ints, so 2^18 rows take seconds.
"""
import numpy as np

from marlin_b200 import _lib, fields
from marlin_b200 import r1cs as gr1cs

COLUMN_MODES = ("uniform", "hot", "instance")


def _next_pow2(n):
    s = 1
    while s < n:
        s *= 2
    return s


class Generated:
    """One generated system.  `r1cs`: the padded, squared `marlin_b200.r1cs.R1CS`.  `public_input`: canonical ints without
    the leading one (what a verifier is given).  `nnz`: entries of the joint matrix (the |K| the index will use).  For
    small systems (`keep_rows=True`) also `rows` = (a_rows, b_rows, c_rows) as `from_rows` takes them, `instance` and
    `witness` (unpadded canonical ints), and `circuit(field)` -> the same system as an oracle circuit."""

    def __init__(self, curve_id, r1cs, public_input, nnz, live, free, echo):
        self.curve_id = curve_id
        self.r1cs = r1cs
        self.public_input = public_input
        self.nnz = nnz
        self.live, self.free, self.echo = live, free, echo
        self.rows = self.instance = self.witness = None

    @property
    def H(self):
        return _next_pow2(self.r1cs.num_constraints)

    @property
    def K(self):
        return _next_pow2(self.nnz)

    @property
    def X(self):
        return self.r1cs.num_instance

    def circuit(self, field):
        """oracle circuit `gen(cs)` for `oracle.r1cs.synthesize`: same variables in the same order, same rows."""
        assert self.rows is not None, "generate(..., keep_rows=True) for an oracle circuit"
        n_in = len(self.instance)
        instance, witness = list(self.instance), list(self.witness)
        a_rows, b_rows, c_rows = self.rows

        def gen(cs):
            var = [("i", 0)]
            var += [cs.new_input_variable(v) for v in instance[1:]]
            var += [cs.new_witness_variable(v) for v in witness]
            lc = lambda row: [(c, var[i]) for c, i in row]
            for ra, rb, rc in zip(a_rows, b_rows, c_rows):
                cs.enforce_constraint(lc(ra), lc(rb), lc(rc))
            assert len(var) == n_in + len(witness)

        return gen


def _draw_terms(rnd, spec, n):
    if isinstance(spec, int):
        return np.full(n, spec, dtype=np.int64)
    lo, hi = spec
    return rnd.integers(lo, hi + 1, size=n)


def generate(curve_id, seed, num_public, live, free, echo=0, terms=((3, 3), (3, 3), (1, 1)), columns="uniform", hot=4,
             hot_share=0.5, keep_rows=False):
    """curve_id: 0 BLS12-381, 1 BN254.  num_public: public inputs (0 allowed).  live: rows with an output witness.
    free: free witnesses.  echo: extra rows repeating a live row.  terms: per matrix an int or an inclusive (lo, hi)
    range; for C it counts the output witness, so C >= 1.  columns: "uniform" over the free variables, "hot" (a share
    `hot_share` of the terms land on `hot` columns: One, the first public input and free witnesses) or "instance"
    (three quarters of the terms on One and the public inputs)."""
    assert columns in COLUMN_MODES and live >= 1 and free + num_public >= 1
    assert (terms[2] if isinstance(terms[2], int) else terms[2][0]) >= 1, "C holds at least the output witness"
    p = fields.FR_MODULUS[curve_id]
    rnd = np.random.default_rng(seed)
    n_in = 1 + num_public                    # unformatted instance: One + public inputs
    n_wit = free + live                      # free witnesses, then one output per live row (before the permutation)
    n_var = n_in + n_wit

    def rand_fe(n):
        limbs = rnd.integers(0, 1 << 64, size=(n, 4), dtype=np.uint64, endpoint=False).astype(object)
        return (limbs[:, 0] + (limbs[:, 1] << 64) + (limbs[:, 2] << 128) + (limbs[:, 3] << 192)) % p

    def coeffs(n):
        """1, p - 1, small (2..65535) or random, a quarter each; never zero"""
        kind = rnd.integers(0, 4, size=n)
        out = np.empty(n, dtype=object)
        out[kind == 0] = 1
        out[kind == 1] = p - 1
        small = kind == 2
        out[small] = rnd.integers(2, 1 << 16, size=int(small.sum())).astype(object)
        big = kind == 3
        r = rand_fe(int(big.sum()))
        out[big] = np.where(r == 0, 1, r)
        return out

    # logical variables: 0 One, 1..num_public inputs, then witnesses; `perm` places witness k at column n_in + perm[k]
    perm = rnd.permutation(n_wit)
    free_vars = np.concatenate([np.arange(n_in), n_in + perm[:free]])
    out_vars = n_in + perm[free:]
    n_free = len(free_vars)
    if columns == "hot":
        hot_vars = np.asarray([0] + ([1] if num_public else []) + list(free_vars[n_in:n_in + hot]), dtype=np.int64)[:hot]
    instance_cols = np.arange(n_in)

    def pick(n):
        idx = free_vars[rnd.integers(0, n_free, size=n)]
        if columns == "hot":
            h = rnd.random(n) < hot_share
            idx[h] = hot_vars[rnd.integers(0, len(hot_vars), size=int(h.sum()))]
        elif columns == "instance":
            h = rnd.random(n) < 0.75
            idx[h] = instance_cols[rnd.integers(0, n_in, size=int(h.sum()))]
        return idx

    def matrix(counts):
        """per live row `counts[r]` distinct free columns -> (rows, cols) with duplicates inside a row dropped"""
        rows = np.repeat(np.arange(live), counts)
        cols = pick(len(rows))
        key = np.unique(rows.astype(np.int64) * n_var + cols)
        return key // n_var, key % n_var

    a_r, a_c = matrix(_draw_terms(rnd, terms[0], live))
    b_r, b_c = matrix(_draw_terms(rnd, terms[1], live))
    cf_r, cf_c = matrix(_draw_terms(rnd, terms[2], live) - 1)
    a_v, b_v, cf_v = coeffs(len(a_r)), coeffs(len(b_r)), coeffs(len(cf_r))

    # assignment by logical variable: One, public inputs, free witnesses random; outputs solved below
    z = np.zeros(n_var, dtype=object)
    z[0] = 1
    z[1:n_in] = rand_fe(num_public)
    z[free_vars[n_in:]] = rand_fe(free)

    def row_sums(r, c, v):
        s = np.zeros(live, dtype=object)
        if len(r):
            prod = v * z[c] % p
            starts = np.flatnonzero(np.r_[True, r[1:] != r[:-1]])
            s[r[starts]] = np.add.reduceat(prod, starts) % p
        return s

    az, bz, cfz = row_sums(a_r, a_c, a_v), row_sums(b_r, b_c, b_v), row_sums(cf_r, cf_c, cf_v)
    out_coeff = coeffs(live)
    inv = np.frompyfunc(lambda x: pow(int(x), -1, p), 1, 1)
    z[out_vars] = (az * bz - cfz) % p * inv(out_coeff) % p
    c_r = np.concatenate([cf_r, np.arange(live)])
    c_c = np.concatenate([cf_c, out_vars])
    c_v = np.concatenate([cf_v, out_coeff])

    # echo rows: (k1 A_j) * (k2 B_j) = (k1 k2 C_j), appended after the live rows
    mats = [[a_r, a_c, a_v], [b_r, b_c, b_v], [c_r, c_c, c_v]]
    if echo:
        src = rnd.integers(0, live, size=echo)
        k1, k2 = coeffs(echo), coeffs(echo)
        for m, k in zip(mats, (k1, k2, k1 * k2 % p)):
            r, c, v = m
            order = np.argsort(r, kind="stable")
            r, c, v = r[order], c[order], v[order]
            ptr = np.searchsorted(r, np.arange(live + 1))
            cnt = ptr[src + 1] - ptr[src]
            e_row = np.repeat(np.arange(echo), cnt)
            first = np.repeat(ptr[src], cnt)
            within = np.arange(len(e_row)) - np.repeat(np.cumsum(cnt) - cnt, cnt)
            take = first + within
            m[0] = np.concatenate([r, live + e_row])
            m[1] = np.concatenate([c, c[take]])
            m[2] = np.concatenate([v, v[take] * k[e_row] % p])
    n_con = live + echo

    # formatting [reference constraint_systems.rs:45-81]: pad the input, shift witness columns, square the matrices
    ni = _next_pow2(n_in)
    shift = ni - n_in
    nv = ni + n_wit
    n = max(nv, n_con)
    inst_vals = np.concatenate([z[:n_in], np.zeros(shift, dtype=object)])
    wit_vals = np.concatenate([z[n_in:], np.ones(n - nv, dtype=object)])
    R = (1 << 256) % p

    def mont_limbs(vals):
        m = np.asarray(vals, dtype=object) * R % p
        return np.stack([((m >> (64 * k)) & ((1 << 64) - 1)).astype(np.uint64) for k in range(4)], axis=1).reshape(len(vals), 4)

    out = []
    joint = []
    for r, c, v in mats:
        c = np.where(c < n_in, c, c + shift)
        # emit each row's terms in random order (the ABI must not rely on sorted rows)
        order = np.lexsort((rnd.random(len(r)), r))
        r, c, v = r[order], c[order].astype(np.uint64), v[order]
        row_ptr = np.searchsorted(r, np.arange(n + 1)).astype(np.uint64)
        if len(c) == 0:  # the placeholder `from_rows` emits for an empty matrix
            out.append((row_ptr, np.zeros(1, dtype=np.uint64), np.zeros((1, 4), dtype=np.uint64)))
        else:
            out.append((row_ptr, c, mont_limbs(v)))
        joint.append(r.astype(np.int64) * n + c.astype(np.int64))
        if keep_rows:
            ptr = [int(x) for x in row_ptr]
            out[-1] += ([[(int(x), int(i)) for i, x in zip(c[ptr[k]:ptr[k + 1]], v[ptr[k]:ptr[k + 1]])] for k in range(n_con)],)
    nnz = len(np.unique(np.concatenate(joint)))
    r1cs = gr1cs.R1CS(curve_id, ni, out[0][:3], out[1][:3], out[2][:3], mont_limbs(inst_vals), mont_limbs(wit_vals))
    g = Generated(curve_id, r1cs, [int(x) for x in z[1:n_in]], nnz, live, free, echo)
    if keep_rows:
        # unpadded numbering: witness columns before the input padding, as a circuit would write them
        unshift = lambda rows: [[(cf, i if i < n_in else i - shift) for cf, i in row] for row in rows]
        g.rows = tuple(unshift(m[3]) for m in out)
        g.instance = [int(x) for x in z[:n_in]]
        g.witness = [int(x) for x in z[n_in:]]
    return g


def shape(g):
    """"square" (as many variables as constraints before squaring), "tall" (more constraints) or "squat" (more variables)"""
    nv = g.X + g.free + g.live
    nc = g.live + g.echo
    return "square" if nv == nc else ("tall" if nc > nv else "squat")


# Small systems the Python oracle proves in seconds (|H| <= 256), shared by the CPU and GPU parity tests.  Between them
# they cover |X| = 1, 2, 4 and |H|/2; |K| < |H|, |K| = |H| and |K| >= 16 |H|; tall, squat and square shapes; hot columns;
# empty A and B rows; both curves (0 BLS12-381, 1 BN254) and both PC schemes (test_general_r1cs_cpu checks the coverage).
SMALL_CASES = {
    "x1-square": dict(curve=0, scheme="marlin_kzg10", seed=11, num_public=0, live=40, free=23, echo=24, terms=(3, 3, 1)),
    "x2-tall-hot": dict(curve=1, scheme="sonic_kzg10", seed=12, num_public=1, live=50, free=10, echo=40,
                        terms=((0, 4), (0, 4), (1, 3)), columns="hot"),
    "x4-squat-k-below-h": dict(curve=0, scheme="sonic_kzg10", seed=13, num_public=3, live=12, free=80, terms=(2, 2, 1)),
    "k-equals-h": dict(curve=1, scheme="marlin_kzg10", seed=14, num_public=2, live=16, free=44, terms=((0, 2), (1, 2), 1)),
    "x-half-h": dict(curve=1, scheme="marlin_kzg10", seed=15, num_public=31, live=24, free=4, echo=32, terms=(2, 2, 1),
                     columns="instance"),
    "k-far-above-h": dict(curve=0, scheme="sonic_kzg10", seed=16, num_public=3, live=12, free=12, echo=16,
                          terms=(12, 12, 4)),
    "hot-tall-empty-rows": dict(curve=0, scheme="marlin_kzg10", seed=17, num_public=7, live=60, free=20, echo=100,
                                terms=((0, 6), (0, 6), (1, 3)), columns="hot"),
}


def small_case(name, keep_rows=True):
    spec = dict(SMALL_CASES[name])
    spec.pop("scheme")
    return generate(spec.pop("curve"), keep_rows=keep_rows, **spec)


def satisfied(g):
    """(A z) o (B z) == C z on the padded system (canonical ints), for the generator's own self-check."""
    p = fields.FR_MODULUS[g.curve_id]
    c = g.r1cs
    to_int = lambda limbs: np.asarray([fields.fr_from_mont(g.curve_id, v) for v in _lib.limbs_to_ints(limbs)], dtype=object)
    z = np.concatenate([to_int(c.instance), to_int(c.witness)])
    res = []
    for row_ptr, col, coeff in (c.a, c.b, c.c):
        ne = int(row_ptr[-1])
        v = to_int(coeff[:ne]) * z[col[:ne].astype(np.int64)] % p if ne else np.zeros(0, dtype=object)
        s = np.zeros(c.num_constraints, dtype=object)
        rows = np.repeat(np.arange(c.num_constraints), np.diff(row_ptr.astype(np.int64)))
        np.add.at(s, rows, v)
        res.append(s % p)
    return bool(np.all(res[0] * res[1] % p == res[2]))
