"""R1CS instances in the array form the C ABI takes (`b2m_matrix`: CSR with Montgomery
coefficients), plus the reference's padding rules applied on the host:
`pad_input_for_indexer_and_prover` and `make_matrices_square` [reference
src/ahp/constraint_systems.rs:45-81, 282-290].  Variable numbering: One -> 0, instance k -> k,
witness k -> num_instance + k [U ark-relations].  Circuit synthesis itself (ark-relations'
ConstraintSystem DSL) is outside the hot path; the two circuit families the reference benches and
tests with are built here directly, vectorised so that 2^20+ constraints take milliseconds.
"""
import numpy as np

from . import _lib, fields


def _next_pow2(n):
    s = 1
    while s < n:
        s *= 2
    return s


class R1CS:
    """Padded, squared instance: matrices as CSR numpy arrays, assignments as Montgomery limbs."""

    def __init__(self, curve_id, num_instance, a, b, c, instance, witness, num_variables=None):
        self.curve_id = curve_id
        self.num_instance = num_instance          # formatted (includes the leading one), power of two
        self.a, self.b, self.c = a, b, c          # each: (row_ptr u64[n+1], col u64[nnz], coeff u64[nnz,4])
        self.instance = instance                  # u64[num_instance, 4], or None (matrices only)
        self.witness = witness                    # u64[num_witness, 4], or None (matrices only)
        self.num_constraints = len(a[0]) - 1
        # without an assignment the variable count is given (Marlin.load_r1cs)
        self.num_variables = num_instance + len(witness) if witness is not None else num_variables
        self.circom = None                        # marlin_b200.circom.CircomInfo of an instance loaded from circom files

    def matrices(self):
        out = []
        for row_ptr, col, coeff in (self.a, self.b, self.c):
            m = _lib.Matrix()
            m.row_ptr = row_ptr.ctypes.data
            m.col = col.ctypes.data
            m.coeff = coeff.ctypes.data
            out.append(m)
        return out

    def public_input(self):
        """unformatted public input as canonical python ints"""
        return [fields.fr_from_mont(self.curve_id, v) for v in _lib.limbs_to_ints(self.instance[1:])]


def _csr(rows_cols, rows_coeffs, n_rows):
    """rows_cols: list of per-row column lists (python), only for small instances."""
    row_ptr = np.zeros(n_rows + 1, dtype=np.uint64)
    cols, coeffs = [], []
    for r in range(n_rows):
        cols += rows_cols[r]
        coeffs += rows_coeffs[r]
        row_ptr[r + 1] = len(cols)
    col = np.asarray(cols, dtype=np.uint64).reshape(-1)
    coeff = _lib.ints_to_limbs(coeffs, 4) if coeffs else np.zeros((0, 4), dtype=np.uint64)
    if len(col) == 0:
        col = np.zeros(1, dtype=np.uint64)
        coeff = np.zeros((1, 4), dtype=np.uint64)
    return row_ptr, col, coeff


class Shape:
    """The padded, squared shape of an instance with ni0 formatted inputs (One included), num_witness witnesses and
    num_constraints rows [reference src/ahp/constraint_systems.rs:45-81, src/ahp/indexer.rs:151-167]:
    ni = next_pow2(ni0) instance entries, the last `shift` = ni - ni0 of them zero; column c of a variable goes to c when
    c < ni0 and to c + shift otherwise; with nv = ni + num_witness, `pad_rows` empty rows are appended when nv > nc, else
    `pad_witness` witnesses equal to one; `size` = rows = variables of the result."""

    def __init__(self, ni0, num_witness, num_constraints):
        self.ni0 = ni0
        self.ni = _next_pow2(ni0)
        self.shift = self.ni - ni0
        nv = self.ni + num_witness
        self.pad_rows = max(nv - num_constraints, 0)
        self.pad_witness = max(num_constraints - nv, 0)
        self.size = max(nv, num_constraints)

    def column(self, c):
        return c if c < self.ni0 else c + self.shift


def from_rows(curve_id, a_rows, b_rows, c_rows, instance, witness):
    """Generic (small) instance: *_rows[r] = [(coeff, col), ...] with canonical integer coefficients;
    instance / witness are canonical integers (instance includes the leading one).  Pads and squares (Shape)."""
    instance = list(instance)
    witness = list(witness)
    sh = Shape(len(instance), len(witness), len(a_rows))
    ni = sh.ni
    instance += [0] * sh.shift

    def remap(rows):
        return [[(c, sh.column(i)) for c, i in row] for row in rows] + [[] for _ in range(sh.pad_rows)]

    a_rows, b_rows, c_rows = remap(a_rows), remap(b_rows), remap(c_rows)
    witness += [1] * sh.pad_witness
    n = len(a_rows)
    mont = lambda v: fields.fr_to_mont(curve_id, v)
    mats = []
    for rows in (a_rows, b_rows, c_rows):
        mats.append(_csr([[i for _, i in row] for row in rows], [[mont(c) for c, _ in row] for row in rows], n))
    inst = _lib.ints_to_limbs([mont(v) for v in instance], 4)
    wit = _lib.ints_to_limbs([mont(v) for v in witness], 4)
    return R1CS(curve_id, ni, mats[0], mats[1], mats[2], inst, wit)


def _single_entry_csr(n_rows, n_live, col, one_limbs):
    """rows 0..n_live-1 hold the single entry (1, col); the rest are empty."""
    row_ptr = np.minimum(np.arange(n_rows + 1, dtype=np.uint64), np.uint64(n_live))
    cols = np.full(max(n_live, 1), col, dtype=np.uint64)
    coeff = np.tile(one_limbs, (max(n_live, 1), 1))
    return row_ptr, cols, coeff


def dummy_circuit(curve_id, a, b, num_variables, num_constraints):
    """`DummyCircuit` [reference benches/bench.rs:25-67]: witnesses a, b (+ num_variables - 3 copies of a),
    public input c = a*b, num_constraints - 1 copies of a*b = c and one empty constraint."""
    p = fields.FR_MODULUS[curve_id]
    mont = lambda v: np.asarray(_lib.ints_to_limbs([fields.fr_to_mont(curve_id, v)], 4)[0])
    one, a_l, b_l = mont(1), mont(a), mont(b)
    ni = 2                       # [one, c]: already a power of two
    n_w = 2 + (num_variables - 3)
    nv = ni + n_w
    nc = num_constraints
    live = num_constraints - 1
    pad_w = 0
    if nv > nc:
        nc = nv                  # dummy 0*0 = 0 constraints
    else:
        pad_w = nc - nv          # unconstrained witnesses equal to one
    witness = np.empty((n_w + pad_w, 4), dtype=np.uint64)
    witness[:n_w] = a_l
    witness[1] = b_l
    witness[n_w:] = one
    instance = np.stack([one, mont(a * b % p)])
    # columns: c -> 1, a -> ni + 0, b -> ni + 1
    A = _single_entry_csr(nc, live, ni + 0, one)
    B = _single_entry_csr(nc, live, ni + 1, one)
    C = _single_entry_csr(nc, live, 1, one)
    return R1CS(curve_id, ni, A, B, C, instance, witness)


def test_circuit(curve_id, a, b, num_constraints, num_variables):
    """`Circuit` of the reference's tests [reference src/test.rs:8-50]: inputs c = a*b, d = c*b."""
    p = fields.FR_MODULUS[curve_id]
    c = a * b % p
    d = c * b % p
    instance = [1, c, d]
    witness = [a, b] + [a] * (num_variables - 3)
    wa, wb = 3, 4  # before input padding: instance has 3 entries -> witness columns start at 3
    a_rows = [[(1, wa)] for _ in range(num_constraints - 1)] + [[(1, 1)]]
    b_rows = [[(1, wb)] for _ in range(num_constraints)]
    c_rows = [[(1, 1)] for _ in range(num_constraints - 1)] + [[(1, 2)]]
    return from_rows(curve_id, a_rows, b_rows, c_rows, instance, witness)
