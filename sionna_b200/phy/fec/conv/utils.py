"""Generator polynomials and the trellis of rate-1/n convolutional codes (mirror of fec/conv/utils.py:10-190)."""
import numpy as np

from ..utils import int2bin, bin2int

# Moon, "Error Correction Coding", tables of best free distance; K = 5 at rate 1/2 is the GSM 05.03 4.1.3 code.
_POLYS = {
    1 / 2: {3: ("101", "111"), 4: ("1101", "1011"), 5: ("10011", "11011"), 6: ("110101", "101111"),
            7: ("1011011", "1111001"), 8: ("11100101", "10011111")},
    1 / 3: {3: ("101", "111", "111"), 4: ("1011", "1101", "1111"), 5: ("10101", "11011", "11111"),
            6: ("100111", "101011", "111101"), 7: ("1111001", "1100101", "1011011"),
            8: ("10010101", "11011001", "11110111")},
}


def polynomial_selector(rate, constraint_length):
    """Generator polynomials (tuple of 0/1 strings) of the rate-``rate`` code with the given constraint length
    (fec/conv/utils.py:10-65): rate 1/2 or 1/3, constraint length 3 ... 8."""
    if not isinstance(constraint_length, int):
        raise TypeError("constraint_length must be int.")
    if not 2 < constraint_length < 9:
        raise ValueError("Unsupported constraint_length.")
    if rate not in (1 / 2, 1 / 3):
        raise ValueError("Unsupported rate.")
    return _POLYS[rate][constraint_length]


class Trellis:
    """State transitions and output symbols of a rate-1/n convolutional code (fec/conv/utils.py:68-190).

    The register of K = ``len(gen_poly[0])`` bits holds the new bit followed by the K - 1 state bits; the state is the
    K - 1 most recent bits with the newest as MSB. With ``rsc`` the first polynomial is the feedback polynomial: the
    new bit is the input plus the feedback parity of the state. All tables are int32 NumPy arrays:
    ``to_nodes[s, b]`` next state from s with input b; ``from_nodes[s, :]`` the two predecessors of s, in the order
    in which the loops over (input, state) reach them; ``op_mat[s, s']`` output symbol of s -> s' (-1: no edge);
    ``op_by_tonode`` / ``ip_by_tonode[s, :]`` output symbol / input of the transitions into s in from_nodes order;
    ``op_by_fromnode[s, b]`` output symbol from s with input b. Symbols hold output bit j at bit n - 1 - j."""

    def __init__(self, gen_poly, rsc=True):
        self.rsc = rsc
        self.gen_poly = gen_poly
        self.constraint_length = len(gen_poly[0])
        self.conv_k = 1
        self.conv_n = len(gen_poly)
        self.ni = 2 ** self.conv_k
        self.ns = 2 ** (self.constraint_length - 1)
        self._mu = self.constraint_length - 1
        if rsc:
            self.fb_poly = [int(x) for x in gen_poly[0]]
            assert self.fb_poly[0] == 1
        self._generate_transitions()

    def _generate_transitions(self):
        ns, ni, mu = self.ns, self.ni, self._mu
        polys = [[int(c) for c in p] for p in self.gen_poly]
        to_nodes = np.full((ns, ni), -1, np.int32)
        from_nodes = np.full((ns, ni), -1, np.int32)
        op_mat = np.full((ns, ns), -1, np.int32)
        ip_by_tonode = np.full((ns, ni), -1, np.int32)
        op_by_tonode = np.full((ns, ni), -1, np.int32)
        op_by_fromnode = np.full((ns, ni), -1, np.int32)
        filled = np.zeros(ns, int)
        for b in range(ni):                                  # input outer, state inner: fixes the from_nodes order
            for s in range(ns):
                state_bits = int2bin(s, mu)
                new_bit = b
                if self.rsc:
                    new_bit = (b + sum(x * f for x, f in zip(state_bits, self.fb_poly[1:]))) % 2
                reg = [new_bit] + state_bits
                nxt = bin2int(reg[:-1])
                op = bin2int([sum(r * g for r, g in zip(reg, p)) % 2 for p in polys])
                slot = filled[nxt]
                to_nodes[s, b] = nxt
                from_nodes[nxt, slot] = s
                op_mat[s, nxt] = op
                op_by_tonode[nxt, slot] = op
                ip_by_tonode[nxt, slot] = b
                op_by_fromnode[s, b] = op
                filled[nxt] += 1
        self.to_nodes, self.from_nodes, self.op_mat = to_nodes, from_nodes, op_mat
        self.ip_by_tonode, self.op_by_tonode, self.op_by_fromnode = ip_by_tonode, op_by_tonode, op_by_fromnode


def _select_gen_poly(gen_poly, rate, constraint_length, poly_msg):
    """The constructors' gen_poly checks (encoding.py:107-125, decoding.py:94-118): given polynomials must be equally
    long 0/1 strings; otherwise rate and constraint length pick a tabulated code."""
    if gen_poly is not None:
        if not all(isinstance(p, str) for p in gen_poly):
            raise TypeError(poly_msg)
        if not all(len(p) == len(gen_poly[0]) for p in gen_poly):
            raise ValueError("Each polynomial must be of same length.")
        if not all(all(c in "01" for c in p) for p in gen_poly):
            raise ValueError("Each polynomial must be a string of 0's and 1's.")
        return gen_poly
    if constraint_length not in (3, 4, 5, 6, 7, 8):
        raise ValueError("Constraint length must be between 3 and 8.")
    if rate not in (1 / 2, 1 / 3):
        raise ValueError("Rate must be 1/3 or 1/2.")
    return polynomial_selector(rate, constraint_length)


def _trellis_tables(trellis):
    """Host tables the decoder entry points take: contiguous int32 from_nodes, op_by_tonode, ip_by_tonode."""
    return tuple(np.ascontiguousarray(t, np.int32) for t in (trellis.from_nodes, trellis.op_by_tonode,
                                                              trellis.ip_by_tonode))
