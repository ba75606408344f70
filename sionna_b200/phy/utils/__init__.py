"""Utilities (mirror of sionna.phy.utils for the hot path)."""
from .tensors import expand_to_rank, flatten_dims, flatten_last_dims, insert_dims, split_dim
from .misc import complex_normal, ebnodb2no, hard_decisions, sim_ber, db_to_lin, lin_to_db
from .metrics import compute_ber, compute_bler, count_errors, count_block_errors, ErrorCounter
from .linalg import inv_cholesky, matrix_pinv
