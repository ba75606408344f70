"""LDPC belief-propagation decoders (mirror of /root/reference/src/sionna/phy/fec/ldpc/decoding.py).

``LDPCBPDecoder`` (decoding.py:13-637) and ``LDPC5GDecoder`` (:1169-1536) keep the reference's constructor
arguments, ``call(llr_ch, /, *, num_iter=None, msg_v2c=None)`` signature, logit sign convention and
``msg_v2c`` state layout. All arithmetic runs in ``sb_ldpc_decode`` (``csrc/ldpc_bp.cu``): one CTA per
codeword with the codeword's edge messages resident in shared memory for every iteration; rate recovery
(:1431-1475) and output slicing / re-interleaving (:1486-1536) are folded into the kernel's load and store
index maps, so the decoder moves 4*n bytes in and 4*k (or 4*n) bytes out per codeword and nothing else.
"""
import os
import types
import numpy as np
import scipy as sp
import scipy.sparse  # noqa: F401
import torch

from ...block import Block
from ...._lib import Handle, lib, check, ptr, current_stream
from .encoding import LDPC5GEncoder

_CN_RULES = {"boxplus-phi": 0, "boxplus": 1, "minsum": 2, "min": 2, "offset-minsum": 3, "identity": 4}
_VN_RULES = {"sum": 0, "identity": 1}


def _i32(a):
    return np.ascontiguousarray(np.asarray(a), dtype=np.int32)


class _GraphHandle(Handle):
    """Owns one ``sb_ldpc_graph`` (host plan + per-device copies of its tables)."""

    def __init__(self, num_cn, num_vn, cn_idx, vn_idx, in_map=None, n_in=0, out_vn=None, n_out=0, schedule=None,
                 cn_view=None):
        cn_idx, vn_idx = _i32(cn_idx), _i32(vn_idx)
        in_map = None if in_map is None else _i32(in_map)
        out_vn = None if out_vn is None else _i32(out_vn)
        n_sub = n_active = 0
        if schedule is not None:
            schedule = _i32(schedule)
            n_sub, n_active = schedule.shape
        args = (num_cn, num_vn, len(vn_idx), ptr(cn_idx), ptr(vn_idx), ptr(in_map), int(n_in), ptr(out_vn), int(n_out),
                ptr(schedule), int(n_sub), int(n_active))
        if cn_view is None:
            super().__init__("ldpc_graph", *args)
        else:
            cn_view = _i32(cn_view)
            super().__init__("ldpc_graph", *args, ptr(cn_view), create="sb_ldpc_graph_create_ordered")
        self.num_edges = len(vn_idx)
        self.n_in = int(n_in) if in_map is not None else num_vn
        self.n_out = int(n_out) if out_vn is not None else num_vn
        self._ws = None

    def on_chip(self):
        return bool(lib().sb_ldpc_graph_on_chip(self.handle))

    def set_qc(self, z, base_row, base_col, shift):
        """Declare the lifted-base-graph structure (enables the index-free QC kernel); returns False if rejected."""
        r, c, s = _i32(base_row), _i32(base_col), _i32(shift)
        return lib().sb_ldpc_graph_set_qc(self.handle, int(z), len(r), ptr(r), ptr(c), ptr(s)) == 0

    def is_qc(self):
        return bool(lib().sb_ldpc_graph_is_qc(self.handle))

    def qc_opening(self):
        return bool(lib().sb_ldpc_graph_qc_opening(self.handle))

    def workspace(self, device):
        need = lib().sb_ldpc_workspace_bytes(self.handle)
        if need == 0:
            return None, 0
        if self._ws is None or self._ws.numel() < need or self._ws.device != device:
            self._ws = torch.empty(need, dtype=torch.uint8, device=device)
        return self._ws, need

    def export(self):
        dims = np.zeros(10, np.int32)
        check(lib().sb_ldpc_graph_export(self.handle, ptr(dims), None, None, None, None, None, None), "export")
        c, n, e, lc, lv = (int(x) for x in dims[:5])
        out = {"dims": dims, "cn_order": np.zeros(c, np.int32), "vn_order": np.zeros(n, np.int32),
               "slot_of_edge": np.zeros(e, np.int32), "vn_slot": np.zeros(e, np.int32),
               "cn_off": np.zeros(lc + 1, np.int32), "vn_off": np.zeros(lv + 1, np.int32)}
        check(lib().sb_ldpc_graph_export(self.handle, ptr(dims), ptr(out["cn_order"]), ptr(out["vn_order"]),
                                         ptr(out["slot_of_edge"]), ptr(out["vn_slot"]), ptr(out["cn_off"]),
                                         ptr(out["vn_off"])), "export")
        return out


class LDPCBPDecoder(Block):
    # pylint: disable=line-too-long
    r"""LDPCBPDecoder(pcm, cn_update="boxplus-phi", vn_update="sum", cn_schedule="flooding", hard_out=True, num_iter=20, llr_max=20., v2c_callbacks=None, c2v_callbacks=None, return_state=False, precision=None)

    Iterative belief-propagation decoder for arbitrary binary parity-check matrices
    (reference: decoding.py:13-637). Inputs are logits ``log p(x=1)/p(x=0)`` of shape ``[..., n]``; the output is
    the hard-decided codeword (``hard_out``) or soft logits, plus the ``[num_edges, batch]`` VN->CN message
    state when ``return_state`` is set. ``cn_update`` is one of ``"boxplus-phi"`` (default), ``"boxplus"``,
    ``"minsum"`` / ``"min"``, ``"offset-minsum"``, ``"identity"``; ``vn_update`` one of ``"sum"``, ``"identity"``.

    ``cn_update`` / ``vn_update`` may also be callables on ragged messages and ``v2c_callbacks`` / ``c2v_callbacks``
    lists of callables (decoding.py:79-126; `sionna_b200.phy.fec.ldpc.utils.RaggedMessages` plays the role of the
    ragged tensor): such decoders run the unfused path - one kernel launch per half-iteration on ``[num_edges, batch]``
    tensors in the reference's layouts and list orders - instead of the fused shared-memory kernels.

    Extension (keyword ``early_stop=True``, not in the reference, 5G / quasi-cyclic codes only): every codeword stops
    as soon as its hard decisions satisfy all parity checks instead of always running ``num_iter`` iterations
    (decoding.py:105-107); ``decoder.num_iter_run`` then holds the iterations each codeword of the last call ran, and
    its output equals a fixed ``num_iter_run``-iteration decode bit for bit. Off by default.

    Extension (keyword ``sum_order``, not in the reference): ``"ascending"`` (default) combines the messages of a node
    in ascending neighbour index, which the quasi-cyclic fast path needs; ``"reference"`` walks them in the reference's
    own list orders (``np.argsort`` results of decoding.py:286, 329) on the generic kernel. fp32 sums depend on their
    order; for codewords that do not converge BP amplifies the last-bit difference, so only ``"reference"`` reproduces
    the reference's arithmetic bit for bit (for the rules without transcendental functions).
    """

    def __init__(self, pcm, cn_update="boxplus-phi", vn_update="sum", cn_schedule="flooding", hard_out=True,
                 num_iter=20, llr_max=20., v2c_callbacks=None, c2v_callbacks=None, return_state=False,
                 precision=None, **kwargs):
        if "cn_type" in kwargs:
            raise TypeError("'cn_type' is deprecated; use 'cn_update' instead.")
        self._early_stop = bool(kwargs.pop("early_stop", False))
        self.num_iter_run = None                            # [batch] int32: iterations per codeword of the last call
        sum_order = kwargs.pop("sum_order", "ascending")
        if sum_order not in ("ascending", "reference"):
            raise ValueError("sum_order must be 'ascending' or 'reference'.")
        self._sum_order = sum_order
        super().__init__(precision=precision, **kwargs)
        if not isinstance(hard_out, bool):
            raise TypeError("hard_out must be bool.")
        if not isinstance(num_iter, int):
            raise TypeError("num_iter must be int.")
        if num_iter < 0:
            raise ValueError("num_iter cannot be negative.")
        if not isinstance(return_state, bool):
            raise TypeError("return_state must be bool.")
        if isinstance(pcm, np.ndarray):
            if not np.array_equal(pcm, pcm.astype(bool)):
                raise ValueError("PC matrix must be binary.")
        elif isinstance(pcm, (sp.sparse.csr_matrix, sp.sparse.csc_matrix)):
            if not np.array_equal(pcm.data, pcm.data.astype(bool)):
                raise ValueError("PC matrix must be binary.")
        else:
            raise TypeError("Unsupported dtype of pcm.")
        if not isinstance(llr_max, (int, float)):
            raise TypeError("llr_max must be int or float.")

        self._pcm = pcm
        self._hard_out = hard_out
        self._num_iter = num_iter
        self._return_state = return_state
        self._num_cns, self._num_vns = pcm.shape[0], pcm.shape[1]
        self._llr_max = float(llr_max)

        # callbacks / callable node updates (decoding.py:79-126): honoured on the unfused path (one launch per
        # half-iteration, csrc/ldpc_bp_flat.cu); the fused kernels run when neither is given
        def _cb_list(name, cbs):
            if cbs is None:
                return []
            if isinstance(cbs, (list, tuple)):
                for c in cbs:
                    if not callable(c):
                        raise TypeError(f"{name} must be a list of callables.")
                return list(cbs)
            if callable(cbs):
                return [cbs]
            raise TypeError(f"{name} must be a list of callables.")
        self._v2c_callbacks = _cb_list("v2c_callbacks", v2c_callbacks)
        self._c2v_callbacks = _cb_list("c2v_callbacks", c2v_callbacks)

        schedule = None
        if isinstance(cn_schedule, str) and cn_schedule == "flooding":
            self._scheduling = "flooding"
            self._cn_schedule = np.arange(self._num_cns, dtype=np.int32)[None, :]
        elif isinstance(cn_schedule, (np.ndarray, torch.Tensor)):
            cs = np.asarray(cn_schedule.cpu() if isinstance(cn_schedule, torch.Tensor) else cn_schedule).astype(np.int32)
            self._scheduling = "custom"
            if cs.ndim != 2:
                raise ValueError("cn_schedule must be of rank 2.")
            if cs.max() >= self._num_cns:
                raise ValueError("cn_schedule can only contain values smaller number_cns.")
            if cs.min() < 0:
                raise ValueError("cn_schedule cannot contain negative values.")
            self._cn_schedule = cs
            schedule = cs
        else:
            raise ValueError("cn_schedule can be 'flooding' or an array of ints.")

        # edge list in the reference's VN order (decoding.py:277-292): same NumPy calls, same (unstable) argsort
        if isinstance(pcm, np.ndarray):
            pcm = sp.sparse.csr_matrix(pcm)
        self._cn_idx, self._vn_idx, _ = sp.sparse.find(pcm)
        idx = np.argsort(self._vn_idx)
        self._cn_idx = self._cn_idx[idx]
        self._vn_idx = self._vn_idx[idx]
        self._num_edges = len(self._vn_idx)

        self._cn_fn = self._vn_fn = None
        if isinstance(cn_update, str) and cn_update in _CN_RULES:
            self._cn_rule = _CN_RULES[cn_update]
        elif callable(cn_update):
            self._cn_rule, self._cn_fn = _CN_RULES["identity"], cn_update
        else:
            raise TypeError("Provided cn_update not supported.")
        if isinstance(vn_update, str) and vn_update in _VN_RULES:
            self._vn_rule = _VN_RULES[vn_update]
        elif callable(vn_update):
            self._vn_rule, self._vn_fn = _VN_RULES["identity"], vn_update
        else:
            raise TypeError("Provided vn_update not supported.")
        self._unfused = bool(self._v2c_callbacks or self._c2v_callbacks or self._cn_fn or self._vn_fn)
        self._flat = None                                   # device index tables of the unfused path (lazy)
        self._offset = 0.5  # default of cn_update_offset_minsum (decoding.py:755)

        in_map, n_in, out_vn, n_out = self._io_maps()
        cn_view = np.argsort(self._cn_idx) if sum_order == "reference" else None     # v2c_perm, decoding.py:329
        self._graph = _GraphHandle(self._num_cns, self._num_vns, self._cn_idx, self._vn_idx, in_map, n_in,
                                   out_vn, n_out, schedule, cn_view)

    def _io_maps(self):
        """Hook for subclasses folding rate matching into the kernel's load/store maps."""
        return None, 0, None, 0

    # ---- properties (decoding.py:351-410) -------------------------------------------------------------
    @property
    def pcm(self):
        return self._pcm

    @property
    def num_cns(self):
        return self._num_cns

    @property
    def num_vns(self):
        return self._num_vns

    @property
    def n(self):
        return self._num_vns

    @property
    def coderate(self):
        return (self._num_vns - self._num_cns) / self._num_vns

    @property
    def num_edges(self):
        return self._num_edges

    @property
    def num_iter(self):
        return self._num_iter

    @num_iter.setter
    def num_iter(self, num_iter):
        if not isinstance(num_iter, int):
            raise TypeError("num_iter must be int.")
        if num_iter < 0:
            raise ValueError("num_iter cannot be negative.")
        self._num_iter = num_iter

    @property
    def llr_max(self):
        return self._llr_max

    @llr_max.setter
    def llr_max(self, value):
        if value < 0:
            raise ValueError("llr_max cannot be negative.")
        self._llr_max = float(value)

    @property
    def return_state(self):
        return self._return_state

    @property
    def on_chip(self):
        """True if the decoding graph runs on the shared-memory-resident path."""
        return self._graph.on_chip()

    # ---- Block protocol -----------------------------------------------------------------------------
    def build(self, input_shape, **kwargs):
        assert input_shape[-1] == self._num_vns, "Last dimension must be of length n."

    # ---- unfused path: callbacks / callable node updates ------------------------------------------------------
    def _flat_tables(self, dev):
        """Index tensors of the reference's message layouts (decoding.py:277-345) on `dev`."""
        if self._flat is not None and self._flat["dev"] == dev:
            return self._flat
        e, n, c = self._num_edges, self._num_vns, self._num_cns
        v2c_perm = np.argsort(self._cn_idx)                               # :329 CN view: position j <- edge v2c_perm[j]
        c2v_perm = np.argsort(v2c_perm)                                   # :336 edge e -> its CN-view position
        vn_ptr = np.zeros(n + 1, np.int64)
        np.cumsum(np.bincount(self._vn_idx, minlength=n), out=vn_ptr[1:])
        cn_ptr = np.zeros(c + 1, np.int64)
        np.cumsum(np.bincount(self._cn_idx, minlength=c), out=cn_ptr[1:])
        _, _, out_vn, n_out = self._io_maps()
        out_vn = np.arange(n) if out_vn is None else np.asarray(out_vn)

        def t32(a):
            return torch.from_numpy(np.ascontiguousarray(a, np.int32)).to(dev)
        f = {"dev": dev, "v2c_perm": t32(v2c_perm), "c2v_perm": t32(c2v_perm), "vn_ptr": t32(vn_ptr), "cn_ptr": t32(cn_ptr),
             "vn_of_edge": t32(self._vn_idx), "out_vn": t32(out_vn), "n_out": int(len(out_vn)),
             "vn_splits": torch.from_numpy(vn_ptr).to(dev), "cn_splits": torch.from_numpy(cn_ptr).to(dev),
             "v2c_perm64": torch.from_numpy(v2c_perm.astype(np.int64)).to(dev),
             "c2v_perm64": torch.from_numpy(c2v_perm.astype(np.int64)).to(dev)}
        if self._scheduling != "flooding":
            subs = []
            for row in self._cn_schedule:                                  # active CNs of every sub-iteration
                pos = np.concatenate([np.arange(cn_ptr[cn], cn_ptr[cn + 1]) for cn in row]) if len(row) else np.zeros(0, np.int64)
                lens = np.array([cn_ptr[cn + 1] - cn_ptr[cn] for cn in row], np.int64)
                splits = np.concatenate([[0], np.cumsum(lens)])
                subs.append({"cns": t32(row), "pos": torch.from_numpy(pos.astype(np.int64)).to(dev),
                             "splits": torch.from_numpy(splits).to(dev)})
            f["subs"] = subs
        # rate recovery + clipping through a 0-iteration launch of the fused kernel with an identity output map
        in_map, n_in, _, _ = self._io_maps()
        f["rr_graph"] = self._graph if in_map is None else _GraphHandle(c, n, self._cn_idx, self._vn_idx, in_map, n_in)
        self._flat = f
        return f

    def _decode_unfused(self, llr2d, num_iter, msg_v2c):
        from .utils import RaggedMessages
        L = lib()
        dev, b = llr2d.device, llr2d.shape[0]
        f = self._flat_tables(dev)
        e, n, c = self._num_edges, self._num_vns, self._num_cns
        st = current_stream()
        # [B, N] clipped channel logits incl. punctured / filler positions (decoding.py:552-554, 1444-1475)
        g = f["rr_graph"]
        x0 = torch.empty((b, n), dtype=torch.float32, device=dev)
        ws, ws_bytes = g.workspace(dev)
        check(L.sb_ldpc_decode(g.handle, ptr(llr2d), b, 0, self._cn_rule, self._vn_rule, self._offset, self._llr_max, 0,
                               None, None, ptr(x0), ptr(ws), ws_bytes, st), "sb_ldpc_decode (rate recovery)")
        st_in = None
        if msg_v2c is not None:
            st_in = torch.as_tensor(msg_v2c).to(device=dev, dtype=torch.float32).contiguous()
            if tuple(st_in.shape) != (e, b):
                raise ValueError("msg_v2c must have shape [num_edges, batch_size].")
        llr = torch.empty((n, b), dtype=torch.float32, device=dev)
        v2c = torch.empty((e, b), dtype=torch.float32, device=dev)
        c2v = torch.zeros((e, b), dtype=torch.float32, device=dev)                                  # :581
        xhat = llr                                                                                  # :607 (0 iterations)
        check(L.sb_ldpc_flat_init(ptr(x0), ptr(f["vn_of_edge"]), ptr(st_in), ptr(llr), ptr(v2c), b, n, e, st),
              "sb_ldpc_flat_init")
        xbuf = torch.empty((n, b), dtype=torch.float32, device=dev)
        subs = f.get("subs") or [None]
        for it in range(int(num_iter)):
            for sub in subs:
                # ---- CN update of the active nodes (:479-483) ---------------------------------------------------
                if self._cn_fn is not None:
                    msg_in = v2c.index_select(0, f["v2c_perm64"] if sub is None else f["v2c_perm64"].index_select(0, sub["pos"]))
                    rag = RaggedMessages(msg_in, f["cn_splits"] if sub is None else sub["splits"])
                    rag = self._cn_fn(rag, self._llr_max)
                else:
                    check(L.sb_ldpc_flat_cn(ptr(v2c), ptr(c2v), ptr(f["cn_ptr"]), ptr(f["v2c_perm"]),
                                            None if sub is None else ptr(sub["cns"]),
                                            c if sub is None else int(sub["cns"].numel()), b, self._cn_rule, self._offset,
                                            self._llr_max, st), "sb_ldpc_flat_cn")
                    rag = None
                    if self._c2v_callbacks:
                        rag = RaggedMessages(c2v if sub is None else c2v.index_select(0, sub["pos"]),
                                             f["cn_splits"] if sub is None else sub["splits"])
                for cb in self._c2v_callbacks:                                                      # :484-486
                    rag = cb(rag, it)
                if rag is not None:
                    vals = rag.flat_values.to(torch.float32)
                    if sub is None:
                        c2v = vals.contiguous()                                                     # :500
                    else:
                        c2v.index_copy_(0, sub["pos"], vals)                                        # :489-497
                # ---- full VN update (:506-511) -------------------------------------------------------------------
                if self._vn_fn is not None:
                    rag_v = RaggedMessages(c2v.index_select(0, f["c2v_perm64"]), f["vn_splits"])
                    rag_v, xhat = self._vn_fn(rag_v, llr, self._llr_max)
                    v2c = rag_v.flat_values.to(torch.float32).contiguous()
                    xhat = xhat.to(torch.float32).contiguous()
                else:
                    check(L.sb_ldpc_flat_vn(ptr(c2v), ptr(llr), ptr(f["vn_ptr"]), ptr(f["c2v_perm"]), ptr(v2c), ptr(xbuf),
                                            n, b, self._vn_rule, self._llr_max, st), "sb_ldpc_flat_vn")
                    xhat = xbuf
                if self._v2c_callbacks:                                                             # :513-515
                    rag_v = RaggedMessages(v2c, f["vn_splits"])
                    for cb in self._v2c_callbacks:
                        rag_v = cb(rag_v, it + 1, xhat)
                    v2c = rag_v.flat_values.to(torch.float32).contiguous()
        out = torch.empty((b, f["n_out"]), dtype=torch.float32, device=dev)
        st_out = torch.empty((e, b), dtype=torch.float32, device=dev) if self._return_state else None
        check(L.sb_ldpc_flat_out(ptr(xhat), ptr(f["out_vn"]), ptr(out), ptr(v2c), ptr(st_out), b, f["n_out"], e,
                                 int(self._hard_out), st), "sb_ldpc_flat_out")
        return out, st_out

    def _decode_early(self, llr2d, num_iter, msg_v2c):
        """``early_stop=True``: at most ``num_iter`` iterations, every codeword stops once its hard decisions form a
        codeword (``sb_ldpc_decode_early``); ``self.num_iter_run`` holds the iterations each codeword ran."""
        if msg_v2c is not None or self._return_state:
            raise ValueError("early_stop cannot be combined with a decoder state (msg_v2c / return_state)")
        if self._vn_rule != _VN_RULES["sum"] or self._cn_rule == _CN_RULES["identity"]:
            raise ValueError("early_stop needs a check-node rule and the 'sum' variable-node rule")
        g, dev, b = self._graph, llr2d.device, llr2d.shape[0]
        out = torch.empty((b, g.n_out), dtype=torch.float32, device=dev)
        self.num_iter_run = torch.empty(b, dtype=torch.int32, device=dev)
        check(lib().sb_ldpc_decode_early(g.handle, ptr(llr2d), b, int(num_iter), self._cn_rule, self._offset, self._llr_max,
                                         int(self._hard_out), ptr(out), ptr(self.num_iter_run), current_stream()),
              "sb_ldpc_decode_early")
        return out, None

    def _decode(self, llr2d, num_iter, msg_v2c):
        if self.precision != "single":
            raise NotImplementedError("sb_ldpc_decode is an fp32 kernel; precision='double' is not available.")
        if self._unfused:
            return self._decode_unfused(llr2d, num_iter, msg_v2c)
        if self._early_stop:
            return self._decode_early(llr2d, num_iter, msg_v2c)
        g = self._graph
        dev = llr2d.device
        b = llr2d.shape[0]
        out = torch.empty((b, g.n_out), dtype=torch.float32, device=dev)
        st_in = st_out = None
        if msg_v2c is not None:
            msg_v2c = torch.as_tensor(msg_v2c).to(device=dev, dtype=torch.float32)
            if tuple(msg_v2c.shape) != (self._num_edges, b):
                raise ValueError("msg_v2c must have shape [num_edges, batch_size].")
            st_in = msg_v2c.t().contiguous()
        if self._return_state:
            st_out = torch.empty((b, self._num_edges), dtype=torch.float32, device=dev)
        ws, ws_bytes = g.workspace(dev)
        check(lib().sb_ldpc_decode(g.handle, ptr(llr2d), b, int(num_iter), self._cn_rule, self._vn_rule,
                                   self._offset, self._llr_max, int(self._hard_out), ptr(st_in), ptr(st_out),
                                   ptr(out), ptr(ws), ws_bytes, current_stream()), "sb_ldpc_decode")
        return out, (st_out.t().contiguous() if st_out is not None else None)

    def call(self, llr_ch, /, *, num_iter=None, msg_v2c=None):
        if num_iter is None:
            num_iter = self._num_iter
        shape = list(llr_ch.shape)
        llr2d = llr_ch.reshape(-1, self._num_vns).contiguous()
        x, st = self._decode(llr2d, num_iter, msg_v2c)
        x = x.reshape(shape[:-1] + [x.shape[-1]])
        if not self._return_state:
            return x
        return x, st


class LDPC5GDecoder(LDPCBPDecoder):
    # pylint: disable=line-too-long
    r"""LDPC5GDecoder(encoder, cn_update="boxplus-phi", vn_update="sum", cn_schedule="flooding", hard_out=True, return_infobits=True, num_iter=20, llr_max=20., v2c_callbacks=None, c2v_callbacks=None, prune_pcm=True, return_state=False, precision=None)

    BP decoder for 5G NR LDPC codes including rate recovery (reference: decoding.py:1169-1536): takes ``[..., n]``
    logits of the rate-matched codeword and returns the ``k`` information bits (``return_infobits``) or all ``n``
    codeword positions. ``prune_pcm`` removes the trailing punctured degree-1 VNs and their CNs (:1344-1378);
    ``cn_schedule="layered"`` updates groups of Z check nodes sequentially (:1384-1390).
    """

    def __init__(self, encoder, cn_update="boxplus-phi", vn_update="sum", cn_schedule="flooding", hard_out=True,
                 return_infobits=True, num_iter=20, llr_max=20., v2c_callbacks=None, c2v_callbacks=None,
                 prune_pcm=True, return_state=False, precision=None, **kwargs):
        if not isinstance(encoder, LDPC5GEncoder):
            raise TypeError("encoder must be of class LDPC5GEncoder.")
        self._encoder = encoder
        pcm = encoder.pcm
        if not isinstance(return_infobits, bool):
            raise TypeError("return_info must be bool.")
        self._return_infobits = return_infobits
        if not isinstance(return_state, bool):
            raise TypeError("return_state must be bool.")
        if "cn_type" in kwargs:
            raise TypeError("'cn_type' is deprecated; use 'cn_update' instead.")
        if not isinstance(prune_pcm, bool):
            raise TypeError("prune_pcm must be bool.")
        self._prune_pcm = prune_pcm
        k_filler = encoder.k_ldpc - encoder.k
        nb_punc_bits = (encoder.n_ldpc - k_filler) - encoder.n - 2 * encoder.z
        if prune_pcm:
            # first index of the trailing run of degree-1 columns (decoding.py:1346-1352)
            dv = np.asarray(pcm.sum(axis=0)).ravel()
            last_pos = encoder.n_ldpc
            for idx in range(encoder.n_ldpc - 1, 0, -1):
                if dv[idx] == 1:
                    last_pos = idx
                else:
                    break
            if isinstance(cn_schedule, str) and cn_schedule == "layered":
                nb_punc_bits = int(np.floor(nb_punc_bits / encoder.z) * encoder.z)
            self._n_pruned = int(max(last_pos, encoder.n_ldpc - nb_punc_bits))
            self._nb_pruned_nodes = encoder.n_ldpc - self._n_pruned
            if self._nb_pruned_nodes < 0:
                raise ArithmeticError("Internal error: number of pruned nodes must be positive.")
            if self._nb_pruned_nodes > 0:
                pcm = pcm[:-self._nb_pruned_nodes, :-self._nb_pruned_nodes]
        else:
            self._nb_pruned_nodes = 0
            self._n_pruned = encoder.n_ldpc
        if isinstance(cn_schedule, str) and cn_schedule == "layered":
            z = encoder.z
            num_blocks = int(pcm.shape[0] / z)
            cn_schedule = np.stack([np.arange(z) + i * z for i in range(num_blocks)], axis=0)
        super().__init__(sp.sparse.csr_matrix(pcm), cn_update=cn_update, vn_update=vn_update,
                         cn_schedule=cn_schedule, hard_out=hard_out, num_iter=num_iter, llr_max=llr_max,
                         v2c_callbacks=v2c_callbacks, c2v_callbacks=c2v_callbacks, return_state=return_state,
                         precision=precision, **kwargs)
        # the decoding graph is a (possibly truncated) lifted base graph: let the C side use its QC fast path
        if os.environ.get("SB_LDPC_DISABLE_QC", "0") != "1" and self._sum_order == "ascending":
            br, bc = np.nonzero(encoder._bm >= 0)
            self._graph.set_qc(encoder.z, br, bc, encoder._bm[br, bc] % encoder.z)

    @property
    def encoder(self):
        return self._encoder

    def _io_maps(self):
        """Fold decoding.py:1436-1475 (input) and :1486-1536 (output) into gather maps over the pruned VNs."""
        enc = self._encoder
        k, k_ldpc, z, n = enc.k, enc.k_ldpc, enc.z, enc.n
        k_filler = k_ldpc - k
        v = np.arange(self._n_pruned)
        q = np.where(v < k, v, v - k_filler)                  # position in [0(2Z) | llr(n) | 0(punct)]
        i = q - 2 * z                                         # position in the (de-interleaved) received word
        src = i if enc.out_int_inv is None else np.asarray(enc.out_int_inv)[np.clip(i, 0, n - 1)]
        in_map = np.where((i >= 0) & (i < n), src, -1)
        in_map = np.where((v >= k) & (v < k_ldpc), -2, in_map).astype(np.int32)
        if self._return_infobits:
            out_vn = np.arange(k, dtype=np.int32)
        else:
            out_vn = enc._tx_vn()
        return in_map, n, out_vn, len(out_vn)

    def build(self, input_shape, **kwargs):
        if input_shape[-1] != self.encoder.n:
            raise ValueError("Last dimension must be of length n.")
        self._old_shape_5g = input_shape

    def call(self, llr_ch, /, *, num_iter=None, msg_v2c=None):
        if num_iter is None:
            num_iter = self._num_iter
        shape = list(llr_ch.shape)
        llr2d = llr_ch.reshape(-1, self.encoder.n).contiguous()
        x, st = self._decode(llr2d, num_iter, msg_v2c)
        x = x.reshape(shape[:-1] + [x.shape[-1]])
        if self._return_state:
            return x, st
        return x
