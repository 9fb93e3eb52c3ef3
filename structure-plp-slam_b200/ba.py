"""ctypes binding of the local bundle adjuster (plp_ba_* / plp_local_ba).  Marshalling only."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .capi import Context, PlpError, _P  # noqa: F401


class BaProblem(C.Structure):
    _fields_ = [("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("focal_x_baseline", C.c_double), ("setup_type", C.c_int32),
                ("n_kf", C.c_int32), ("kf_pose_cw", _P), ("kf_fixed", _P),
                ("n_pts", C.c_int32), ("pt_pos_w", _P),
                ("n_pt_edges", C.c_int32), ("pt_edge_kf", _P), ("pt_edge_lm", _P), ("pt_edge_obs", _P),
                ("pt_edge_inv_sigma_sq", _P),
                ("n_lines", C.c_int32), ("line_plucker", _P),
                ("n_line_edges", C.c_int32), ("line_edge_kf", _P), ("line_edge_lm", _P), ("line_edge_obs", _P),
                ("line_edge_inv_sigma_sq", _P),
                ("n_plane_edges", C.c_int32), ("plane_edge_lm", _P), ("plane_edge_fn", _P)]


class BaCfg(C.Structure):
    _fields_ = [("num_first_iter", C.c_int32), ("num_second_iter", C.c_int32), ("num_ctas", C.c_int32)]


class BaResult(C.Structure):
    _fields_ = [("kf_pose_cw", _P), ("pt_pos_w", _P), ("line_plucker", _P), ("pt_edge_outlier", _P),
                ("line_edge_outlier", _P), ("iters_first", C.c_int32), ("iters_second", C.c_int32),
                ("lm_tries", C.c_int32), ("final_chi2", C.c_double)]


class BaComm:
    """NCCL communicator for landmark-sharded BA (one per rank)."""

    def __init__(self, ctx: Context, unique_id: bytes, world: int, rank: int):
        self._ctx, self._lib = ctx, ctx._lib
        h = C.c_void_p()
        buf = (C.c_uint8 * 128).from_buffer_copy(unique_id)
        ctx._check(self._lib.plp_ba_comm_init(ctx.handle, buf, C.c_int(world), C.c_int(rank), C.byref(h)))
        self.handle, self.world, self.rank = h, world, rank

    @staticmethod
    def unique_id(ctx: Context) -> bytes:
        buf = (C.c_uint8 * 128)()
        ctx._check(ctx._lib.plp_ba_comm_unique_id(buf))
        return bytes(buf)

    def allreduce_count(self) -> int:
        self._lib.plp_ba_comm_allreduce_count.restype = C.c_uint64
        return int(self._lib.plp_ba_comm_allreduce_count(self.handle))

    def peer_active(self) -> bool:
        """True if the small all-reduces run as the one-shot kernel over NVLink peer memory instead of ncclAllReduce."""
        return bool(self._lib.plp_ba_comm_peer_active(self.handle))

    def peer_count(self) -> int:
        self._lib.plp_ba_comm_peer_count.restype = C.c_uint64
        return int(self._lib.plp_ba_comm_peer_count(self.handle))

    def close(self):
        if self.handle is not None:
            self._lib.plp_ba_comm_destroy(self.handle)
            self.handle = None


class LocalBA:
    """optimize::local_bundle_adjuster[_extended_line|_extended_plane] on one GPU (or one shard of it)."""

    def __init__(self, ctx: Context, problem_struct, n_sizes, num_first_iter=5, num_second_iter=10, num_ctas=0,
                 comm: BaComm | None = None):
        """problem_struct: a ctypes struct with the plp_ba_problem layout (kept alive by the caller);
        n_sizes = (n_kf, n_pts, n_lines, n_pt_edges, n_line_edges)."""
        self._ctx, self._lib = ctx, ctx._lib
        self.sizes = n_sizes
        cfg = BaCfg(num_first_iter, num_second_iter, num_ctas)
        h = C.c_void_p()
        self._h = None
        ctx._check(self._lib.plp_ba_create(ctx.handle, C.byref(problem_struct), C.byref(cfg),
                                           comm.handle if comm else None, C.byref(h)))
        self._h = h

    def solve(self, force_stop=None):
        n_kf, n_pts, n_lines, n_pe, n_le = self.sizes
        out = dict(kf_pose_cw=np.zeros((n_kf, 4, 4)), pt_pos_w=np.zeros((max(n_pts, 1), 3)),
                   line_plucker=np.zeros((max(n_lines, 1), 6)), pt_edge_outlier=np.zeros(max(n_pe, 1), np.uint8),
                   line_edge_outlier=np.zeros(max(n_le, 1), np.uint8))
        r = BaResult(*[out[k].ctypes.data_as(_P) for k in ("kf_pose_cw", "pt_pos_w", "line_plucker", "pt_edge_outlier",
                                                           "line_edge_outlier")], 0, 0, 0, 0.0)
        fs = None if force_stop is None else force_stop.ctypes.data_as(_P)
        self._ctx._check(self._lib.plp_ba_solve(self._h, fs, C.byref(r)))
        out["pt_pos_w"] = out["pt_pos_w"][:n_pts]
        out["line_plucker"] = out["line_plucker"][:n_lines]
        out["pt_edge_outlier"] = out["pt_edge_outlier"][:n_pe]
        out["line_edge_outlier"] = out["line_edge_outlier"][:n_le]
        out.update(iters_first=r.iters_first, iters_second=r.iters_second, lm_tries=r.lm_tries, final_chi2=r.final_chi2)
        return out

    def bench_tries(self, tries: int):
        it, tr = C.c_int32(0), C.c_int32(0)
        self._ctx._check(self._lib.plp_ba_bench_tries(self._h, C.c_int(tries), C.byref(it), C.byref(tr)))
        return it.value, tr.value

    def debug_try(self, n_free: int):
        """plp_ba_debug_try: (S upper blocks [n_pairs, 6, 6], g, bp, chi2, dp, lambda) of the first real LM try."""
        n_pairs = n_free * (n_free + 1) // 2
        packed, dp, lam = np.zeros(n_pairs * 36 + 12 * n_free + 1), np.zeros(6 * n_free), C.c_double(0.0)
        self._ctx._check(self._lib.plp_ba_debug_try(self._h, packed.ctypes.data_as(_P), dp.ctypes.data_as(_P), C.byref(lam)))
        nS = n_pairs * 36
        return dict(S=packed[:nS].reshape(n_pairs, 6, 6), g=packed[nS:nS + 6 * n_free],
                    bp=packed[nS + 6 * n_free:nS + 12 * n_free], chi2=float(packed[-1]), dp=dp, lam=lam.value, packed=packed)

    def close(self):
        if self._h is not None:
            self._lib.plp_ba_destroy(self._h)
            self._h = None


def shard_boundaries(edges_per_landmark, world: int):
    """Contiguous landmark blocks balanced by edge count (SURVEY.md section 8(e)): returns world+1 boundaries."""
    w = np.asarray(edges_per_landmark, np.int64) + 1
    cum = np.concatenate([[0], np.cumsum(w)])
    bounds = [0]
    for r in range(1, world):
        bounds.append(int(np.searchsorted(cum, cum[-1] * r / world)))
    bounds.append(len(w))
    return [min(max(b, 0), len(w)) for b in bounds]


def shard_edges(edge_lm, lm_begin: int, lm_end: int):
    """Indices of the (landmark-sorted) edges owned by the landmark block [lm_begin, lm_end) and their local
    landmark indices."""
    edge_lm = np.asarray(edge_lm)
    sel = np.nonzero((edge_lm >= lm_begin) & (edge_lm < lm_end))[0]
    return sel, (edge_lm[sel] - lm_begin).astype(np.int32)


def global_ba(ctx: Context, problem_struct, n_sizes, num_iter=20, use_huber_kernel=True, force_stop=None):
    """optimize::global_bundle_adjuster::optimize (global_bundle_adjuster.cc:64-253) through plp_global_ba."""
    n_kf, n_pts, n_lines, n_pe, n_le = n_sizes
    out = dict(kf_pose_cw=np.zeros((n_kf, 4, 4)), pt_pos_w=np.zeros((max(n_pts, 1), 3)),
               line_plucker=np.zeros((max(n_lines, 1), 6)), pt_edge_outlier=np.zeros(max(n_pe, 1), np.uint8),
               line_edge_outlier=np.zeros(max(n_le, 1), np.uint8))
    r = BaResult(*[out[k].ctypes.data_as(_P) for k in ("kf_pose_cw", "pt_pos_w", "line_plucker", "pt_edge_outlier",
                                                       "line_edge_outlier")], 0, 0, 0, 0.0)
    fs = None if force_stop is None else force_stop.ctypes.data_as(_P)
    ctx._check(ctx._lib.plp_global_ba(ctx.handle, C.byref(problem_struct), C.c_int(num_iter),
                                      C.c_int(1 if use_huber_kernel else 0), fs, C.byref(r)))
    out["pt_pos_w"] = out["pt_pos_w"][:n_pts]
    out["line_plucker"] = out["line_plucker"][:n_lines]
    out.update(iters_first=r.iters_first, lm_tries=r.lm_tries, final_chi2=r.final_chi2)
    return out
