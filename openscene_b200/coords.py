"""Host side of the coordinate manager: owns the per-tensor-stride coordinate sets, their hash
tables and the kernel-map cache, all built by ``libosb200`` (csrc/coords.cu).

Mirrors what MinkowskiEngine's CoordinateManager does for the reference (SURVEY.md 8a a4-a6):
one forward of MinkUNet builds the stride-1 set, four coarser sets and 10 kernel maps, each once.
"""
import ctypes
import os

import torch

from . import _cabi as C


def _next_pow2(n):
    p = 1
    while p < n:
        p <<= 1
    return p


def _deinterleave(key, axis):
    """Bits axis, axis+3, ... of the low 54 key bits -> one 18-bit field (inverse of the Morton interleave)."""
    v = 0
    for i in range(18):
        v |= ((key >> (3 * i + axis)) & 1) << i
    return v


def occgrid_enabled():
    return os.environ.get('OSB_OCCGRID', '1') != '0'


class CoordSet:
    """One coordinate set (internal Morton order) + its lazily built neighbour-lookup structure: an occupancy grid
    (csrc/common.cuh) when the set is non-negative and small enough, the hash table otherwise."""
    __slots__ = ('coords', 'n', 'slots', 'cap', 'ts', 'grid', 'grid_args', '_grid_plan', '_status')

    def __init__(self, coords, ts, grid_plan=None, status=None):
        self.coords, self.n, self.ts = coords, coords.shape[0], ts
        self.slots, self.cap = None, 0
        self.grid, self.grid_args = None, None
        self._grid_plan, self._status = grid_plan, status      # (log2_ts, nbits, n_batch) or None

    def ensure_lookup(self):
        """Build (once) whichever structure serves this set; returns self."""
        if self._grid_plan is None:
            return self.ensure_hash()
        if self.grid is None:
            log2_ts, nbits, n_batch = self._grid_plan
            nbytes = C.lib().osb_occgrid_bytes(nbits, n_batch)
            self.grid = torch.empty(nbytes, dtype=torch.uint8, device=self.coords.device)
            C.call('osb_occgrid_build', C.ptr(self.coords), self.n, log2_ts, nbits, n_batch, C.ptr(self.grid), C.ptr(self._status),
                   C.stream_ptr())
            self.grid_args = (log2_ts, nbits, n_batch)
        return self

    def ensure_hash(self):
        if self.slots is None:
            self.cap = _next_pow2(max(4 * self.n, 16))      # load factor <= 0.25: short probe chains (the longest of 32 lanes gates a warp)
            self.slots = torch.empty(self.cap * 16, dtype=torch.uint8, device=self.coords.device)
            C.call('osb_hash_build', C.ptr(self.coords), self.n, C.ptr(self.slots), self.cap, C.stream_ptr())
        return self


class KernelMap:
    """Output-stationary map: nbr[k, o] = input row feeding output row o through offset k (-1: none)."""
    __slots__ = ('nbr', 'K', 'n_in', 'n_out', 'pairs_per_k', '_t')

    def __init__(self, nbr, K, n_in, n_out, pairs_per_k=None):
        self.nbr, self.K, self.n_in, self.n_out, self.pairs_per_k = nbr, K, n_in, n_out, pairs_per_k
        self._t = None

    def transposed(self):
        """Map with input/output roles swapped (transposed conv forward, conv dgrad)."""
        if self._t is None:
            nbr_t = torch.empty((self.K, self.n_in), dtype=torch.int32, device=self.nbr.device)
            C.call('osb_kernel_map_transpose', C.ptr(self.nbr), self.n_out, self.K, C.ptr(nbr_t), self.n_in,
                   C.stream_ptr())
            # no back-reference from the transposed map: a reference cycle would keep both device buffers alive until the
            # cyclic garbage collector runs (never, inside a gc-disabled serving / benchmark loop)
            self._t = KernelMap(nbr_t, self.K, self.n_out, self.n_in)
        return self._t

    def num_pairs(self):
        if self.pairs_per_k is None:
            return int((self.nbr >= 0).sum().item())
        return int(self.pairs_per_k.sum().item())


class CoordinateManager:
    def __init__(self, coordinates, pyramid_levels=0):
        """coordinates: int32 CUDA tensor [N,4] = (batch, x, y, z), unique rows, caller order.
        pyramid_levels > 0 builds the tensor-stride 2, 4, ... sets in the same native call (one host sync for the
        whole encoder pyramid instead of two per level)."""
        C.require_cuda(coordinates, 'coordinates')
        coords = coordinates.to(torch.int32).contiguous()
        assert coords.dim() == 2 and coords.shape[1] == 4, "coordinates must be [N,4] (batch,x,y,z)"
        n = coords.shape[0]
        if n == 0:
            raise RuntimeError("openscene_b200: empty coordinate set")
        dev = coords.device
        self.device = dev
        with torch.cuda.device(dev):
            coords_int = torch.empty_like(coords)
            self.perm = torch.empty(n, dtype=torch.int32, device=dev)
            self.inv_perm = torch.empty(n, dtype=torch.int32, device=dev)
            cs = CoordSet(coords_int, 1)
            use_grid = occgrid_enabled()
            if not use_grid:                                   # with the grid the level-0 hash is built only if it turns out to be needed
                cs.cap = _next_pow2(max(4 * n, 16))
                cs.slots = torch.empty(cs.cap * 16, dtype=torch.uint8, device=dev)
            ws_bytes = C.lib().osb_coordset_workspace_bytes(n)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            status = (ctypes.c_int32 * 6)(0, 0, 0, 0, 0, 0)
            pyr = None
            if pyramid_levels > 0:
                L = pyramid_levels
                lvl = torch.empty((L, n, 4), dtype=torch.int32, device=dev)
                par = torch.empty((L, n), dtype=torch.int32, device=dev)
                counts = (ctypes.c_int64 * (L + 1))()
                C.call('osb_coordset_pyramid', C.ptr(coords), n, L, C.ptr(coords_int), C.ptr(self.perm), C.ptr(self.inv_perm),
                       C.ptr(cs.slots), cs.cap, C.ptr(lvl), C.ptr(par), counts, status, C.ptr(ws), ws_bytes, C.stream_ptr())
                pyr = (lvl, par, list(counts))
            else:
                C.call('osb_coordset_build', C.ptr(coords), n, C.ptr(coords_int), C.ptr(self.perm), C.ptr(self.inv_perm),
                       C.ptr(cs.slots), cs.cap, status, C.ptr(ws), ws_bytes, C.stream_ptr())
        if status[0] & 1:
            raise RuntimeError("openscene_b200: coordinate out of range (need 0 <= batch < 1024, |x|,|y|,|z| < 2^17-256)")
        if status[0] & 2:
            raise RuntimeError("openscene_b200: duplicate coordinates in SparseTensor input; the reference's loaders "
                               "always voxelise first (dataset/voxelizer.py:128), so rows are unique per scene")
        # occupancy-grid plan from the OR / AND of the Morton keys (status[2..5]): all coordinates non-negative (bit 17 of
        # every biased field set in the AND), nbits0 = bit length of the largest coordinate, batch bound = OR of the batch ids
        self._grid0 = None
        self.grid_status = None
        if use_grid:
            k_or = (status[2] & 0xffffffff) | ((status[3] & 0xffffffff) << 32)
            k_and = (status[4] & 0xffffffff) | ((status[5] & 0xffffffff) << 32)
            nonneg = all((_deinterleave(k_and, a) >> 17) & 1 for a in range(3))
            if nonneg:
                nbits0 = max(_deinterleave(k_or, a) & 0x1ffff for a in range(3)).bit_length()
                self._grid0 = (nbits0, int(k_or >> 54) + 1)
                self.grid_status = torch.zeros(1, dtype=torch.int32, device=dev)
        cs._grid_plan, cs._status = self._grid_plan(1), self.grid_status
        self.sets = {1: cs}
        self.parent_of = {}
        self.kmaps = {}
        self._ws = ws
        if pyr is not None:
            lvl, par, counts = pyr
            ts = 1
            for l in range(len(counts) - 1):
                self.sets[2 * ts] = CoordSet(lvl[l, :counts[l + 1]], 2 * ts, self._grid_plan(2 * ts), self.grid_status)
                self.parent_of[(ts, 2 * ts)] = par[l, :counts[l]]
                ts *= 2

    def _grid_plan(self, ts):
        """(log2_ts, nbits, n_batch) of the occupancy grid for the set at tensor stride ts, or None (use the hash)."""
        if self._grid0 is None or ts & (ts - 1):
            return None
        nbits0, n_batch = self._grid0
        log2_ts = ts.bit_length() - 1
        nbits = max(2, nbits0 - log2_ts)
        if nbits > 9 or C.lib().osb_occgrid_bytes(nbits, n_batch) == 0:
            return None
        return (log2_ts, nbits, n_batch)

    # -- coordinate sets -------------------------------------------------------------------
    def stride(self, ts, s):
        """Tensor stride ts -> ts*s: unique(floor(c/(ts*s))*(ts*s)); cached."""
        new = ts * s
        if new not in self.sets:
            fine = self.sets[ts]
            with torch.cuda.device(self.device):
                coarse = torch.empty_like(fine.coords)
                parent = torch.empty(fine.n, dtype=torch.int32, device=self.device)
                n_c = ctypes.c_int64(0)
                ws_bytes = C.lib().osb_coordset_workspace_bytes(fine.n)
                if self._ws.numel() < ws_bytes:
                    self._ws = torch.empty(ws_bytes, dtype=torch.uint8, device=self.device)
                C.call('osb_coordset_stride', C.ptr(fine.coords), fine.n, new, C.ptr(coarse), C.ptr(parent),
                       ctypes.byref(n_c), C.ptr(self._ws), self._ws.numel(), C.stream_ptr())
            self.sets[new] = CoordSet(coarse[:n_c.value].contiguous(), new, self._grid_plan(new), self.grid_status)
            self.parent_of[(ts, new)] = parent
        return new

    # -- kernel maps -----------------------------------------------------------------------
    def kernel_map(self, ts_in, ts_out, kernel_size, dilation=1):
        """Map of a conv reading the set at ts_in and writing the set at ts_out."""
        key = (ts_in, ts_out, kernel_size, dilation)
        km = self.kmaps.get(key)
        if km is None:
            cout = self.sets[ts_out]
            K = kernel_size ** 3
            with torch.cuda.device(self.device):
                cin = self.sets[ts_in].ensure_lookup()
                nbr = torch.empty((K, cout.n), dtype=torch.int32, device=self.device)
                pairs = torch.empty(K, dtype=torch.int32, device=self.device)
                if cin.grid is not None:
                    C.call('osb_kernel_map_build_grid', C.ptr(cout.coords), cout.n, C.ptr(cin.grid), *cin.grid_args,
                           kernel_size, kernel_size, kernel_size, ts_in * dilation, C.ptr(nbr), C.ptr(pairs), C.stream_ptr())
                else:
                    C.call('osb_kernel_map_build', C.ptr(cout.coords), cout.n, C.ptr(cin.slots), cin.cap,
                           kernel_size, kernel_size, kernel_size, ts_in * dilation, C.ptr(nbr), C.ptr(pairs),
                           C.stream_ptr())
            km = KernelMap(nbr, K, cin.n, cout.n, pairs)
            self.kmaps[key] = km
        return km

    def batch_index(self, ts):
        """(int32 batch index of every row in ``.F`` order, batch count = largest index + 1) of the set at ts.  The count
        is read from the device once per set and cached."""
        cache = self.__dict__.setdefault('_batch_index', {})
        hit = cache.get(ts)
        if hit is None:
            b = self.coords_external(ts)[:, 0].contiguous()
            hit = cache[ts] = (b, int(b.max().item()) + 1)
        return hit

    def coords_external(self, ts):
        """int32 [N,4] in the caller's row order (stride 1) / internal order (coarser sets)."""
        c = self.sets[ts].coords
        return c[self.inv_perm.long()] if ts == 1 else c
