"""masked_l2_nn -- raft::distance::masked_l2_nn: the fused L2 1-NN restricted by a row x group adjacency mask
(the nearest-neighbour step of connect_components: for every point the nearest point in another component)."""
from __future__ import annotations

import torch

from .. import _lib
from ..common import auto_sync_handle, cai_wrapper
from .fused_l2_nn import _check_xy

NO_CANDIDATE = 0x7FFFFFFF   # key of a row without any adjacent row of Y (value FLT_MAX)


@auto_sync_handle
def masked_l2_nn(X, Y, adj, group_idxs, sqrt=False, xn=None, yn=None, handle=None):
    """For every row i of X, (index, distance) of the nearest row j of Y among the rows whose group g has
    adj[i, g] != 0.  Returns (indices int32 [m], distances float32 [m]) as torch tensors, like fused_l2_nn.

    adj: bool or uint8 [m, num_groups] (a torch tensor or any __cuda_array_interface__ object), rows contiguous.
    group_idxs: integer [num_groups], the END of every group (inclusive scan of the group sizes): group g holds the rows
    [group_idxs[g-1], group_idxs[g]) of Y; rows at or after group_idxs[-1] are in no group.  Ties go to the smaller j;
    a row without an adjacent row gets index 0x7fffffff and distance FLT_MAX.  sqrt: Euclidean instead of squared
    distances.  xn / yn: optional precomputed squared row norms.  A group_idxs that decreases or leaves [0, n] raises
    LogicError (checked on the device; this call synchronises)."""
    x_cai, y_cai = _check_xy(X, Y)
    m, k = x_cai.shape
    n = y_cai.shape[0]
    with torch.cuda.stream(handle.torch_stream):
        a = torch.as_tensor(adj, device=handle.device)
        if a.dtype not in (torch.bool, torch.uint8):
            raise TypeError("adj must be bool or uint8, got %s" % a.dtype)
        if a.dim() != 2 or a.shape[0] != m:
            raise ValueError("adj must have shape (%d, num_groups), got %s" % (m, tuple(a.shape)))
        num_groups = a.shape[1]
        if num_groups > 1 and a.stride(1) != 1:
            raise ValueError("adj must be row-major with contiguous rows")
        ld_adj = a.stride(0) if m > 1 else num_groups
        g = torch.as_tensor(group_idxs, device=handle.device)
        if g.dtype.is_floating_point or g.dtype.is_complex or g.dtype == torch.bool:
            raise TypeError("group_idxs must be an integer array, got %s" % g.dtype)
        if g.dim() != 1 or g.shape[0] != num_groups:
            raise ValueError("group_idxs must have shape (%d,), got %s" % (num_groups, tuple(g.shape)))
        if g.dtype != torch.int32 and g.numel() and (int(g.min()) < 0 or int(g.max()) > n):
            # (checked before the narrowing: a wider value would wrap into the int32 range and could look valid)
            raise _lib.LogicError("group_idxs must be non-decreasing and lie in [0, n]")
        g = g.to(torch.int32).contiguous()
        kvp = torch.empty((m, 2), dtype=torch.int32, device=handle.device)
    L = _lib.lib()
    ws = handle.workspace(L.b2d_masked_l2_nn_workspace_bytes(m, n, k, num_groups))
    xn_p = cai_wrapper(xn).data if xn is not None else None
    yn_p = cai_wrapper(yn).data if yn is not None else None
    _lib.check(L.b2d_masked_l2_nn(handle.stream_ptr, kvp.data_ptr(), x_cai.data, k, y_cai.data, k, xn_p, yn_p,
                                  a.data_ptr(), ld_adj, g.data_ptr(), num_groups, m, n, k, 1 if sqrt else 0, 1,
                                  ws.data_ptr(), ws.numel()))
    idx, dist = kvp[:, 0], kvp[:, 1].view(torch.float32)
    if m > 0:
        # an invalid group_idxs leaves {0x7fffffff, NaN} in every row, which no valid call produces
        handle.sync()
        if int(idx[0]) == NO_CANDIDATE and bool(torch.isnan(dist[0])):
            raise _lib.LogicError("group_idxs must be non-decreasing and lie in [0, n]")
    return idx, dist
