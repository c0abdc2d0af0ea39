"""Open exploration tours over a cost matrix (tslam_tour_open, include/tslam.h; DESIGN.md section 7)."""
import math

import numpy as np

from . import _capi as capi


def solve_open_tour(C, restarts=64, seed=0, max_passes=None):
    """Order the goals 1..n-1 of the cost matrix C [n, n] (a torch CUDA tensor or a numpy array, f32; node 0 the start)
    into an open tour from node 0: `restarts` 2-opt / Or-opt local searches, restart 0 from the nearest-neighbour tour,
    the others from seeded shuffles.  max_passes (moves per restart) defaults to 64 * n.  Returns a dict:
      order        int64[m]: the kept goals (C[0][g] finite) in visiting order, from the best restart
      unreachable  int64[n-1-m]: the other goals, ascending
      inf_legs     infinite legs of the best tour; cost: its finite legs' exact sum, as f64 (q * U)
      tours int32[R,n] (-1 past m), cost2 int64[R,2] (inf legs, q), passes int32[R], converged bool[R], best, m,
      unit_exp (U = 2^unit_exp)
    Raises TslamError (E_INVALID) on a matrix or argument the contract refuses."""
    import torch
    if isinstance(C, torch.Tensor):
        if not C.is_cuda:
            raise ValueError("solve_open_tour needs a CUDA tensor or a numpy array")
        c = C.detach().to(torch.float32).contiguous()
    else:
        c = torch.from_numpy(np.ascontiguousarray(np.asarray(C, np.float32))).to(capi.device())
    if c.dim() != 2 or c.shape[0] != c.shape[1]:
        raise ValueError(f"the cost matrix must be [n, n], not {tuple(c.shape)}")
    n, R = int(c.shape[0]), int(restarts)
    mp = 64 * n if max_passes is None else int(max_passes)
    L = capi.load()
    rows = max(R, 1)  # a refused R still reaches the library, which names it
    tours = torch.empty((rows, max(n, 1)), dtype=torch.int32, device=c.device)
    cost2 = torch.empty((rows, 2), dtype=torch.int64, device=c.device)
    passes = torch.empty(rows, dtype=torch.int32, device=c.device)
    conv = torch.empty(rows, dtype=torch.uint8, device=c.device)
    best = torch.empty(1, dtype=torch.int32, device=c.device)
    info2 = np.zeros(2, np.int32)
    capi.check(L.tslam_tour_open(n, capi.tptr(c) if n else None, R, int(seed) & ((1 << 64) - 1), mp, capi.tptr(tours),
                                 capi.tptr(cost2), capi.tptr(passes), capi.tptr(conv), capi.tptr(best), capi.np_ptr(info2),
                                 capi.stream_ptr()))
    tours, cost2 = tours.cpu().numpy(), cost2.cpu().numpy()
    b, m, ue = int(best.item()), int(info2[0]), int(info2[1])
    order = tours[b, 1:m + 1].astype(np.int64)
    return dict(order=order, unreachable=np.setdiff1d(np.arange(1, n), order), inf_legs=int(cost2[b, 0]),
                cost=math.ldexp(float(cost2[b, 1]), ue), tours=tours, cost2=cost2, passes=passes.cpu().numpy(),
                converged=conv.cpu().numpy().astype(bool), best=b, m=m, unit_exp=ue)
