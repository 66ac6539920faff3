"""Operands for the codebook-lookup tests (test_vq_lookup_cpu.py checks the construction, test_gpu_vq_lookup.py uses it).

Two grids on which every intermediate of the search is exact in fp32, in the kernel's order (csrc/vq.cu vq_dist: sum z^2
sequentially, 2z.E as one multiply and seven fmas, then (zz - dot) + ek) and in any other order (the oracle's):

* the tie grid: z in Z/8 and E in Z/2, both with |.| <= 1.  Squares and products 2 z E are multiples of 2^-6, and every
  partial sum stays below 2^5 in magnitude, so it fits in 11 significant bits.  Distances collide often (the minimum is
  shared by 10 to 30 % of the rows), and a correct kernel has exactly one answer: the first fp64 argmin.
* the ulp grid: integers.  Every code has one large component E_0 (2905 for planted codes, 2912 .. 2950 for the others)
  and small ones in [-4, 4]; rows have |z| <= 4.  Every distance lies in [2^23, 2^24), where adjacent integers are
  adjacent floats, and every partial sum is an integer below 2^24.  A planted row is (0, c) with c a point of
  {-3, 0, 3}^7 of its own; its planted codes are (2905, c), at distance D = 2905^2, or (2905, c + e_1), at D + 1: one
  ulp further.  Every other code is at D + 4 or more (other planted codes differ from c by 3 in some component).
"""
import torch

LROWS = (0, 63, 64, 127, 128, 255, 256, 383, 384, 511)     # row offsets in a cluster block: every rows-per-thread slot, every owner CTA
KINDS = ("tie", "last", "first")     # all planted codes at D | only the last at D | only the first at D (the others at D + 1)
A_PLANT, A_LO, A_HI = 2905, 2912, 2950


def tuples(n_codes):
    """Disjoint code tuples to plant ties in: the planted winner is the first of a tuple, or its last."""
    per = n_codes // 8
    t = [(2 * per, 2 * per + 7), (2 * per + 3, 2 * per + 4),        # one group of 8 codes: its ends, its middle pair
         (3 * per, 4 * per - 1),                                    # first and last code of one slice
         (per - 1, per), (7 * per - 1, 7 * per),                    # adjacent slices
         (0, n_codes - 1),                                          # the whole table
         (per + 5, 4 * per + 1, 6 * per + 6)]                       # a three-way tie over three slices
    if per >= 16:
        t.append((5 * per + 7, 5 * per + 8))                        # adjacent groups of one slice
    flat = [k for c in t for k in c]
    assert len(set(flat)) == len(flat) and max(flat) < n_codes
    return t


def lattice(p):
    """The p-th point of {-3, 0, 3}^7."""
    return [3 * ((p // 3 ** i) % 3) - 3 for i in range(7)]


def e2_of(E):
    """sum E^2 by the reference's expression (modules/codebook.py:84), as the engine packs it."""
    return (E.t() ** 2).sum(dim=0)


def ulp_table(n_codes, kind, seed):
    """Codebook on the ulp grid with the tuples of `tuples` planted for `kind`.  Returns (E, plants): plants[p] =
    (codes, winner, c), the codes of tuple p, its expected index and the z_1..7 of the rows that see it."""
    g = torch.Generator().manual_seed(seed)
    E = torch.empty(n_codes, 8)
    E[:, 0] = torch.randint(A_LO, A_HI + 1, (n_codes,), generator=g).float()
    E[:, 1:] = torch.randint(-4, 5, (n_codes, 7), generator=g).float()
    plants = []
    for p, codes in enumerate(tuples(n_codes)):
        c = lattice(p)
        near = {"tie": codes, "last": codes[-1:], "first": codes[:1]}[kind]
        for k in codes:
            E[k, 0] = A_PLANT
            E[k, 1:] = torch.tensor(c, dtype=torch.float32)
            if k not in near:
                E[k, 1] += 1
        plants.append((codes, near[0], c))
    return E, plants


def planted_rows(M, rows_per_block, n_plants, device="cpu"):
    """Rows at the offsets LROWS (those below rows_per_block) of every cluster block, and the tuple each one sees: the
    tuple index moves with the block, so every tuple meets every offset once there are enough blocks."""
    r = torch.arange(M, device=device)
    slot = torch.full((rows_per_block,), -1, dtype=torch.int64, device=device)
    lr = [x for x in LROWS if x < rows_per_block]
    slot[torch.tensor(lr, device=device)] = torch.arange(len(lr), device=device)
    s = slot[r % rows_per_block]
    rows = r[s >= 0]
    return rows, (rows // rows_per_block + s[s >= 0]) % n_plants


def ulp_rows(M, rows_per_block, plants, seed, device="cpu"):
    """z [M, 8] on the ulp grid: planted rows (0, c) at the LROWS offsets, every other row random with |z| <= 4.
    Returns (z, rows, want): the planted rows and their expected indices."""
    g = torch.Generator(device=device).manual_seed(seed)
    z = torch.randint(-4, 5, (M, 8), generator=g, device=device).float()
    rows, which = planted_rows(M, rows_per_block, len(plants), device)
    cs = torch.tensor([[0.0] + p[2] for p in plants], device=device)
    z[rows] = cs[which]
    want = torch.tensor([p[1] for p in plants], device=device)[which]
    return z, rows, want


def tie_grid(M, n_codes, seed, device="cpu"):
    """(z, E) on the tie grid."""
    g = torch.Generator(device=device).manual_seed(seed)
    z = torch.randint(-8, 9, (M, 8), generator=g, device=device).float() / 8
    E = torch.randint(-2, 3, (n_codes, 8), generator=g, device=device).float() / 2
    return z, E


def grid_projection(z, C, seed):
    """(x [M, C], Wt [8, C], b [8]) with x . Wt^T + b == z exactly: Wt = [I | W'], W' in {-1, 0, 1}, x[:, 8:] in [-2, 2],
    b in [-8, 8] integers and x[:, :8] = z - b - x[:, 8:] . W'^T.  With z on either grid every product and partial sum of
    the projection, in any order, is on the grid of z and below 2^12 in magnitude, so the kernel's projection is exact."""
    dev = z.device
    g = torch.Generator(device=dev).manual_seed(seed)
    M = z.shape[0]
    Wt = torch.zeros(8, C, device=dev)
    Wt[:, :8] = torch.eye(8, device=dev)
    Wt[:, 8:] = torch.randint(-1, 2, (8, C - 8), generator=g, device=dev).float()
    b = torch.randint(-8, 9, (8,), generator=g, device=dev).float()
    x = torch.empty(M, C, device=dev)
    x[:, 8:] = torch.randint(-2, 3, (M, C - 8), generator=g, device=dev).float()
    x[:, :8] = (z.double() - b.double() - x[:, 8:].double() @ Wt[:, 8:].double().t()).float()
    return x, Wt, b


def ref_argmin(z, E, chunk=4096):
    """First argmin of the fp64 distances sum_c (z_c - E_c)^2, expanded as zz - 2 z.E + ee (exact on both grids)."""
    zd, Ed = z.double(), E.double()
    ee = (Ed * Ed).sum(1)
    out = []
    for i in range(0, zd.shape[0], chunk):
        zc = zd[i:i + chunk]
        d = (zc * zc).sum(1, keepdim=True) - 2.0 * zc @ Ed.t() + ee
        out.append(torch.argmin(d, dim=1))
    return torch.cat(out) if out else torch.empty(0, dtype=torch.int64, device=z.device)
