"""Test infrastructure of tests/test_full_size_exact_gpu.py: on-device references of the bench workloads, an
element-by-element comparison that runs in row blocks, and the tile or CTA that wrote a given element of C.

Everything here takes torch tensors on any device, so the CPU suite (tests/test_full_size_exact_cpu.py) runs the same
code on small shapes.

* `exact_operands`: the exact data of tensor_numerics.full_size_scheme, drawn with a seeded torch.Generator in row
  blocks on the given device; "tf32" with A's last row times 2^20, so that float runs on TF32, "tf32h" without.
* `fp64_reference`: the FP64 product in row blocks of A, stored once in the output type (modulo 256 for uint8).
* `min_plus_reference`, `sequential_half_reference`: Naive<>'s order of operations for (Add, Min) and half
  (Multiply, Add), one torch op per Map and per Reduce, each rounding once.
* `Tally`: counts wrong elements over row blocks and reports the first one with the tile that wrote it.
* `check_guard`: the bytes after C still hold the poison.
"""
import tensor_numerics as tn

# default tuning of the wgmma GEMM (gemm_wgmma.cuh, capi.cu): clusters of two 128-row CTAs, BN = 256, raster
# groups of 2048 rows
WGMMA_TILE, WGMMA_RASTER_TILES = 256, 2048 // 256
SEMIRING_TILE = 128          # semiring_tile_kernel and semiring_ring_kernel: one 128 x 128 C tile per CTA
DMMA_TILE_COLS = 128
GUARD = 4096
ROW_BLOCK = 4096


def _cdiv(a, b):
    return (a + b - 1) // b


# ---- which tile or CTA wrote an element of C --------------------------------------------------------------------

def wgmma_tile_coord(t, tiles_r, tiles_c, raster=WGMMA_RASTER_TILES):
    """(row tile, column tile) of persistent tile t of one problem: the device's tile_coord (gemm_wgmma.cuh)."""
    per_group = raster * tiles_c
    g = t // per_group
    first = g * raster
    gsize = min(raster, tiles_r - first)
    i = t - g * per_group
    return first + i % gsize, i // gsize


def wgmma_tile_index(r, c, tiles_r, tiles_c, raster=WGMMA_RASTER_TILES):
    """The persistent tile index of (row tile r, column tile c): the inverse of wgmma_tile_coord."""
    g = r // raster
    first = g * raster
    return g * raster * tiles_c + c * min(raster, tiles_r - first) + (r - first)


def wgmma_locator(n, m, sms):
    """(row, col) -> where the default-tuning wgmma GEMM computed C[row, col] on a GPU with `sms` SMs."""
    tiles_r, tiles_c = _cdiv(n, WGMMA_TILE), _cdiv(m, WGMMA_TILE)
    groups = min(tiles_r * tiles_c, sms // 2)

    def locate(row, col):
        r, c = row // WGMMA_TILE, col // WGMMA_TILE
        t = wgmma_tile_index(r, c, tiles_r, tiles_c)
        return ("wgmma tile (row tile %d, column tile %d) of %d x %d: persistent tile %d of %d, CTA group %d of %d, "
                "its tile #%d" % (r, c, WGMMA_TILE, WGMMA_TILE, t, tiles_r * tiles_c, t % groups, groups, t // groups))
    return locate


def grid_locator(kernel, tile_rows, tile_cols, n, m):
    """(row, col) -> the blockIdx of the non-persistent kernel (one tile_rows x tile_cols C tile per CTA)."""
    def locate(row, col):
        return "%s CTA blockIdx (x %d, y %d) of a %d x %d grid of %d x %d tiles" % (
            kernel, col // tile_cols, row // tile_rows, _cdiv(m, tile_cols), _cdiv(n, tile_rows), tile_rows, tile_cols)
    return locate


def dmma_tile_rows(n, m, sms, forced=0):
    """Rows of the DMMA kernel's C tile: the host's choice in gemm_dmma.cu (64 when it saves more than a wave)."""
    if forced:
        return forced
    t128, t64 = _cdiv(n, 128) * _cdiv(m, DMMA_TILE_COLS), _cdiv(n, 64) * _cdiv(m, DMMA_TILE_COLS)
    return 64 if 0.5 * 1.05 * _cdiv(t64, sms) < _cdiv(t128, sms) else 128


# ---- comparison -------------------------------------------------------------------------------------------------

_INT_VIEW = {1: "uint8", 2: "int16", 4: "int32", 8: "int64"}


def _bits(torch, x):
    return x if x.element_size() == 1 else x.view(getattr(torch, _INT_VIEW[x.element_size()]))


class Tally:
    """Wrong elements of one C, accumulated over row blocks.  mode "value": equal as numbers (+0 == -0: the sign of a
    zero sum is not pinned; NaN, the poison, equals nothing); "bits": the same bytes.  `poison` (a byte) also counts
    the elements whose every byte still holds it."""

    def __init__(self, torch, what, locate, mode, poison):
        self.torch, self.what, self.locate, self.mode, self.poison = torch, what, locate, mode, poison
        self.bad = self.poisoned = self.total = 0
        self.first = None

    def add(self, row0, got, want):
        torch = self.torch
        if self.mode == "value":
            wrong = ~(got == want)
        else:
            wrong = _bits(torch, got) != _bits(torch, want)
        raw = got.contiguous().view(torch.uint8).reshape(got.shape[0], got.shape[1], got.element_size())
        self.poisoned += int((raw == self.poison).all(dim=2).sum())
        count = int(wrong.sum())
        self.total += got.numel()
        if count and self.first is None:
            i = int(wrong.reshape(-1).to(torch.uint8).argmax())   # the first wrong element in row-major order
            r, c = divmod(i, got.shape[1])
            self.first = (row0 + r, c, got[r, c].item(), want[r, c].item())
        self.bad += count

    def check(self):
        if self.bad:
            row, col, g, w = self.first
            raise AssertionError(
                "%s: %d of %d elements wrong (%d still hold the poison byte 0x%02X); first at (row %d, col %d): "
                "got %r, want %r; %s" % (self.what, self.bad, self.total, self.poisoned, self.poison, row, col, g, w,
                                         self.locate(row, col)))


def compare(torch, what, c, want, locate, mode, poison, row_block=ROW_BLOCK):
    """Every element of C (n x m) against `want` (a tensor of the same shape, or a function (r0, r1) -> the rows
    r0:r1 of it), in row blocks; raises with the Tally report."""
    t = Tally(torch, what, locate, mode, poison)
    for r0 in range(0, c.shape[0], row_block):
        r1 = min(r0 + row_block, c.shape[0])
        t.add(r0, c[r0:r1], want(r0, r1) if callable(want) else want[r0:r1])
    t.check()


def check_guard(torch, what, guard, poison):
    """The bytes after C (a uint8 tensor) all still hold the poison."""
    changed = guard != poison
    count = int(changed.sum())
    if count:
        i = int(changed.to(torch.uint8).argmax())
        raise AssertionError("%s: the call wrote %d of the %d guard bytes after C; first at byte +%d: 0x%02X" % (
            what, count, guard.numel(), i, int(guard[i])))


# ---- data -------------------------------------------------------------------------------------------------------

def exact_operands(torch, path, n, k, m, seed, device, row_block=ROW_BLOCK):
    """A (n x k) and B (k x m) of path's exact data (tensor_numerics.full_size_scheme), in its input type on
    `device`.  uint8: full-range bytes.  Adjacent rows of A and adjacent columns of B never share a scale.  "tf32":
    the "tf32h" data with A's last row times tensor_numerics.PLANT_SCALE (exact; its values are no halves, so the
    float GEMM runs on TF32)."""
    dt = {"tf32": torch.float32, "tf32h": torch.float32, "tf32x3": torch.float32, "f16": torch.float16,
          "bf16": torch.bfloat16, "dmma": torch.float64, "u8": torch.uint8}[path]
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    if path == "u8":
        return (torch.randint(0, 256, (n, k), generator=g, device=device, dtype=torch.uint8),
                torch.randint(0, 256, (k, m), generator=g, device=device, dtype=torch.uint8))
    lim, (ea0, ea1), (eb0, eb1) = tn.full_size_scheme(path, k)
    # float64 holds every value of every input type exactly; one block at a time keeps the temporaries small
    wide = torch.float64 if path == "dmma" else torch.float32

    def ints(rows, cols):
        v = torch.randint(1, lim + 1, (rows, cols), generator=g, device=device, dtype=torch.int32)
        s = torch.randint(0, 2, (rows, cols), generator=g, device=device, dtype=torch.int32) * 2 - 1
        return (v * s).to(wide)

    def fill(out, cols, scale):
        for r0 in range(0, out.shape[0], row_block):
            r1 = min(r0 + row_block, out.shape[0])
            out[r0:r1] = (ints(r1 - r0, cols) * scale(r0, r1)).to(dt)
        return out

    ea = ea0 + torch.arange(n, device=device) % (ea1 - ea0 + 1)
    eb = eb0 + torch.arange(m, device=device) % (eb1 - eb0 + 1)
    col_scale = torch.exp2(eb.to(wide))[None, :]
    a = fill(torch.empty((n, k), device=device, dtype=dt), k, lambda r0, r1: torch.exp2(ea[r0:r1].to(wide))[:, None])
    b = fill(torch.empty((k, m), device=device, dtype=dt), m, lambda r0, r1: col_scale)
    if path == "tf32":
        a[n - 1] *= tn.PLANT_SCALE
    return a, b


def fp64_reference(torch, path, a, b, row_block=ROW_BLOCK):
    """C = A B evaluated in FP64 (exact for the exact data), stored once in path's output type: float32 for the TF32
    paths, FP64 -> float32 (exact) -> half / bfloat16, float64 for DMMA, the exact sum modulo 256 for uint8."""
    out = {"tf32": torch.float32, "tf32h": torch.float32, "tf32x3": torch.float32, "f16": torch.float16,
           "bf16": torch.bfloat16, "dmma": torch.float64, "u8": torch.uint8}[path]
    b64 = b.to(torch.float64)
    c = torch.empty((a.shape[0], b.shape[1]), device=a.device, dtype=out)
    for r0 in range(0, a.shape[0], row_block):
        r1 = min(r0 + row_block, a.shape[0])
        c64 = a[r0:r1].to(torch.float64) @ b64
        if path == "u8":
            c[r0:r1] = torch.remainder(c64, 256.0).to(torch.uint8)
        elif path in ("f16", "bf16"):
            c[r0:r1] = c64.to(torch.float32).to(out)
        else:
            c[r0:r1] = c64.to(out)
        del c64
    del b64
    return c


def min_plus_reference(torch, a, b):
    """float (Add, Min): C = min over k of (A[:, k] + B[k, :]), one float addition per element and k, in k order."""
    at = a.t().contiguous()
    c = torch.full((a.shape[0], b.shape[1]), float("inf"), device=a.device, dtype=a.dtype)
    tmp = torch.empty_like(c)
    for kk in range(a.shape[1]):
        torch.add(at[kk].unsqueeze(1), b[kk].unsqueeze(0), out=tmp)
        torch.minimum(c, tmp, out=c)
    return c


def sequential_half_reference(torch, a, b):
    """half (Multiply, Add) as Naive<half>: C = 0, then for each k in order tmp = A[:, k] * B[k, :] rounded to half,
    C = C + tmp rounded to half.  Two separate torch ops: each evaluates in float32 and rounds once to half, which
    is the correctly rounded half result (float32 has more than 2 x 11 + 2 bits)."""
    at = a.t().contiguous()
    c = torch.zeros((a.shape[0], b.shape[1]), device=a.device, dtype=a.dtype)
    tmp = torch.empty_like(c)
    for kk in range(a.shape[1]):
        torch.mul(at[kk].unsqueeze(1), b[kk].unsqueeze(0), out=tmp)
        torch.add(c, tmp, out=c)
    return c
