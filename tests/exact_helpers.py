"""Poisoned inputs, guarded outputs and element-wise comparisons shared by the exact kernel tests.

Every operand is a view into a larger buffer whose padding columns and trailing rows hold NaN, so a kernel that reads past
a row or ignores the row stride picks up NaN. Every output is an interior view surrounded by sentinel guard bands that must
come back bit-unchanged, so a kernel that writes past its view is caught.
"""
import pytest
import torch

bf16, f32 = torch.bfloat16, torch.float32

GUARD_R, GUARD_C = 128, 256                      # guard band around every output: one tile of rows / a 256-wide tile of columns
PAD_R, PAD_C = 128, 64                           # NaN rows after / NaN columns right of every input view
_SENTINEL_BITS = {bf16: (torch.int16, 0x7FA5), f32: (torch.int32, 0x7FA5A5A5)}   # NaN payloads no kernel writes


def _poisoned(x: torch.Tensor, col0: int = 0, pad_c: int = PAD_C) -> torch.Tensor:
    """x [r, c] copied into a NaN buffer [r + 128, col0 + c + pad_c] at column col0: a view whose row stride runs into NaN
    columns and whose rows are followed by NaN rows (1-D: N values followed by 256 NaNs)"""
    if x.dim() == 1:
        buf = torch.full((x.shape[0] + 256,), float("nan"), dtype=x.dtype, device=x.device)
        buf[: x.shape[0]] = x
        return buf[: x.shape[0]]
    r, c = x.shape
    buf = torch.full((r + PAD_R, col0 + c + pad_c), float("nan"), dtype=x.dtype, device=x.device)
    buf[:r, col0:col0 + c] = x
    return buf[:r, col0:col0 + c]


class Guarded:
    """an output view [rows, cols] inside a sentinel-filled buffer with GUARD_R rows above / below and GUARD_C columns left /
    right (16-byte aligned: the view starts 256 elements into a row and the row stride is cols + 512). `shift` moves the view
    that many elements right (a start that is not 16-byte aligned) and `ld_extra` widens the row stride."""

    def __init__(self, rows, cols, dtype, dev, init=None, shift=0, ld_extra=0):
        itype, bits = _SENTINEL_BITS[dtype]
        self.buf = torch.full((rows + 2 * GUARD_R, cols + 2 * GUARD_C + ld_extra), bits, dtype=itype, device=dev).view(dtype)
        self.rows, self.cols, self.itype, self.bits, self.c0 = rows, cols, itype, bits, GUARD_C + shift
        self.view = self.buf[GUARD_R:GUARD_R + rows, self.c0:self.c0 + cols]
        if init is not None:
            self.view.copy_(init)

    def check(self, what):
        b = self.buf.view(self.itype).clone()
        b[GUARD_R:GUARD_R + self.rows, self.c0:self.c0 + self.cols] = self.bits
        bad = b != self.bits
        if bad.any():
            r, c = bad.nonzero()[0].tolist()
            pytest.fail(f"{what}: {int(bad.sum())} guard elements overwritten; first at buffer ({r}, {c}) = output "
                        f"({r - GUARD_R}, {c - self.c0}) of a [{self.rows}, {self.cols}] view")


def _ulp_bf16(x):
    """spacing of bf16 numbers at |x| (fp64), normal range"""
    return torch.pow(2.0, torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126))) - 7)


def _ulp_f32(x):
    return torch.pow(2.0, torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126))) - 23)


def _where(bad, what, tile_m=128, tile_n=None):
    r, c = bad.nonzero()[0].tolist()
    tile = f" = tile (m {r // tile_m}, n {c // tile_n})" if tile_n else ""
    return f"{what}: {int(bad.sum())} of {bad.numel()} elements wrong; first at (row {r}, col {c}){tile}"


def _expect_equal(got, want, what, tile_m=128, tile_n=None):
    """got (kernel output, any float dtype) == want (same dtype) element for element (+0 == -0), no NaN"""
    g, w = got.double(), want.double()
    bad = (g != w) | torch.isnan(g)
    if bad.any():
        r, c = bad.nonzero()[0].tolist()
        pytest.fail(_where(bad, what, tile_m, tile_n) + f": got {g[r, c].item()!r}, want {w[r, c].item()!r}")


def _expect_close(got, ref, tol, what, tile_m=128, tile_n=None):
    """|got - ref| <= tol element-wise (fp64), no NaN"""
    g = got.double()
    bad = ~((g - ref).abs() <= tol)
    if bad.any():
        r, c = bad.nonzero()[0].tolist()
        pytest.fail(_where(bad, what, tile_m, tile_n) + f": got {g[r, c].item()!r}, ref {ref[r, c].item()!r}, "
                    f"tol {tol[r, c].item() if torch.is_tensor(tol) else tol!r}")
