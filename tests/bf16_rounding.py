"""The rounding-aware checker of the fp64 contract tests (`test_row_kernels_contract_gpu.py`,
`test_train_kernels_contract_gpu.py`).

A bf16 output y "rounds z within E" (z the float64 reference, E a bound of the kernel's fp32 error before its final
bf16 rounding) when
  (a) |y - z| <= E + ulp_bf16(|z| + E) / 2, and
  (b) y == RN_bf16(z) wherever no bf16 rounding midpoint lies in [z - E, z + E].
(b) is the sharp part: away from ties the output is the correctly rounded float64 value, bit for bit (values compared,
so +0 == -0).  `rounds_twice` checks an output that is rounded twice: its inner bf16 value has at most two candidates,
and the outer operation is exact in fp32 and rounded once.

Every check records, per family, the worst err / E (err = |y - z| - ulp_bf16(y) / 2, a lower bound of the kernel's
error before its last rounding) and the fraction of elements whose E interval held a rounding midpoint;
`print_report` prints and clears them.
"""
import torch

U = 2.0 ** -24

REPORT = {}                        # family -> [worst err / E, tie elements, elements]


def bf16_ulp(a):
    """ulp of bf16 at |a| (float64): 2^(e - 8) for |a| in [2^(e-1), 2^e), never below the subnormal step 2^-133."""
    _, e = torch.frexp(a.abs())
    # the power of two from its bit pattern: torch.pow(2.0, e) on CUDA is not exact in float64
    q = (((e - 8).clamp(min=-133).to(torch.int64) + 1023) << 52).view(torch.float64)
    return torch.where(a == 0, torch.full_like(q, 2.0 ** -133), q)


def rn_bf16(z):
    """Correctly rounded (nearest, ties to even) bf16 value of a float64 tensor, as float64.  One rounding: torch's
    float64 -> bf16 cast goes through fp32 and may round twice."""
    q = bf16_ulp(z)
    return torch.round(z / q) * q


def _note(family, y, z, E, tie):
    err = ((y - z).abs() - 0.5 * bf16_ulp(y)).clamp(min=0)
    note_ratio(family, float((err / E.clamp(min=1e-300)).max()) if err.numel() else 0.0)
    r = REPORT[family]
    r[1] += int(tie.sum())
    r[2] += tie.numel()


def note_ratio(family, ratio):
    r = REPORT.setdefault(family, [0.0, 0, 0])
    r[0] = max(r[0], ratio)


def rounds_mask(y, z, E):
    """Elementwise: does y round z within E?  Returns (ok, tie)."""
    y, z = y.double(), z.double()
    E = torch.as_tensor(E, dtype=torch.float64, device=z.device).expand_as(z) * (1 + 2.0 ** -20)
    tie = rn_bf16(z - E) != rn_bf16(z + E)
    allow = E + 0.5 * bf16_ulp(z.abs() + E)
    ok = torch.where(tie, (y - z).abs() <= allow, y == rn_bf16(z))
    return ok, tie


def rounds(y, z, E, family, what=""):
    ok, tie = rounds_mask(y, z, E)
    if not bool(ok.all()):
        i = int((~ok).flatten().nonzero()[0])
        raise AssertionError(f"{family} {what}: {int((~ok).sum())} / {ok.numel()} elements off; first at flat index {i}: "
                             f"y={y.double().flatten()[i].item()!r} z={z.double().flatten()[i].item()!r} "
                             f"E={torch.as_tensor(E).double().expand_as(z).flatten()[i].item()!r}")
    _note(family, y.double(), z.double(), torch.as_tensor(E, dtype=torch.float64, device=z.device).expand_as(z), tie)


def rounds_twice_mask(y, z_in, E_in, outer):
    """y = RN(outer(c)) for a bf16 candidate c of the inner value: c = RN(z_in) away from ties, RN(z_in -+ E_in) at ties."""
    y, z_in = y.double(), z_in.double()
    E_in = torch.as_tensor(E_in, dtype=torch.float64, device=z_in.device).expand_as(z_in) * (1 + 2.0 ** -20)
    lo, hi = rn_bf16(z_in - E_in), rn_bf16(z_in + E_in)
    tie = lo != hi
    ok = y == outer(rn_bf16(z_in))
    ok |= tie & ((y == outer(lo)) | (y == outer(hi)))
    return ok, tie


def rounds_twice(y, z_in, E_in, outer, family, what=""):
    ok, tie = rounds_twice_mask(y, z_in, E_in, outer)
    if not bool(ok.all()):
        i = int((~ok).flatten().nonzero()[0])
        raise AssertionError(f"{family} {what}: {int((~ok).sum())} / {ok.numel()} elements off; first at flat index {i}: "
                             f"y={y.double().flatten()[i].item()!r} z_inner={z_in.double().flatten()[i].item()!r}")
    # the inner value the kernel must have produced: the allowed candidate whose outer image is y
    c = rn_bf16(z_in.double())
    c = torch.where(y.double() == outer(c), c, torch.where(y.double() == outer(rn_bf16(z_in - E_in)),
                                                           rn_bf16(z_in - E_in), rn_bf16(z_in + E_in)))
    _note(family, c, z_in.double(), torch.as_tensor(E_in, dtype=torch.float64, device=z_in.device).expand_as(z_in), tie)


def within(y, z, E, family, what=""):
    """An fp32 (or wider) output: |y - z| <= E elementwise; records the worst |y - z| / E."""
    y, z = y.double(), z.double()
    E = torch.as_tensor(E, dtype=torch.float64, device=z.device).expand_as(z)
    err = (y - z).abs()
    ok = err <= E * (1 + 2.0 ** -20)
    if not bool(ok.all()):
        i = int((~ok).flatten().nonzero()[0])
        raise AssertionError(f"{family} {what}: {int((~ok).sum())} / {ok.numel()} elements off; first at flat index {i}: "
                             f"y={y.flatten()[i].item()!r} z={z.flatten()[i].item()!r} E={E.flatten()[i].item()!r}")
    note_ratio(family, float((err / E.clamp(min=1e-300)).max()) if err.numel() else 0.0)


def print_report(title):
    if REPORT:
        print(f"\n{title}: family, worst err/E, tie fraction")
        for k, (w, t, n) in sorted(REPORT.items()):
            print(f"  {k:24s} {w:8.4f}  {t / max(n, 1):.2e}  ({n} elements)")
    REPORT.clear()
