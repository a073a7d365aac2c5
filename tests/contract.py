"""The rule a kernel-contract test holds each launch to, and the record of the worst error each key of launches reached.

A launch meets its fp64 contract when its outputs are non-finite exactly where the reference's are, and elsewhere
|got - want| - allow <= BAR S + F: S is the sum of the magnitudes of every term of the element, F the engine's absolute
floor (conv_ref), `allow` the absolute error of an activation the element went through.  `errors` checks the first part
and measures the second; the caller holds the measure to its bar and records it in a `Worst`.
"""
import torch


def errors(got, want, s, allow=0.0, floor=None, bar=None, pre=None, what="launch"):
    """(err / S, err / (BAR S + F)) over the elements where the reference is finite, err = max(|got - want| - allow, 0);
    the second is None without a floor F.  S, F and allow broadcast to the elements.

    Requires got to be non-finite exactly where want is.  With `pre`, the reference's fp64 pre-activation, got may also
    be NaN where pre is non-finite: the tensor-core engines split an Inf into Inf and Inf - Inf, so their activation sees
    NaN where ELU / sigmoid of +-Inf is finite (wmd.h)."""
    got = got.double()
    bad, bad64 = ~torch.isfinite(got), ~torch.isfinite(want)
    extra = bad & ~bad64
    if pre is not None:
        extra &= ~(torch.isnan(got) & ~torch.isfinite(pre))
    assert not bool(extra.any()) and not bool((bad64 & ~bad).any()), \
        "%s: %d non-finite outputs where the reference has %d (%d differ)" % (
            what, int(bad.sum()), int(bad64.sum()), int((bad ^ bad64).sum()))
    d = ((got - want).abs() - allow).clamp(min=0)
    ok = (~bad & ~bad64).expand_as(d)
    d = d[ok]
    if not d.numel():
        return 0.0, None if floor is None else 0.0

    def at(t):
        return torch.as_tensor(t, dtype=torch.float64, device=d.device).expand_as(ok)[ok]
    s = at(s)
    e_s = float((d / s.clamp(min=1e-300)).max())
    return e_s, None if floor is None else float((d / (bar * s + at(floor))).max())


def _max(a, b):
    return b if a is None else (a if b is None else max(a, b))


class Worst(dict):
    """The worst error of each key of launches: key -> (worst err, worst err / (BAR S + F) or None, bar or None,
    launches, most rows or None).  err is err / S, or whatever unit the key's bar is in."""

    def __init__(self, fields):
        super().__init__()
        self.fields = fields            # what the key's parts are, for the report's heading

    def note(self, key, err, bound=None, bar=None, rows=None):
        worst, most, _, count, rows_was = self.get(key, (err, bound, bar, 0, rows))
        self[key] = (max(worst, err), _max(most, bound), bar, count + 1, _max(rows_was, rows))

    def lines(self):
        keys = sorted(self, key=lambda k: tuple(map(str, k)))
        widths = [max(len(str(k[i])) for k in keys) for i in range(len(keys[0]))] if keys else []
        out = ["worst per (%s): err, err / (BAR S + F)  (bar, launches, most rows)" % self.fields]
        for k in keys:
            worst, most, bar, count, rows = self[k]
            notes = ["bar " + ("-" if bar is None else "exact" if bar == 0 else "%.2g" % bar), "%d launches" % count]
            if rows is not None:
                notes.append("%d rows" % rows)
            out.append("  %s  %.2e  %-5s  (%s)" % ("  ".join(str(p).ljust(w) for p, w in zip(k, widths)), worst,
                                                   "-" if most is None else "%.3f" % most, ", ".join(notes)))
        return out

    def module_report(self):
        """The body of a test module's autouse fixture: records only that module's launches, and prints them when its
        last test ends."""
        self.clear()
        yield
        if self:
            print("\n" + "\n".join(self.lines()))
