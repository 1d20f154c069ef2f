"""Launch census helpers shared by the modules that record an engine's kernel launches and require each recorded launch
class to be checked against float64 or exempted to a named test.

A launch class is a hashable descriptor: the entry point followed by sorted (field, value) pairs (`launch_class`).
`classify` sorts recorded classes into checked / exempt / unchecked and finds stale exemptions; it is pure Python so
that its matching logic is tested without a GPU (test_dalle_config_launches_cpu.py).  `OpsRecorder` wraps every public
function of dalle_mtf_b200.ops and hands each launch to a describe function.
"""
import inspect


def launch_class(entry, **fields):
    """(entry, (field, value), ...) with the fields sorted by name."""
    return (entry,) + tuple(sorted(fields.items()))


def fields(cls):
    """The field dict of a launch class."""
    return dict(cls[1:])


def exempt_keys(cls):
    """The EXEMPT keys a class answers to, most specific first: "entry:kind" (when the class has a kind) and "entry"."""
    f = fields(cls)
    return ([f"{cls[0]}:{f['kind']}"] if "kind" in f else []) + [cls[0]]


class Census:
    """Where each recorded class goes.  checkers: [(test name, predicate(cls) -> bool)] in priority order; a class is
    checked by the first present test whose predicate accepts it.  exempt: key (exempt_keys) -> (test id, reason) or
    (test id, reason, within), within(fields) -> bool the shapes the named test covers (a class outside them is not
    exempted).  present: names of the tests that exist in the module (a deleted replay test leaves its classes
    unchecked)."""

    def __init__(self, checkers, exempt, present):
        self.checkers, self.exempt, self.present = list(checkers), dict(exempt), set(present)

    def checker(self, cls):
        for name, pred in self.checkers:
            if name in self.present and pred(cls):
                return name
        return None

    def exemption(self, cls):
        for k in exempt_keys(cls):
            if k in self.exempt:
                v = self.exempt[k]
                return k if len(v) < 3 or v[2](fields(cls)) else None
        return None

    def classify(self, classes):
        """classes: iterable of launch classes.  Returns (checked {cls: test}, exempt {cls: key}, unchecked [cls],
        stale [key]): an exemption is stale when no recorded class answers to it."""
        checked, exempt, unchecked, used = {}, {}, [], set()
        for c in classes:
            name = self.checker(c)
            if name is not None:
                checked[c] = name
                continue
            k = self.exemption(c)
            if k is not None:
                exempt[c] = k
                used.add(k)
            else:
                unchecked.append(c)
        stale = sorted(set(self.exempt) - used)
        return checked, exempt, unchecked, stale


class OpsRecorder:
    """Context manager that wraps every public function of dalle_mtf_b200.ops.  A call at the outermost level (a
    wrapper calling another, as linear_wgrad calls gemm, counts once), or at any level for an entry in `nested`, is
    described by describe(entry, bound_arguments) -> (cls, info) or None (not recorded).  Unless the recorder is
    paused, cls is appended to `launches`; `info` keeps the info of each class's first launch and `tags` the set of
    values `tag` had at its launches (the caller sets `tag` to the phase it runs).  before(entry, args) /
    after(entry, args, state) run around each call."""

    def __init__(self, describe, nested=(), skip=(), before=None, after=None):
        self.describe, self.nested, self.skip = describe, set(nested), set(skip)
        self.before, self.after = before, after
        self.launches = []
        self.info = {}
        self.tags = {}
        self.tag = None
        self.paused = 0
        self._depth = 0

    def __enter__(self):
        import pytest
        from dalle_mtf_b200 import ops
        self._mp = pytest.MonkeyPatch()
        for name, fn in list(vars(ops).items()):
            if inspect.isfunction(fn) and fn.__module__ == ops.__name__ and not name.startswith("_") \
                    and name not in self.skip:
                self._mp.setattr(ops, name, self._wrap(name, fn))
        return self

    def __exit__(self, *exc):
        self._mp.undo()

    def classes(self):
        """The distinct recorded classes in first-launch order."""
        return list(dict.fromkeys(self.launches))

    def _wrap(self, entry, fn):
        sig = inspect.signature(fn)

        def call(*a, **k):
            if self._depth and entry not in self.nested:
                return fn(*a, **k)
            ba = sig.bind(*a, **k)
            ba.apply_defaults()
            A = dict(ba.arguments)
            if not self.paused:
                d = self.describe(entry, A)
                if d is not None:
                    cls, info = d
                    self.launches.append(cls)
                    self.info.setdefault(cls, info)
                    self.tags.setdefault(cls, set()).add(self.tag)
            state = self.before(entry, A) if self.before else None
            self._depth += 1
            try:
                out = fn(*a, **k)
            finally:
                self._depth -= 1
            if self.after:
                self.after(entry, A, state)
            return out
        return call
