"""Every entry point declared in include/dalle_b200.h is exercised by the test suite, or is exempted here with a reason.

A db200_* symbol counts as tested when a tests/test_*.py names it as a whole word, or calls one of the
dalle_mtf_b200/ops.py wrappers that call it (found by walking each wrapper's syntax tree) as an attribute of the ops
module (`ops.colsum(...)`, with whatever name the test file binds the module to).  A new entry point without either
fails this test.
"""
import ast
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# entry points that compute nothing a test could compare, or that need more than one GPU
EXEMPT = {
    "db200_launch_count": "launch counter read by bench.py, no computation",
    "db200_device_check": "called by lib.require_device() before every GPU test",
}
EXEMPT.update({s: "collective of the data-parallel path (tests/test_dp_gpu.py runs it where 2 GPUs exist)" for s in (
    "db200_comm_load_nccl", "db200_comm_unique_id", "db200_comm_create", "db200_comm_destroy", "db200_comm_register",
    "db200_comm_info", "db200_bucket_allreduce_launch", "db200_bucket_reduce_scatter_launch",
    "db200_bucket_all_gather_launch", "db200_bucket_allreduce_wait")})

# entry points that tests reach through a package module rather than by name: (module calling it, test file that
# imports the module).  Both halves are checked below.
REACHED_THROUGH = {
    "db200_embed_fwd_at": ("sampling", "test_sampling_gpu.py"),
    "db200_embed_fwd_at_dev": ("sampling", "test_sampling_gpu.py"),
    "db200_attn_decode_dev": ("sampling", "test_sampling_gpu.py"),
    "db200_sample_rows_at": ("sampling", "test_sampling_gpu.py"),
    "db200_incr_i32": ("sampling", "test_sampling_gpu.py"),
    "db200_crc32c": ("tfrecord", "test_data_cpu.py"),
    "db200_tfrecord_masked_crc": ("tfrecord", "test_data_cpu.py"),
    "db200_tfrecord_frame": ("tfrecord", "test_data_cpu.py"),
    "db200_tfrecord_index": ("tfrecord", "test_data_cpu.py"),
}


def declared_symbols(header_text):
    return sorted(set(re.findall(r"\b(db200_[a-z0-9_]+)\s*\(", header_text)) - {"db200_stream_t"})


def wrappers_by_symbol(ops_source):
    """symbol -> names of the module-level functions of ops.py whose body mentions it (L.load().db200_x(...))."""
    out = {}
    for fn in ast.parse(ops_source).body:
        if isinstance(fn, ast.FunctionDef):
            for node in ast.walk(fn):
                if isinstance(node, ast.Attribute) and node.attr.startswith("db200_"):
                    out.setdefault(node.attr, set()).add(fn.name)
    return out


def ops_calls(test_source):
    """Names called as attributes of dalle_mtf_b200.ops in one test file (`ops.f(...)`, `o.f(...)` after
    `from dalle_mtf_b200 import ops as o`; a file that imports the module also gets the `ops` fixture name)."""
    tree = ast.parse(test_source)
    aliases = set()
    for node in ast.walk(tree):
        if isinstance(node, ast.ImportFrom) and node.module == "dalle_mtf_b200":
            aliases |= {a.asname or a.name for a in node.names if a.name == "ops"}
        elif isinstance(node, ast.Import):
            aliases |= {a.asname for a in node.names if a.name == "dalle_mtf_b200.ops" and a.asname}
    if aliases:
        aliases.add("ops")
    return {node.func.attr for node in ast.walk(tree)
            if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute)
            and isinstance(node.func.value, ast.Name) and node.func.value.id in aliases}


def untested(header_text, ops_source, test_sources):
    wrappers = wrappers_by_symbol(ops_source)
    called = set().union(*(ops_calls(src) for src in test_sources))
    missing = []
    for sym in declared_symbols(header_text):
        if sym in EXEMPT or sym in REACHED_THROUGH:
            continue
        if any(re.search(r"\b%s\b" % sym, src) for src in test_sources):
            continue
        if wrappers.get(sym, set()) & called:
            continue
        missing.append(sym)
    return missing


def _read(*parts):
    with open(os.path.join(ROOT, *parts)) as f:
        return f.read()


def _sources():
    tests = [_read("tests", os.path.basename(p)) for p in sorted(glob.glob(os.path.join(ROOT, "tests", "test_*.py")))
             if os.path.basename(p) != os.path.basename(__file__)]   # naming a symbol here is not testing it
    return _read("include", "dalle_b200.h"), _read("dalle_mtf_b200", "ops.py"), tests


def test_every_entry_point_is_tested_or_exempted():
    header, ops_source, tests = _sources()
    assert len(declared_symbols(header)) >= 60
    missing = untested(header, ops_source, tests)
    assert not missing, f"entry points of include/dalle_b200.h that no test calls (add a test or an exemption): {missing}"


def test_exemptions_name_declared_entry_points_and_hold():
    header, ops_source, _ = _sources()
    declared = set(declared_symbols(header))
    stale = sorted((set(EXEMPT) | set(REACHED_THROUGH)) - declared)
    assert not stale, f"exemptions for symbols the header no longer declares: {stale}"
    wrappers = wrappers_by_symbol(ops_source)
    for sym, (module, test_file) in REACHED_THROUGH.items():
        src = _read("dalle_mtf_b200", module + ".py")
        uses = re.search(r"\b%s\b" % sym, src) or any(re.search(r"\bops\.%s\(" % w, src) for w in wrappers.get(sym, ()))
        assert uses, f"{sym}: dalle_mtf_b200/{module}.py no longer calls it"
        test_src = _read("tests", test_file)
        assert re.search(r"dalle_mtf_b200(\.%s\b| import [\w, ]*\b%s\b)" % (module, module), test_src), \
            f"{sym}: tests/{test_file} does not import dalle_mtf_b200.{module}"


def test_a_new_entry_point_without_a_test_is_reported():
    header, ops_source, tests = _sources()
    header += "\nint db200_new_kernel(db200_stream_t stream, const float* x, int n);\n"
    assert untested(header, ops_source, tests) == ["db200_new_kernel"]
    # a longer symbol that contains it, or a bare call of a same-named function, does not count
    assert untested(header, ops_source, tests + ["L.load().db200_new_kernel_v2(s)\nnew_kernel(x)\n"]) == \
        ["db200_new_kernel"]
    ops_source += "\ndef new_kernel(x):\n    check(L.load().db200_new_kernel(stream_ptr(), ptr(x), 1), 'new')\n"
    assert untested(header, ops_source, tests + ["new_kernel(x)\n"]) == ["db200_new_kernel"]
    assert untested(header, ops_source, tests + ["from dalle_mtf_b200 import ops as o\no.new_kernel(x)\n"]) == []
