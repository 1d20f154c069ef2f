"""What DalleEngine accepts, checked without a GPU.

dalle_engine.validate_geometry is the one rule the constructor applies to n_embd, n_heads, the sequence lengths and the
vocabulary sizes.  Here it is held against the dispatch facts of the CUDA sources, parsed from the text as
test_abi_coverage_cpu.py parses the header:
  * the `case` widths of both LayerNorm switches in csrc/rowops.cu (forward and backward) are LAYERNORM_WIDTHS;
  * every head-dim guard of csrc/attn.cu and csrc/decode.cu accepts exactly HEAD_DIMS;
  * sampling.FILTER_MAX_IDS is SF_SMEM_BYTES / 4 of csrc/decode.cu, the ids one filtered draw holds.
A width added to one switch alone, a head dim added to one guard, or a changed constant fails.  Then the accept /
refuse verdict of every geometry of the edge table tests/test_dalle_config_space_gpu.py runs, the sampler's filter
limit, and every shipped configs/dalle_*_b200.json.
"""
import glob
import json
import os
import re
from types import SimpleNamespace

import pytest

from dalle_mtf_b200 import lib as L
from dalle_mtf_b200.dalle_engine import HEAD_DIMS, LAYERNORM_WIDTHS, validate_geometry
from dalle_mtf_b200.sampling import FILTER_MAX_IDS, DalleSampler

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dalle_mtf_b200", "csrc")


def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _function_body(src, name):
    """The text of the C function `name` from its signature to its closing brace at column 0."""
    m = re.search(r"\b%s\s*\([^;]*?\)\s*\{" % re.escape(name), src)
    assert m, name
    end = src.index("\n}", m.end())
    return src[m.start():end]


def layernorm_switch_widths(rowops_src):
    """{entry point: sorted case widths} of the two LayerNorm dispatch switches."""
    out = {}
    for fn in ("db200_layernorm_fwd", "layernorm_bwd_impl"):   # db200_layernorm_bwd(_ex) dispatch through the latter
        body = _function_body(rowops_src, fn)
        sw = body[body.index("switch"):]
        out[fn] = sorted(int(c) for c in re.findall(r"\bcase\s+(\d+)\s*:", sw))
    return out


def head_dim_guards(src):
    """The set of head dims each head-dim guard of a source accepts: `dh == a || dh == b` requirements and
    `dh != a && dh != b` refusals."""
    guards = [set(map(int, re.findall(r"dh == (\d+)", g)))
              for g in re.findall(r"DB200_REQUIRE\(\s*(dh == \d+(?:\s*\|\|\s*dh == \d+)*)\s*,", src)]
    guards += [set(map(int, re.findall(r"dh != (\d+)", g)))
               for g in re.findall(r"if \((dh != \d+(?:\s*&&\s*dh != \d+)*)\)\s*return set_error", src)]
    return guards


def _const_int(src, name):
    """The value of `constexpr int NAME = <integer product>;` (a product of literals or of constants defined so)."""
    m = re.search(r"constexpr\s+int\s+%s\s*=\s*([^;]+);" % name, src)
    assert m, name
    value = 1
    for term in re.split(r"\s*\*\s*", m.group(1).strip()):
        value *= int(term) if term.isdigit() else _const_int(src, term)
    return value


def filtered_sampling_limit(decode_src):
    """SF_MAX_N, which decode.cu defines as SF_SMEM_BYTES / 4 (checked)."""
    m = re.search(r"constexpr\s+int\s+SF_MAX_N\s*=\s*SF_SMEM_BYTES\s*/\s*4\s*;", decode_src)
    assert m, "SF_MAX_N is no longer SF_SMEM_BYTES / 4"
    return _const_int(decode_src, "SF_SMEM_BYTES") // 4


# ------------------------------------------------------------------------------------------------ C dispatch facts
def test_layernorm_widths_are_the_cases_of_both_switches():
    widths = layernorm_switch_widths(_read("rowops.cu"))
    for fn, cases in widths.items():
        assert cases == sorted(LAYERNORM_WIDTHS), (fn, cases, LAYERNORM_WIDTHS)


def test_head_dims_are_what_every_attention_and_decode_guard_accepts():
    attn, decode = head_dim_guards(_read("attn.cu")), head_dim_guards(_read("decode.cu"))
    assert len(attn) >= 8 and len(decode) >= 1, (attn, decode)   # fwd / bwd of global, local, axial and conv; decode
    for g in attn + decode:
        assert g == set(HEAD_DIMS), g


def test_the_sampler_limit_is_the_filtered_kernels():
    assert FILTER_MAX_IDS == filtered_sampling_limit(_read("decode.cu")) == 51200


def test_the_parsers_see_a_width_added_to_one_switch():
    src = _read("rowops.cu")
    i = src.index("case 2048:", src.index("static int layernorm_bwd_impl("))
    widths = layernorm_switch_widths(src[:i] + "case 1536: break;\n    " + src[i:])
    assert 1536 in widths["layernorm_bwd_impl"] and 1536 not in widths["db200_layernorm_fwd"]
    guards = head_dim_guards('DB200_REQUIRE(dh == 64 || dh == 96 || dh == 128, E, "x");')
    assert guards == [{64, 96, 128}]
    assert _const_int("constexpr int A = 100 * 1024;\nconstexpr int B = A * 2;", "B") == 204800


# ------------------------------------------------------------------------------------------------ the edge table
# Accepted rows: name -> ((n_embd, n_layers, n_heads, text_vocab_size, image_vocab_size, text_seq_len, image_seq_len,
# batch), engine keywords).  tests/test_dalle_config_space_gpu.py runs each against float64 and through generation.
EDGE_ROWS = {
    # widths and head dims: LayerNorm with 1, 3 and 8 chunks per thread, the ping-pong GEMM at K = 768 (12 k-blocks),
    # the hand-off GEMM at K = 2048 (q|k|v) and K = 8192 (W2)
    "d256 h4": ((256, 2, 4, 300, 64, 24, 64, 2), {}),
    "d768 h12": ((768, 2, 12, 300, 64, 24, 64, 2), {}),
    "d768 h6": ((768, 2, 6, 300, 64, 24, 64, 2), {}),
    "d2048 h16 L1": ((2048, 1, 16, 300, 64, 24, 64, 1), {}),
    # text length: text_rows = 0 (an empty text block of the masked products, prefill at P = 1), short, odd
    "text_seq_len 1": ((256, 2, 2, 300, 64, 1, 64, 3), {}),
    "text_seq_len 8": ((256, 2, 2, 300, 64, 8, 64, 3), {}),
    "text_seq_len 127": ((256, 2, 2, 300, 64, 127, 64, 2), {}),
    # image length: ragged attention tiles, 1 x 1 and 2 x 2 grids for axial, conv and row / column positions
    "image_seq_len 1 grid 1x1": ((256, 2, 2, 300, 64, 24, 1, 3),
                                 {"types": ["axial_row", "conv"], "row_col": True}),
    "image_seq_len 4 grid 2x2": ((256, 2, 2, 300, 64, 24, 4, 3),
                                 {"types": ["axial_col", "conv"], "row_col": True}),
    "image_seq_len 63": ((256, 2, 2, 300, 64, 24, 63, 2), {}),
    "image_seq_len 64 local": ((256, 2, 2, 300, 64, 24, 64, 2), {"types": ["local", "global"]}),
    "image_seq_len 65 S 129": ((256, 2, 2, 300, 64, 64, 65, 2), {}),
    "S 385": ((256, 2, 2, 300, 64, 128, 257, 1), {}),
    # vocabulary: Vpad - V = 0 and 63, image_offset = 0 and 7 (mod 8), with and without per-position padding
    "V 384 offset 304": ((256, 2, 2, 304, 79, 24, 64, 2), {}),
    "V 385 offset 303": ((256, 2, 2, 303, 81, 24, 64, 2), {}),
    "per-position padding V 384 offset 303": ((256, 2, 2, 279, 80, 24, 64, 2), {"pp": True}),
    "per-position padding V 385 offset 304": ((256, 2, 2, 280, 80, 24, 64, 2), {"pp": True}),
    "image_vocab_size 1": ((256, 2, 2, 300, 1, 24, 64, 2), {}),
    "image_vocab_size 2": ((256, 2, 2, 300, 2, 24, 64, 2), {}),
    # mask descriptors at their extremes
    "local radius 1": ((256, 2, 2, 300, 64, 24, 64, 2), {"types": ["local", "global"], "radius": 1}),
    "local radius > S": ((256, 2, 2, 300, 64, 24, 64, 2), {"types": ["local", "global"], "radius": 1000}),
    "conv kernel 1": ((256, 2, 2, 300, 64, 24, 64, 2), {"types": ["conv", "axial_row"], "kernel": 1}),
    "conv kernel 11 on 8x8": ((256, 2, 2, 300, 64, 24, 64, 2), {"types": ["conv", "axial_col"], "kernel": 11}),
}
# (n_embd, n_heads, text_seq_len, image_seq_len, text_vocab_size, image_vocab_size) -> the exception the constructor
# raises; the GPU module builds each through DalleEngine and dalle_model_fn
EDGE_REFUSED = {
    "n_embd 1280": ((1280, 10, 24, 64, 300, 64), L.DB200Error),
    "n_embd 1536": ((1536, 12, 24, 64, 300, 64), L.DB200Error),
    "n_embd 3072": ((3072, 24, 24, 64, 300, 64), L.DB200Error),
    "n_embd 4352": ((4352, 34, 24, 64, 300, 64), L.DB200Error),
    "n_embd 384": ((384, 6, 24, 64, 300, 64), L.DB200Error),
    "n_embd 200": ((200, 2, 24, 64, 300, 64), L.DB200Error),
    "text_seq_len 0": ((256, 2, 0, 64, 300, 64), ValueError),
}
REFUSED = dict(EDGE_REFUSED, **{
    "head dim 32": ((256, 8, 24, 64, 300, 64), L.DB200Error),
    "head dim 256": ((512, 2, 24, 64, 300, 64), L.DB200Error),
    "n_heads does not divide n_embd": ((256, 3, 24, 64, 300, 64), ValueError),
    "image_seq_len 0": ((256, 2, 24, 0, 300, 64), ValueError),
    "image_vocab_size 0": ((256, 2, 24, 64, 300, 0), ValueError),
    "text_vocab_size 0": ((256, 2, 24, 64, 0, 64), ValueError),
    "n_heads 0": ((256, 0, 24, 64, 300, 64), ValueError),
    "text_seq_len 8.0": ((256, 2, 8.0, 64, 300, 64), ValueError),
    "image_seq_len True": ((256, 2, 24, True, 300, 64), ValueError),
})


@pytest.mark.parametrize("name", sorted(EDGE_ROWS))
def test_edge_rows_are_accepted(name):
    (d, nl, H, tv, iv, ts, isl, _), _ = EDGE_ROWS[name]
    assert validate_geometry(d, H, ts, isl, tv, iv, nl) == d // H


@pytest.mark.parametrize("geom", [(4096, 32, 256, 1024, 50258, 8192), (256, 4, 4, 4, 64, 51201),
                                  (256, 2, 8, 16, 1, 64)])
def test_other_edges_are_accepted(geom):
    assert validate_geometry(*geom) == geom[0] // geom[1]


@pytest.mark.parametrize("name", sorted(REFUSED))
def test_refused_geometries_name_the_knob(name):
    geom, exc = REFUSED[name]
    with pytest.raises(exc) as e:
        validate_geometry(*geom)
    if exc is L.DB200Error:   # a DB200Error is not a ValueError, so callers telling them apart keep working
        assert not isinstance(e.value, ValueError)
        assert ("LayerNorm" in str(e.value)) == (geom[0] not in LAYERNORM_WIDTHS)
        assert str(LAYERNORM_WIDTHS if geom[0] not in LAYERNORM_WIDTHS else HEAD_DIMS) in str(e.value)
    else:
        knob = name.split()[0]
        assert knob in str(e.value), (knob, str(e.value))


def test_every_layernorm_width_with_each_head_dim_is_accepted_and_nothing_between():
    for d in range(256, 4096 + 1, 256):
        for dh in HEAD_DIMS:
            if d in LAYERNORM_WIDTHS:
                assert validate_geometry(d, d // dh, 8, 16, 10, 10) == dh
            else:
                with pytest.raises(L.DB200Error, match="LayerNorm"):
                    validate_geometry(d, d // dh, 8, 16, 10, 10)


def _sampler(image_vocab_size):
    """A DalleSampler over a stand-in engine: argument validation reads nothing else."""
    return DalleSampler(SimpleNamespace(text_vocab_size=64, image_vocab_size=image_vocab_size))


def test_the_sampler_refuses_a_filter_past_the_limit_and_nothing_else():
    at, past = _sampler(FILTER_MAX_IDS), _sampler(FILTER_MAX_IDS + 1)
    assert at._filter(8, None) == (8, 1.0) and at._filter(None, 0.9) == (0, 0.9)
    for k, p in ((8, None), (None, 0.9), (8, 0.9), (FILTER_MAX_IDS, None)):
        with pytest.raises(ValueError, match="image_vocab_size"):
            past._filter(k, p)
    # no active filter: the unfiltered kernels run, which have no such limit
    assert past._filter(None, None) is None and past._filter(None, 1.0) is None
    assert past._filter(FILTER_MAX_IDS + 1, 1.0) is None


def test_every_shipped_configuration_is_accepted():
    from dalle_mtf_b200.model_fns import vae_grid_size
    from dalle_mtf_b200.utils import fetch_model_params
    paths = sorted(glob.glob(os.path.join(ROOT, "configs", "dalle_*_b200.json")))
    assert len(paths) >= 10
    for path in paths:
        with open(path) as f:
            p = json.load(f)
        W = vae_grid_size(fetch_model_params(p["vae_model"]), p["dataset"]["image_size"])
        validate_geometry(p["n_embd"], p["n_heads"], p["text_seq_len"], W * W, p["text_vocab_size"],
                          p["image_vocab_size"], p["n_layers"])
