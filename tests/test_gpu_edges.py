"""GPU (-m gpu): probes placed at chosen offsets from the places where the page kernels change code path or run out of
room, compared with the oracle in full (char and byte offsets).

Edges, relative to a 2 KB page: its start, the end of its first 32 B chunk, +256 B (BPE halo, LONG_PRETOK_MIN), +416 B
(WordPiece halo: 104 characters of 4 bytes), +1 KB (one K1 iteration); and the 1024-page block of the page and tile
scans (2 MiB).  Every page holds one probe whose start or end lies at edge + delta.  Two forms: the filler before a
probe is a document of its own (a document boundary at the probe) or text of the same document (the regex context
continues into the probe)."""
import json
import random
import numpy as np
import pytest
import helpers

pytestmark = pytest.mark.gpu

from tokenizers_b200 import Tokenizer, _lib  # noqa: E402
from oracle import oracle as orc  # noqa: E402
from helpers import PAGE, DELTAS, place, page_slots, check  # noqa: E402
from helpers import WIDE, BERT_PROBES, word, bpe_probes, wordpiece_probes, scan_block_slots  # noqa: E402


def wordpiece_json(max_chars):
    """the wordpiece asset with `max_input_chars_per_word` patched and the 4-byte letters of the probes (and their ##
    forms) added to the vocabulary: a word of them is then [UNK] only because of its length"""
    j = json.loads(helpers.asset_json("wordpiece"))
    j["model"]["max_input_chars_per_word"] = max_chars
    v = j["model"]["vocab"]
    nxt = max(v.values()) + 1
    for c in WIDE[4]:
        for t in (c, "##" + c):
            v[t], nxt = nxt, nxt + 1
    return json.dumps(j)


@pytest.mark.parametrize("form", ["doc", "text"])
@pytest.mark.parametrize("name", ["gpt2_style", "llama3_style"])
def test_bpe_probes_at_page_edges(name, form):
    check(helpers.pipeline_json(name), place(page_slots(bpe_probes()), form), f"{name} {form}")


@pytest.mark.parametrize("form", ["doc", "text"])
def test_bpe_probes_without_regex(form):
    probes = [p for p in bpe_probes() if len(p.encode()) >= 16 or not p]
    check(helpers.pipeline_json("gpt2_noregex"), place(page_slots(probes, DELTAS[::3]), form), f"noregex {form}", wcache=(True,))


@pytest.mark.parametrize("form", ["doc", "text"])
@pytest.mark.parametrize("max_chars", [100, 104])
def test_wordpiece_probes_at_page_edges(max_chars, form):
    check(wordpiece_json(max_chars), place(page_slots(wordpiece_probes(max_chars)), form), f"wordpiece max_chars={max_chars} {form}")


@pytest.mark.parametrize("name", ["gpt2_style", "llama3_style", "wordpiece"])
def test_probes_at_the_scan_block_edge(name):
    probes = (bpe_probes() if name != "wordpiece" else wordpiece_probes(100))
    sel = [probes[i] for i in range(0, len(probes), max(1, len(probes) // 8))][:8]
    for form in ("doc", "text"):
        check(wordpiece_json(100) if name == "wordpiece" else helpers.pipeline_json(name), place(scan_block_slots(sel), form), f"{name} 2 MiB {form}", wcache=(True,), byte_offsets=False)


@pytest.mark.parametrize("coords", ["input", "normalized"])
def test_bert_expanding_characters_at_page_edges(coords):
    """Hangul (three jamo with strip_accents), CJK (spaces around it), accents (stripped) straddling page edges of the
    input or of the normalized batch"""
    tj = helpers.pipeline_json("bert_uncased")
    nz = orc.BertNormalizer(**helpers.BERT_UNCASED)
    measure = (lambda s: len(s.encode("utf-8"))) if coords == "input" else (lambda s: len(nz.normalize(s.encode("utf-8"))[0]))
    for form in ("doc", "text"):
        check(tj, place(page_slots(BERT_PROBES, [-9, -3, -2, -1, 0, 1, 2, 3, 9]), form, measure), f"bert {coords} {form}",
              wcache=(True,), byte_offsets=False)


LONG_STARTS = [0, 1000, 2047]   # page offsets of a long word's first byte (a 417-byte split passes the halo only from 2047)


def long_word_slots(words):
    """each word at a document's start, after a space inside a document and at a document's end (the context is part of
    the probe), with its first byte at each of LONG_STARTS"""
    slots, k = [], 1
    for w in words:
        for ctx in ("{} tail", "head {} tail", "head {}"):
            for d in LONG_STARTS:
                slots.append((ctx.format(w), k * PAGE + d - ctx.index("{}"), "start"))
                k += 2 + len(w.encode()) // PAGE
    return slots


@pytest.mark.parametrize("name", ["gpt2_prefix", "wordpiece", "bert_uncased"])
def test_long_pretokens_at_document_edges(name):
    """BPE pre-tokens of more than 256 bytes, whose tokens come from the long pre-pass (with add_prefix_space the
    inserted space belongs to the one at a document's start), and WordPiece splits longer than the 416-byte halo ([UNK],
    characters counted past the halo)"""
    rng = random.Random(4)
    if name == "gpt2_prefix":
        words = [word(rng, n, w) for n in (257, 300, 2100) for w in (1, 2, 3)]
    else:
        words = [word(rng, n, w) for n in (417, 2100) for w in (1, 2, 4)]
    tj = wordpiece_json(100) if name == "wordpiece" else helpers.pipeline_json(name)
    check(tj, place(long_word_slots(words), "doc"), f"long words {name}", byte_offsets=name != "bert_uncased")


ADDED_SPANS = [(" " * k + "<mask>", "end") for k in (249, 250)] + [("<mask>" + " " * k, "start") for k in (0, 1)] + \
              [("[SEP2]" + " " * k, "start") for k in (249, 250)] + [(" " * k + "<both>" + " " * k, "start") for k in (124, 125)]


def test_added_token_spans_at_page_edges():
    """spans of 255 / 256 bytes after lstrip / rstrip (ADDED_MAX_SPAN), one starting on a page's last byte; 257 is refused"""
    tj = helpers.pipeline_json("added_gpt2_style")
    tok, ref = Tokenizer.from_str(tj), helpers.oracle_backed_tokenizer(tj)
    assert tok._dev_added
    for form in ("doc", "text"):
        slots, k = [], 1
        for probe, anchor in ADDED_SPANS:
            for e in (0, 256):
                for d in (-2, -1, 0, 1, 2):
                    slots.append(("x" + probe + "y" if form == "text" else probe, k * PAGE + e + d, anchor))
                    k += 1
        docs = place(slots, form)
        data, off = helpers.pack_docs(docs)
        for byte_offsets in (False, True):
            exp = helpers.host_added_csr(ref, data, off, byte_offsets)
            assert np.count_nonzero(exp[0] >> 31) >= len(slots)
            got = tok._engine_rows(data, off, _lib.WANT_OFFSETS | _lib.WANT_WORD_IDS | _lib.FLAG_ADDED_IDS | (_lib.OFFSETS_BYTES if byte_offsets else 0))
            helpers.assert_csr_equal(got, exp, docs, f"added spans {form} bytes={byte_offsets}")
    for over in (" " * 251 + "<mask>", "[SEP2]" + " " * 251, " " * 126 + "<both>" + " " * 125):
        docs = place([(over, PAGE - 1, "start")], "doc")
        with pytest.raises(_lib.B2TError) as ei:
            tok._engine_rows(*helpers.pack_docs(docs), _lib.WANT_OFFSETS | _lib.FLAG_ADDED_IDS)
        assert ei.value.code == _lib.B2T_ERR_UNSUPPORTED
        enc = tok.encode_batch(docs, add_special_tokens=False)   # and the tokenizer splits it on the host instead
        exp = ref.encode_batch(docs, add_special_tokens=False)
        assert [list(e.ids) for e in enc] == [list(e.ids) for e in exp]
