"""ctypes front-end of the CPU oracle (oracle/b2t_oracle.c).  TEST INFRASTRUCTURE ONLY -- see the C file's header.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this module.
"""
import ctypes, json, os, re, subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liboracle.so")
_RANGES = os.path.join(_HERE, "..", "tokenizers_b200", "csrc", "unicode_ranges.inc")
_BERT = os.path.join(_HERE, "..", "tokenizers_b200", "csrc", "bert_tables.inc")   # per-character facts probed from the reference (tools/gen_bert_tables.py)

PT_GPT2, PT_LLAMA3, PT_WHITESPACE, PT_BYTELEVEL_NOREGEX, PT_BERT = 0, 1, 2, 3, 4
MODEL_BPE, MODEL_WORDPIECE = 0, 1
OFF_BYTE, OFF_CHAR = 0, 1

LLAMA3_PATTERN = (r"(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n]*"
                  r"|\s*[\r\n]+|\s+(?!\S)|\s+")


def build(force=False):
    src = os.path.join(_HERE, "b2t_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-s", "-C", _HERE, "-B", "liboracle.so"])
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(build())
        L.orc_create.restype = ctypes.c_void_p
        L.orc_create.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p, ctypes.c_uint32] + [ctypes.c_void_p] * 3 + \
            [ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_char_p,
             ctypes.c_uint32, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32]
        L.orc_destroy.argtypes = [ctypes.c_void_p]
        L.orc_encode_batch.restype = ctypes.c_int
        L.orc_encode_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_int]
        L.orc_encode_batch_norm.restype = ctypes.c_int
        L.orc_encode_batch_norm.argtypes = [ctypes.c_void_p] * 6 + [ctypes.c_uint32, ctypes.c_int]
        L.orc_n_tokens.restype = ctypes.c_uint64
        L.orc_n_tokens.argtypes = [ctypes.c_void_p]
        for f in ("orc_ids", "orc_offsets", "orc_word_ids", "orc_row_ptr"):
            getattr(L, f).restype = ctypes.c_void_p
            getattr(L, f).argtypes = [ctypes.c_void_p]
        L.orc_pretokenize.restype = ctypes.c_uint32
        L.orc_pretokenize.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint32]
        _lib = L
    return _lib


_tables = {}


def class_table(scheme):
    """0x110000-entry uint8 class table. scheme 'onig': 1=\\p{L} 2=\\p{N} 3=\\s 0=other; 'rust': 1=\\w 3=\\s 0=other."""
    if scheme not in _tables:
        txt = open(_RANGES).read()
        def ranges(name):
            body = re.search(r"%s\[\]\[2\] = \{(.*?)\};" % name, txt, re.S).group(1)
            return [(int(a, 16), int(b, 16)) for a, b in re.findall(r"\{0x([0-9A-F]+),0x([0-9A-F]+)\}", body)]
        t = np.zeros(0x110000, dtype=np.uint8)
        if scheme == "bert":   # BertPreTokenizer: 3 = whitespace (removed), 0 = punctuation (isolated), 1 = the rest
            bt = _bert_tables()
            t[:] = 1
            for a, b in bt["PUNCT"]:
                t[a:b + 1] = 0
            for a, b in bt["WS"]:
                t[a:b + 1] = 3
        elif scheme == "onig":
            for name, v in (("B2T_ONIG_L", 1), ("B2T_ONIG_N", 2), ("B2T_ONIG_S", 3)):
                for a, b in ranges(name):
                    t[a:b + 1] = v
        else:
            for name, v in (("B2T_RUST_W", 1), ("B2T_RUST_S", 3)):
                for a, b in ranges(name):
                    t[a:b + 1] = v
        _tables[scheme] = t
    return _tables[scheme]


_bert = None


def _bert_tables():
    """bert_tables.inc -> {"REMOVE" | "TOSPACE" | "CHINESE" | "MN" | "WS" | "PUNCT": [(lo, hi)], "NFD" | "LOWER": {cp: [cps]}}"""
    global _bert
    if _bert is None:
        txt = open(_BERT).read()
        out = {}
        for name in ("REMOVE", "TOSPACE", "CHINESE", "MN", "CCC", "WS", "PUNCT"):
            body = re.search(r"B2T_BERT_%s\[\]\[2\] = \{(.*?)\};" % name, txt, re.S).group(1)
            out[name] = [(int(a, 16), int(b, 16)) for a, b in re.findall(r"\{0x([0-9A-F]+),0x([0-9A-F]+)\}", body)]
        for name in ("NFD", "LOWER"):
            body = re.search(r"B2T_BERT_%s\[\] = \{(.*?)\};" % name, txt, re.S).group(1)
            flat = [int(x, 16) for x in re.findall(r"0x([0-9A-F]+)", body)]
            m, i = {}, 0
            while i < len(flat):
                m[flat[i]] = flat[i + 2:i + 2 + flat[i + 1]]
                i += 2 + flat[i + 1]
            out[name] = m
        _bert = out
    return _bert


class BertNormalizer:
    """normalizers/bert.rs:92-136 restated on code points, with the alignment bookkeeping of NormalizedString reduced to what
    the offsets need: every normalized character remembers the original character it came from (tokenizer/normalizer.rs:317-428:
    characters added by a step inherit the alignment of the character they came from, removed characters take theirs away)."""

    def __init__(self, clean_text=True, handle_chinese_chars=True, strip_accents=None, lowercase=True):
        self.clean, self.chinese, self.lower = bool(clean_text), bool(handle_chinese_chars), bool(lowercase)
        self.strip = self.lower if strip_accents is None else bool(strip_accents)   # bert.rs:128
        bt = _bert_tables()
        def member(rs):
            t = np.zeros(0x110000, dtype=bool)
            for a, b in rs:
                t[a:b + 1] = True
            return t
        self._remove, self._tospace, self._chin, self._mn = member(bt["REMOVE"]), member(bt["TOSPACE"]), member(bt["CHINESE"]), member(bt["MN"])
        self._ccc = member(bt["CCC"])
        self._nfd, self._low = bt["NFD"], bt["LOWER"]
        self._cache = {}

    def image(self, cp):
        r = self._cache.get(cp)
        if r is None:
            seq = [cp]
            if self.clean:
                if self._remove[cp]:
                    seq = []
                elif self._tospace[cp]:
                    seq = [0x20]
            if self.chinese:
                seq = [y for x in seq for y in ((0x20, x, 0x20) if self._chin[x] else (x,))]
            if self.strip:
                dec = []
                for x in seq:
                    if 0xAC00 <= x <= 0xD7A3:   # Hangul: L V [T]
                        si = x - 0xAC00
                        dec += [0x1100 + si // 588, 0x1161 + (si % 588) // 28] + ([0x11A7 + si % 28] if si % 28 else [])
                    else:
                        dec += self._nfd.get(x, [x])
                seq = [x for x in dec if not self._mn[x]]
            if self.lower:
                seq = [y for x in seq for y in self._low.get(x, [x])]
            r = self._cache[cp] = "".join(map(chr, seq)).encode("utf-8")
        return r

    def normalize(self, doc):
        """doc: bytes (valid UTF-8) -> (normalized bytes, uint32[len, 2]: original byte range of the character behind every byte)"""
        import unicodedata
        chars, pos = [], 0            # (code point, original byte range), step by step like the reference
        for ch in doc.decode("utf-8"):
            n = len(ch.encode("utf-8"))
            chars.append((ord(ch), pos, pos + n))
            pos += n
        if self.clean:
            chars = [(0x20 if self._tospace[c] else c, a, b) for c, a, b in chars if not self._remove[c]]
        if self.chinese:
            chars = [y for c, a, b in chars for y in (((0x20, a, b), (c, a, b), (0x20, a, b)) if self._chin[c] else ((c, a, b),))]
        if self.strip:
            dec = []                  # (code point, first piece of its character?)
            for c, a, b in chars:
                if 0xAC00 <= c <= 0xD7A3:
                    si = c - 0xAC00
                    seq = [0x1100 + si // 588, 0x1161 + (si % 588) // 28] + ([0x11A7 + si % 28] if si % 28 else [])
                else:
                    seq = self._nfd.get(c, [c])
                dec += [(x, k == 0) for k, x in enumerate(seq)]
            # canonical ordering (UAX #15): runs of characters with a non-zero combining class are sorted by class, stably;
            # which characters have one is probed from the reference, the class values (stable across Unicode versions) are Python's
            ccc = lambda x: unicodedata.combining(chr(x)) if self._ccc[x] else 0
            i = 0
            while i < len(dec):
                if ccc(dec[i][0]) == 0:
                    i += 1
                    continue
                j = i
                while j < len(dec) and ccc(dec[j][0]) != 0:
                    j += 1
                dec[i:j] = sorted(dec[i:j], key=lambda t: ccc(t[0]))
                i = j
            # NormalizedString::transform (normalizer.rs:347-412) hands the alignments out in the order it consumes the input, not
            # with the code points: a first piece takes the next input character's, any other piece the last consumed one's
            # ((0, 0) before the first).  A mark that sorting moved takes over another character's alignment.
            out, k = [], 0
            for x, first in dec:
                if first:
                    k += 1
                al = chars[k - 1][1:] if k else (0, 0)
                if not self._mn[x]:
                    out.append((x,) + al)
            chars = out
        if self.lower:
            chars = [(y, a, b) for c, a, b in chars for y in self._low.get(c, [c])]
        out, al = bytearray(), []
        for c, a, b in chars:
            e = chr(c).encode("utf-8")
            out += e
            al += [(a, b)] * len(e)
        return bytes(out), np.asarray(al, dtype=np.uint32).reshape(-1, 2)


def _pack(strings):
    bs = [s.encode("utf-8") for s in strings]
    off = np.zeros(len(bs) + 1, dtype=np.uint32)
    np.cumsum([len(b) for b in bs], out=off[1:])
    return np.frombuffer(b"".join(bs) + b"\0", dtype=np.uint8).copy(), off


def parse_config(js):
    """tokenizer.json dict -> dict(model, pretok, add_prefix_space, ignore_merges, ...) or raise ValueError."""
    m, pt = js["model"], js.get("pre_tokenizer")
    cfg = dict(add_prefix_space=0, ignore_merges=0, unk=None, prefix="", max_chars=100, merges=[])
    nz = js.get("normalizer")
    cfg["normalizer"] = None
    if nz is not None:
        if nz.get("type") != "BertNormalizer":
            raise ValueError("only BertNormalizer is restated")
        cfg["normalizer"] = dict(clean_text=nz.get("clean_text", True), handle_chinese_chars=nz.get("handle_chinese_chars", True),
                                 strip_accents=nz.get("strip_accents"), lowercase=nz.get("lowercase", True))
    if pt is None:
        raise ValueError("no pre_tokenizer")
    if pt["type"] == "ByteLevel":
        cfg["pretok"] = PT_GPT2 if pt.get("use_regex", True) else PT_BYTELEVEL_NOREGEX
        cfg["add_prefix_space"] = int(pt.get("add_prefix_space", True))
    elif pt["type"] == "Whitespace":
        cfg["pretok"] = PT_WHITESPACE
    elif pt["type"] == "BertPreTokenizer":
        cfg["pretok"] = PT_BERT
    elif pt["type"] == "Sequence":
        a, b = pt["pretokenizers"]
        ok = (a["type"] == "Split" and a["pattern"].get("Regex") == LLAMA3_PATTERN and a["behavior"] == "Isolated"
              and not a.get("invert", False) and b["type"] == "ByteLevel" and not b.get("use_regex", True)
              and not b.get("add_prefix_space", True))
        if not ok:
            raise ValueError("unsupported Sequence pre_tokenizer")
        cfg["pretok"] = PT_LLAMA3
    else:
        raise ValueError("unsupported pre_tokenizer " + pt["type"])
    if m["type"] == "BPE":
        cfg["model"] = MODEL_BPE
        if m.get("dropout") or m.get("unk_token") or m.get("continuing_subword_prefix") or m.get("end_of_word_suffix") \
                or m.get("byte_fallback") or cfg["pretok"] in (PT_WHITESPACE, PT_BERT) or cfg["normalizer"]:
            raise ValueError("unsupported BPE options")
        cfg["ignore_merges"] = int(m.get("ignore_merges", False))
        cfg["merges"] = [tuple(x.split(" ")) if isinstance(x, str) else tuple(x) for x in m["merges"]]
    elif m["type"] == "WordPiece":
        cfg["model"] = MODEL_WORDPIECE
        if cfg["pretok"] not in (PT_WHITESPACE, PT_BERT):
            raise ValueError("WordPiece is supported behind Whitespace / BertPreTokenizer only")
        cfg["unk"] = m["unk_token"]; cfg["prefix"] = m["continuing_subword_prefix"]; cfg["max_chars"] = m["max_input_chars_per_word"]
    else:
        raise ValueError("unsupported model " + m["type"])
    cfg["vocab"] = m["vocab"]
    return cfg


class Oracle:
    def __init__(self, tokenizer_json):
        js = json.loads(tokenizer_json) if isinstance(tokenizer_json, (str, bytes)) else tokenizer_json
        c = parse_config(js)
        self.cfg = c
        toks = list(c["vocab"].keys())
        self._vb, self._vo = _pack(toks)
        self._vi = np.array([c["vocab"][t] for t in toks], dtype=np.uint32)
        flat = [s for ab in c["merges"] for s in ab]
        self._mb, self._mo = _pack(flat)
        self._cls = class_table("bert" if c["pretok"] == PT_BERT else ("rust" if c["pretok"] == PT_WHITESPACE else "onig"))
        self._norm = BertNormalizer(**c["normalizer"]) if c["normalizer"] else None
        err = ctypes.create_string_buffer(256)
        unk = c["unk"].encode() if c["unk"] is not None else None
        pre = c["prefix"].encode()
        self._h = lib().orc_create(c["model"], c["pretok"], c["add_prefix_space"], c["ignore_merges"], self._cls.ctypes.data,
                                   len(toks), self._vb.ctypes.data, self._vo.ctypes.data, self._vi.ctypes.data,
                                   len(c["merges"]), self._mb.ctypes.data, self._mo.ctypes.data,
                                   unk, len(unk) if unk else 0, pre, len(pre), c["max_chars"], err, 256)
        if not self._h:
            raise ValueError(err.value.decode())

    def __del__(self):
        if getattr(self, "_h", None):
            lib().orc_destroy(self._h); self._h = None

    def encode_batch_csr(self, data, doc_off, offset_type=OFF_CHAR):
        """data: np.uint8[N]; doc_off: np.uint64[n+1] -> (ids u32[T], offsets u32[T,2], word_ids u32[T], row_ptr u64[n+1])."""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        doc_off = np.ascontiguousarray(doc_off, dtype=np.uint64)
        n = len(doc_off) - 1
        base = data.ctypes.data if data.size else 0
        if self._norm is not None:
            raw = data.tobytes()
            parts = [self._norm.normalize(raw[int(doc_off[d]):int(doc_off[d + 1])]) for d in range(n)]
            nb = np.frombuffer(b"".join(p[0] for p in parts) + b"\0", dtype=np.uint8).copy()
            noff = np.zeros(n + 1, dtype=np.uint64)
            if n:
                np.cumsum([len(p[0]) for p in parts], out=noff[1:])
            al = np.ascontiguousarray(np.concatenate([p[1] for p in parts] + [np.zeros((1, 2), dtype=np.uint32)]), dtype=np.uint32)
            rc = lib().orc_encode_batch_norm(self._h, base, doc_off.ctypes.data, nb.ctypes.data, noff.ctypes.data, al.ctypes.data, n, offset_type)
        else:
            rc = lib().orc_encode_batch(self._h, base, doc_off.ctypes.data, n, offset_type)
        if rc != 0:
            raise RuntimeError("oracle: encode failed (missing [UNK] token)")
        T = lib().orc_n_tokens(self._h)
        def view(ptr, count, dt):
            if count == 0:
                return np.zeros(0, dtype=dt)
            return np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_uint8)), shape=(count * np.dtype(dt).itemsize,)).view(dt).copy()
        ids = view(lib().orc_ids(self._h), T, np.uint32)
        offs = view(lib().orc_offsets(self._h), 2 * T, np.uint32).reshape(-1, 2)
        wid = view(lib().orc_word_ids(self._h), T, np.uint32)
        rp = view(lib().orc_row_ptr(self._h), n + 1, np.uint64)
        return ids, offs, wid, rp

    def encode_batch(self, docs, offset_type=OFF_CHAR):
        bs = [d.encode("utf-8") for d in docs]
        off = np.zeros(len(bs) + 1, dtype=np.uint64)
        if bs:
            np.cumsum([len(b) for b in bs], out=off[1:])
        data = np.frombuffer(b"".join(bs), dtype=np.uint8)
        return self.encode_batch_csr(data, off, offset_type)

    def pre_tokenize(self, doc):
        """[(start_byte, end_byte)] in original bytes, like pre_tokenize_str's offsets but in bytes."""
        return [tuple(s) for s in self.pre_tokenize_bytes(doc.encode("utf-8")).tolist()]

    def pre_tokenize_bytes(self, raw):
        """pre_tokenize of one document given as UTF-8 bytes -> np.uint32[k, 2] (for long documents)"""
        b = np.frombuffer(raw, dtype=np.uint8)
        out = np.zeros(2 * (len(b) + 2), dtype=np.uint32)
        k = lib().orc_pretokenize(self._h, b.ctypes.data if b.size else 0, len(b), out.ctypes.data, len(b) + 2)
        return out[:2 * k].reshape(-1, 2)


def dense_rows(ids, row_ptr, *, length, pad_to_multiple_of, max_length, pad_id, truncate_left, pad_left, pre, post):
    """TEST INFRASTRUCTURE.  Plain restatement of what the reference does to a batch of single sequences after the model:
    truncation to max_length - n_added_tokens (tokenizer/mod.rs:1272-1283, utils/truncation.rs:70-166: kept part only),
    the template `pre $A post` (processors/template.rs:646-) and pad_encodings (utils/padding.rs:50-81).
    -> (ids uint32[n, L], attention_mask uint8[n, L], lengths uint32[n]); raises if a row does not fit a fixed length."""
    n = len(row_ptr) - 1
    rows = []
    for d in range(n):
        seq = list(ids[int(row_ptr[d]):int(row_ptr[d + 1])])
        if max_length:
            keep = max_length - len(pre) - len(post)
            if len(seq) > keep:
                seq = seq[len(seq) - keep:] if truncate_left else seq[:keep]
        rows.append(list(pre) + seq + list(post))
    L = length if length else max((len(r) for r in rows), default=0)
    if pad_to_multiple_of and L % pad_to_multiple_of:
        L += pad_to_multiple_of - L % pad_to_multiple_of
    out = np.full((n, L), pad_id, dtype=np.uint32)
    mask = np.zeros((n, L), dtype=np.uint8)
    lens = np.zeros(n, dtype=np.uint32)
    for d, r in enumerate(rows):
        if len(r) > L:
            raise ValueError(f"row {d} has {len(r)} tokens, dense length is {L}")
        a = L - len(r) if pad_left else 0
        out[d, a:a + len(r)] = r
        mask[d, a:a + len(r)] = 1
        lens[d] = len(r)
    return out, mask, lens
