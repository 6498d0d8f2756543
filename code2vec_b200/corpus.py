"""Host mirror of the reference's corpus reader and code-vector writer over the C++ parser in
libc2v_b200.so (`c2v_corpus_*`, `c2v_write_code_vectors`; csrc/c2v_corpus.cpp).

  VocabReader / Vocab      model/dataset_reader.py:15-41, model/dataset.py:53-92 (small text files: plain Python, same
                           semantics -- first occurrence of a name wins, `@question` inserted at index 1 of the terminals)
  CorpusReader             DatasetReader (dataset_reader.py:44-128): same constructor arguments and attributes
                           (path_vocab, terminal_vocab, variable_indexes, label_vocab, QUESTION_TOKEN_*), but the items
                           stay as CSR arrays (`ids`, `ctx_offsets`, `contexts`, `item_labels`, aliases) -- the layout
                           DeviceCorpus uploads -- instead of one Python object per method.  The 80 M context lines of
                           top11 are parsed in C++; Python only normalises the UNIQUE label strings (Unicode lower()).
  write_code_vectors       main.py:393-423 (+ the header of main.py:227-228), one batched C++ call instead of a Python
                           str() per float; byte-identical output.
There is no pure-Python fallback: a missing library raises (the oracle in oracle/corpus_oracle.py is test-only).
"""
import ctypes
import re

import numpy as np

from . import _lib

QUESTION_TOKEN_INDEX = 1            # dataset_reader.py:11
QUESTION_TOKEN_NAME = "@question"   # dataset_reader.py:12

_REDUNDANT_SYMBOL_CHARS = re.compile(r"[_0-9]+")                                          # dataset.py:56
_METHOD_SUBTOKEN_SEPARATOR = re.compile(r"([a-z]+)([A-Z][a-z]+)|([A-Z][a-z]+)")         # dataset.py:57


class Vocab(object):
    """vocabulary (dataset.py:53-92): the first index given to a name wins, freq counts new names only"""

    def __init__(self):
        self.stoi, self.itos, self.itosubtokens, self.freq = {}, {}, {}, {}

    def append(self, name, index=None, subtokens=None):
        if name not in self.stoi:
            if index is None:
                index = len(self.stoi)
            if self.freq.get(index) is None:
                self.freq[index] = 0
            self.stoi[name] = index
            self.itos[index] = name
            if subtokens is not None:
                self.itosubtokens[index] = subtokens
            self.freq[index] += 1

    def get_freq_list(self):
        return [self.freq[i] for i in range(self.len())]

    def len(self):
        return len(self.stoi)

    @staticmethod
    def normalize_method_name(method_name):
        return _REDUNDANT_SYMBOL_CHARS.sub("", method_name)

    @staticmethod
    def get_method_subtokens(method_name):
        return [x.lower() for x in _METHOD_SUBTOKEN_SEPARATOR.split(method_name) if x is not None and x != ""]


class VocabReader(object):
    """`index\\tname` lines (dataset_reader.py:15-41); indices > 0 are shifted by the number of extra tokens"""

    def __init__(self, filename, extra_tokens=()):
        self.filename, self.extra_tokens = filename, list(extra_tokens)

    def read(self):
        vocab = Vocab()
        extra_size = len(self.extra_tokens)
        for name in self.extra_tokens:
            vocab.append(name, 1)                       # dataset_reader.py:25-27 (index stays 1)
        with open(self.filename, mode="r", encoding="utf-8") as f:
            for line in f.readlines():
                data = line.strip(" \r\n\t").split("\t")
                index = int(data[0])
                if index > 0:
                    index += extra_size
                vocab.append(data[1] if len(data) > 1 else "", index)
        return vocab


def _strings(blob, offsets):
    """list of str from a byte blob + [n+1] offsets"""
    off = offsets.tolist()
    return [blob[off[i]:off[i + 1]].decode("utf-8") for i in range(len(off) - 1)]


class ParsedCorpus:
    """The arrays the C++ parser produced (a thin owner of numpy copies; the C++ object is freed right away)."""

    def __init__(self, handle):
        lib = _lib.load()
        try:
            info = _lib.CorpusInfo()
            _lib.check(lib.c2v_corpus_get_info(handle, ctypes.byref(info)), "c2v_corpus_get_info")
            n, nc, na = info.n_items, info.n_contexts, info.n_aliases
            self.ids = np.empty(n, np.int64)
            self.ctx_offsets = np.empty(n + 1, np.int64)
            self.contexts = np.empty((nc, 3), np.int32)
            self.label_offsets = np.empty(n + 1, np.int64)
            label_blob = ctypes.create_string_buffer(max(1, info.label_bytes))
            self.has_label = np.empty(n, np.uint8)
            self.label_pos = np.empty(n, np.int32)
            self.alias_item_offsets = np.empty(n + 1, np.int64)
            self.alias_orig_offsets = np.empty(na + 1, np.int64)
            alias_blob = ctypes.create_string_buffer(max(1, info.alias_bytes))
            self.alias_name_offsets = np.empty(na + 1, np.int64)
            alias_name_blob = ctypes.create_string_buffer(max(1, info.alias_name_bytes))
            P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
            B = lambda b: ctypes.cast(b, ctypes.c_void_p)
            rc = lib.c2v_corpus_export(handle, P(self.ids), P(self.ctx_offsets), P(self.contexts), P(self.label_offsets),
                                       B(label_blob), P(self.has_label), P(self.label_pos), P(self.alias_item_offsets),
                                       P(self.alias_orig_offsets), B(alias_blob), P(self.alias_name_offsets),
                                       B(alias_name_blob))
            _lib.check(rc, "c2v_corpus_export")
            self.label_blob = label_blob.raw[:info.label_bytes]
            self.alias_blob = alias_blob.raw[:info.alias_bytes]
            self.alias_name_blob = alias_name_blob.raw[:info.alias_name_bytes]
            self.n_items, self.n_contexts, self.n_aliases = int(n), int(nc), int(na)
        finally:
            lib.c2v_corpus_free(handle)

    @classmethod
    def parse_files(cls, paths, question_shift=QUESTION_TOKEN_INDEX):
        lib = _lib.load()
        if isinstance(paths, (str, bytes)):
            paths = [paths]
        arr = (ctypes.c_char_p * len(paths))(*[p.encode() if isinstance(p, str) else p for p in paths])
        h = ctypes.c_void_p()
        _lib.check(lib.c2v_corpus_parse_files(arr, len(paths), int(question_shift), ctypes.byref(h)), "c2v_corpus_parse_files")
        return cls(h)

    @classmethod
    def parse_text(cls, text, question_shift=QUESTION_TOKEN_INDEX):
        lib = _lib.load()
        data = text.encode("utf-8") if isinstance(text, str) else bytes(text)
        h = ctypes.c_void_p()
        _lib.check(lib.c2v_corpus_parse_buffer(data, len(data), int(question_shift), ctypes.byref(h)), "c2v_corpus_parse_buffer")
        return cls(h)

    @classmethod
    def load_cache(cls, path):
        lib = _lib.load()
        h = ctypes.c_void_p()
        _lib.check(lib.c2v_corpus_load(path.encode(), ctypes.byref(h)), "c2v_corpus_load")
        return cls(h)

    @staticmethod
    def build_cache(paths, cache_path, question_shift=QUESTION_TOKEN_INDEX):
        """text -> binary cache without going through numpy (parse once, load fast afterwards)"""
        lib = _lib.load()
        if isinstance(paths, (str, bytes)):
            paths = [paths]
        arr = (ctypes.c_char_p * len(paths))(*[p.encode() if isinstance(p, str) else p for p in paths])
        h = ctypes.c_void_p()
        _lib.check(lib.c2v_corpus_parse_files(arr, len(paths), int(question_shift), ctypes.byref(h)), "c2v_corpus_parse_files")
        try:
            _lib.check(lib.c2v_corpus_save(h, cache_path.encode()), "c2v_corpus_save")
        finally:
            lib.c2v_corpus_free(h)


class CorpusReader(object):
    """DatasetReader (dataset_reader.py:44-128) with CSR items.

    Attributes shared with the reference: path_vocab, terminal_vocab, variable_indexes, shuffle_variable_indexes,
    QUESTION_TOKEN_NAME, QUESTION_TOKEN_INDEX, infer_method, infer_variable, label_vocab.
    Instead of `items` (a list of CodeData): n_items, ids [n], ctx_offsets [n+1], contexts [total,3] int32,
    labels [n] (raw), normalized_labels [n] (lower-cased normalised names), item_labels [n] int64 (label_vocab index,
    -1 when infer_method is off), aliases(i) -> dict alias -> normalised original name (CodeData.aliases)."""

    def __init__(self, corpus_path, path_index_path, terminal_index_path, infer_method=True, infer_variable=False,
                 shuffle_variable_indexes=False, cache_path=None):
        self.path_vocab = VocabReader(path_index_path).read()
        self.terminal_vocab = VocabReader(terminal_index_path, extra_tokens=[QUESTION_TOKEN_NAME]).read()
        stoi = self.terminal_vocab.stoi
        self.variable_indexes = [stoi[term] for term in stoi if term.startswith("@var_")]
        self.shuffle_variable_indexes = shuffle_variable_indexes
        self.QUESTION_TOKEN_NAME, self.QUESTION_TOKEN_INDEX = QUESTION_TOKEN_NAME, QUESTION_TOKEN_INDEX
        self.infer_method, self.infer_variable = infer_method, infer_variable
        self.label_vocab = Vocab()
        if cache_path is not None:
            import os
            if not os.path.exists(cache_path):
                ParsedCorpus.build_cache(corpus_path, cache_path)
            self._load(ParsedCorpus.load_cache(cache_path))
        else:
            self._load(ParsedCorpus.parse_files(corpus_path))

    def _load(self, pc):
        self.parsed = pc
        self.n_items = pc.n_items
        self.ids, self.ctx_offsets, self.contexts = pc.ids, pc.ctx_offsets, pc.contexts
        self.labels = _strings(pc.label_blob, pc.label_offsets)
        # normalise each distinct string once (dataset_reader.py:94-98, :120-122)
        norm_cache = {}

        def norm(s):
            r = norm_cache.get(s)
            if r is None:
                n = Vocab.normalize_method_name(s)
                r = norm_cache[s] = (n.lower(), Vocab.get_method_subtokens(n))
            return r

        self.alias_originals = _strings(pc.alias_blob, pc.alias_orig_offsets)
        self.alias_names = _strings(pc.alias_name_blob, pc.alias_name_offsets)
        self.alias_normalized = [norm(s)[0] for s in self.alias_originals]
        self.normalized_labels = [norm(s)[0] if h else None for s, h in zip(self.labels, pc.has_label.tolist())]
        # label vocabulary in line order (dataset_reader.py:99-100, :123-124)
        append = self.label_vocab.append
        a_off = pc.alias_item_offsets.tolist()
        lpos = pc.label_pos.tolist()
        has = pc.has_label.tolist()
        for i in range(self.n_items):
            lo, hi = a_off[i], a_off[i + 1]
            cut = lo + lpos[i] if has[i] else hi
            if self.infer_variable:
                for k in range(lo, cut):
                    if self.alias_names[k].startswith("@var_"):
                        append(self.alias_normalized[k], subtokens=norm(self.alias_originals[k])[1])
            if self.infer_method and has[i]:
                append(self.normalized_labels[i], subtokens=norm(self.labels[i])[1])
            if self.infer_variable:
                for k in range(cut, hi):
                    if self.alias_names[k].startswith("@var_"):
                        append(self.alias_normalized[k], subtokens=norm(self.alias_originals[k])[1])
        stoi = self.label_vocab.stoi
        if self.infer_method:
            self.item_labels = np.asarray([stoi[n] if n is not None else -1 for n in self.normalized_labels], np.int64)
        else:
            self.item_labels = np.full(self.n_items, -1, np.int64)

    def aliases(self, i):
        """CodeData.aliases of item i: alias name -> normalised lower-cased original name (later lines overwrite)"""
        lo, hi = int(self.parsed.alias_item_offsets[i]), int(self.parsed.alias_item_offsets[i + 1])
        d = {}
        for k in range(lo, hi):
            d[self.alias_names[k]] = self.alias_normalized[k]
        return d

    def path_contexts(self, i):
        """CodeData.path_contexts of item i as an [n, 3] int32 view (start, path, end; already +QUESTION_TOKEN_INDEX)"""
        return self.contexts[int(self.ctx_offsets[i]):int(self.ctx_offsets[i + 1])]

    def variable_units(self, item_indices=None):
        """The bags of the variable-name task (dataset_builder.py:152-204): one unit per (item, `@var_*` alias) in the
        reference's order -> (unit_item int64 [U], unit_var_token int64 [U], unit_label int64 [U])."""
        tstoi, lstoi = self.terminal_vocab.stoi, self.label_vocab.stoi
        items = range(self.n_items) if item_indices is None else item_indices
        ui, uv, ul = [], [], []
        for pos, i in enumerate(items):
            al = self.aliases(int(i))
            for alias_name, normalized in al.items():
                if alias_name.startswith("@var_"):
                    ui.append(pos if item_indices is not None else int(i))
                    uv.append(tstoi[alias_name])
                    ul.append(lstoi[normalized])
        return np.asarray(ui, np.int64), np.asarray(uv, np.int64), np.asarray(ul, np.int64)


def read_code_vectors(vector_file, header="auto"):
    """The file write_code_vectors writes, read back -> (vectors float32 [n, H], names [n], header_items or None).
    header: "auto" (the first line is a header when it is two tab-separated integers), True or False.  A write followed
    by a read is bit-exact (every NaN reads back as a NaN)."""
    lib = _lib.load()
    mode = {"auto": -1, True: 1, False: 0}[header]
    h = ctypes.c_void_p()
    _lib.check(lib.c2v_read_code_vectors(str(vector_file).encode(), mode, ctypes.byref(h)), "c2v_read_code_vectors")
    try:
        info = _lib.VectorsInfo()
        _lib.check(lib.c2v_vectors_get_info(h, ctypes.byref(info)), "c2v_vectors_get_info")
        vec = np.empty((info.n, info.H), np.float32)
        offs = np.empty(info.n + 1, np.int64)
        blob = ctypes.create_string_buffer(max(1, info.name_bytes))
        _lib.check(lib.c2v_vectors_export(h, vec.ctypes.data_as(ctypes.c_void_p), offs.ctypes.data_as(ctypes.c_void_p),
                                          ctypes.cast(blob, ctypes.c_void_p)), "c2v_vectors_export")
        names = _strings(blob.raw[:info.name_bytes], offs)
        return vec, names, (None if info.header_items < 0 else int(info.header_items))
    finally:
        lib.c2v_vectors_free(h)


def write_code_vectors(vector_file, mode, code_vectors, labels, label_vocab, header_items=None, encode_size=None,
                       test_result_file=None, ids=None, pred_labels=None, pred_scores=None, result_mode="w"):
    """main.py:393-423 for a whole pass at once.  code_vectors: float32 [n, H] (torch CPU/CUDA tensor or ndarray),
    labels / pred_labels: int [n] into label_vocab (a Vocab or a list of names), pred_scores: float32 [n] (the max
    logit, main.py:411).  header_items: write the `n_items\\tencode_size` first line (main.py:227-228)."""
    lib = _lib.load()

    def host(a, dt):
        if hasattr(a, "detach"):
            a = a.detach().cpu().numpy()
        return np.ascontiguousarray(np.asarray(a), dtype=dt)

    vec = host(code_vectors, np.float32)
    if vec.ndim != 2:
        raise ValueError("code_vectors must be [n, H]")
    n, H = vec.shape
    if encode_size is not None and int(encode_size) != H:
        raise ValueError(f"encode_size {encode_size} != code_vectors.shape[1] {H}")
    lab = host(labels, np.int64)
    names = [label_vocab.itos[i] for i in range(label_vocab.len())] if isinstance(label_vocab, Vocab) else list(label_vocab)
    enc = [s.encode("utf-8") for s in names]
    offs = np.zeros(len(enc) + 1, np.int64)
    np.cumsum([len(b) for b in enc], out=offs[1:])
    blob = b"".join(enc)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p) if a is not None else None
    idv = host(ids, np.int64) if test_result_file is not None else None
    prl = host(pred_labels, np.int64) if test_result_file is not None else None
    prs = host(pred_scores, np.float32) if test_result_file is not None else None
    if lab.shape != (n,) or (prl is not None and (prl.shape != (n,) or prs.shape != (n,) or idv.shape != (n,))):
        raise ValueError("labels / ids / pred_labels / pred_scores must have one entry per code vector")
    rc = lib.c2v_write_code_vectors(str(vector_file).encode(), mode.encode(), -1 if header_items is None else int(header_items),
                                    n, H, P(vec), P(lab), ctypes.cast(ctypes.c_char_p(blob), ctypes.c_void_p), P(offs),
                                    len(enc), str(test_result_file).encode() if test_result_file is not None else None,
                                    result_mode.encode(), P(idv), P(prl), P(prs))
    _lib.check(rc, "c2v_write_code_vectors")
