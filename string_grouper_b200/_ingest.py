"""Host side of the analyzer: pandas Series -> (uint8 bytes, int64 offsets) for the device vectoriser.

The device kernel (csrc/sg_tfidf.cu) implements the analyzer of the reference
(string_grouper/string_grouper.py:365-378) for ASCII text with
the default regex.  This module does what has to stay in Python:

  * validation (string_grouper.py:351-352, :988-995): every element must be a `str`;
  * zero-copy extraction of the Arrow offsets/data buffers of a pandas-3 `str` Series;
  * rows containing non-ASCII characters get `str.lower()` and
    `normalize('NFKD').encode('ASCII','ignore')` here, with the very same Python
    calls as string_grouper.py:372-375 (full Unicode semantics, length-changing);
  * a non-default `regex` is applied here with `re.sub` (string_grouper.py:376),
    the device then neither folds nor strips.
"""
import re
from unicodedata import normalize

import numpy as np
import pandas as pd
import pyarrow as pa

from ._lib import SG_FLAG_IGNORE_CASE, SG_FLAG_STRIP_DEFAULT, SG_LUT_UNKNOWN, SG_SYMBOL_UNKNOWN

DEFAULT_REGEX = r'[,-./]|\s'


def is_series_of_strings(series):
    """Same verdict as StringGrouper._is_series_of_strings (string_grouper.py:988-995), vectorised."""
    if not isinstance(series, pd.Series):
        return False
    if len(series) == 0:
        return True
    if series.dtype == object:
        return pd.api.types.infer_dtype(series, skipna=False) == "string"
    if isinstance(series.dtype, pd.StringDtype) or pd.api.types.is_string_dtype(series.dtype):
        return not bool(series.isna().any())
    return False


def _arrow_buffers(series):
    """(data uint8, offsets int64) of the UTF-8 encoding of `series`, zero-copy when Arrow-backed."""
    arr = pa.array(series, from_pandas=True)
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks() if arr.num_chunks != 1 else arr.chunk(0)
    if pa.types.is_null(arr.type) and len(arr) == 0:
        return np.zeros(0, np.uint8), np.zeros(1, np.int64)
    if not (pa.types.is_string(arr.type) or pa.types.is_large_string(arr.type)):
        if pa.types.is_string_view(arr.type):
            arr = arr.cast(pa.large_string())
        else:
            raise TypeError("input does not consist of strings only (arrow type %s)" % arr.type)
    if arr.null_count:
        raise TypeError("input contains missing values")
    n = len(arr)
    _, off_buf, data_buf = arr.buffers()
    odt = np.int64 if pa.types.is_large_string(arr.type) else np.int32
    offsets = np.frombuffer(off_buf, dtype=odt, count=n + 1, offset=arr.offset * np.dtype(odt).itemsize)
    offsets = offsets.astype(np.int64, copy=False)
    data = np.frombuffer(data_buf, dtype=np.uint8) if data_buf is not None else np.zeros(0, np.uint8)
    lo, hi = int(offsets[0]), int(offsets[-1])
    return data[lo:hi], (offsets - lo) if lo else offsets


def _encode_list(strings):
    arr = pa.array(strings, type=pa.large_string())
    _, off_buf, data_buf = arr.buffers()
    offsets = np.frombuffer(off_buf, dtype=np.int64, count=len(strings) + 1)
    data = np.frombuffer(data_buf, dtype=np.uint8) if data_buf is not None else np.zeros(0, np.uint8)
    return data[:int(offsets[-1])], offsets


def _has_non_ascii(series):
    data, _ = _arrow_buffers(series)
    return bool(data.size) and int(data.max()) >= 0x80


def _pack_code_points(series_list, regex, ignore_case):
    """normalize_to_ascii=False with non-ASCII text: the n-grams are windows of CODE POINTS (string_grouper.py:377-378
    on the un-normalised string).  Python's str.lower() and the regex (whose \\s also matches Unicode white space) run
    here, on every row; the device receives the cleaned text as uint32 code points, offsets count code points, and
    neither folds nor strips (flags = 0)."""
    pat = re.compile(regex)
    cps, lens = [], []
    for s in series_list:
        out = []
        for x in s.tolist():
            if ignore_case:
                x = x.lower()
            out.append(pat.sub('', x))
        lens.append(np.fromiter((len(x) for x in out), dtype=np.int64, count=len(out)))
        cps.append(np.frombuffer("".join(out).encode('utf-32-le', 'surrogatepass'), dtype=np.uint32))
    data = np.concatenate(cps) if len(cps) > 1 else cps[0]
    offsets = np.zeros(sum(len(x) for x in lens) + 1, dtype=np.int64)
    np.cumsum(np.concatenate(lens) if len(lens) > 1 else lens[0], out=offsets[1:])
    return np.ascontiguousarray(data), offsets, 0, False


def pack_strings(series_list, regex=DEFAULT_REGEX, ignore_case=True, normalize_to_ascii=True):
    """Concatenate the Series (master, then duplicates) into one symbol buffer for the device vectoriser.

    Returns (data, offsets int64 [n_total+1], flags for the device analyzer, pristine).  `data` is uint8 (ASCII
    bytes; `pristine` says that they are the callers' strings verbatim, so the device copy can also serve the string
    gather of get_matches) or, for text that keeps non-ASCII characters, uint32 code points (see _pack_code_points).
    """
    default_regex = (regex == DEFAULT_REGEX)
    if not normalize_to_ascii and any(_has_non_ascii(s) for s in series_list):
        return _pack_code_points(series_list, regex, ignore_case)
    flags = 0
    if default_regex:
        flags |= SG_FLAG_STRIP_DEFAULT
        if ignore_case:
            flags |= SG_FLAG_IGNORE_CASE
    datas, offs = [], []
    base = 0
    pristine = default_regex
    host_folded = []            # per Series: case folding already done here (rows of it went through str.lower())
    for s in series_list:
        data, offsets = _arrow_buffers(s)
        n = len(offsets) - 1
        mx = None               # largest byte of `data`; None = not known (after a re-encode)
        folded = False
        if not default_regex:
            # host runs the whole analyzer prefix (string_grouper.py:372-376) with the user's pattern
            pat = re.compile(regex)
            strings = s.tolist()
            out = []
            for x in strings:
                if ignore_case:
                    x = x.lower()
                if normalize_to_ascii:
                    x = normalize('NFKD', x).encode('ASCII', 'ignore').decode()
                out.append(pat.sub('', x))
            data, offsets = _encode_list(out)
        elif (mx := int(data.max()) if data.size else 0) >= 0x80:
            bad = np.unique(np.searchsorted(offsets, np.nonzero(data >= 0x80)[0], side='right') - 1)
            strings = s.tolist()
            for i in bad.tolist():
                x = strings[i]
                if ignore_case:
                    x = x.lower()
                if normalize_to_ascii:
                    x = normalize('NFKD', x).encode('ASCII', 'ignore').decode()
                strings[i] = x
            data, offsets = _encode_list(strings)
            if ignore_case:
                # str.lower() ran BEFORE NFKD (string_grouper.py:372-375), and NFKD can put capital ASCII back
                # ('\u2122' -> 'TM', '\u2116' -> 'No'): those rows must not be folded again.  Fold the untouched
                # (pure ASCII) rows here, byte-wise, and switch the device fold off for the whole call.
                data = data.copy()
                row_bad = np.zeros(n, dtype=bool)
                row_bad[bad] = True
                fold = (data >= 0x41) & (data <= 0x5a) & ~np.repeat(row_bad, np.diff(offsets))
                data[fold] |= 0x20
                folded = True
            pristine = False
            mx = None
        # one scan of the bytes in the common all-ASCII case: the maximum is only taken again after a re-encode
        if mx is None:
            mx = int(data.max()) if data.size else 0
        assert mx < 0x80, "host normalisation left non-ASCII bytes behind"
        datas.append(data)
        host_folded.append(folded)
        offs.append(offsets[:-1] + base if n else np.zeros(0, np.int64))
        base += int(offsets[-1])
    if any(host_folded):
        # one Series was folded on the host: fold the others the same way (ASCII bytes) and clear the device flag
        for k, done in enumerate(host_folded):
            if not done:
                d = datas[k].copy()
                up = (d >= 0x41) & (d <= 0x5a)
                d[up] |= 0x20
                datas[k] = d
        flags &= ~SG_FLAG_IGNORE_CASE
        pristine = False
    offs.append(np.array([base], dtype=np.int64))
    data = np.concatenate(datas) if len(datas) > 1 else np.ascontiguousarray(datas[0])
    offsets = np.concatenate(offs)
    return data, offsets, flags, pristine


def decode_vocab_keys(keys, ngram):
    """Packed 7-bit keys -> the n-gram strings (the sorted vocabulary of the fitted vectoriser)."""
    keys = np.asarray(keys, dtype=np.uint32)
    chars = [((keys >> (7 * (ngram - 1 - q))) & 0x7f).astype(np.uint8) for q in range(ngram)]
    mat = np.stack(chars, axis=1)
    return [bytes(row).decode('ascii') for row in mat]


def is_stripped(c):
    """The default regex class on ASCII, exactly like csrc/sg_tfidf.cu: , - . / and Python's ASCII \\s."""
    return (0x2c <= c <= 0x2f) or (0x09 <= c <= 0x0d) or (0x1c <= c <= 0x20)


def _byte_symbols(data, flags):
    """{byte present in `data`: its character after case folding} for the bytes the default regex does not delete"""
    hist = np.bincount(data, minlength=256) if data.size else np.zeros(256, dtype=np.int64)
    fold, strip = bool(flags & SG_FLAG_IGNORE_CASE), bool(flags & SG_FLAG_STRIP_DEFAULT)
    mapped = {}
    for c in np.nonzero(hist)[0].tolist():
        c2 = (c | 0x20) if (fold and 0x41 <= c <= 0x5a) else c
        if strip and is_stripped(c2):
            continue
        mapped[c] = c2
    return mapped


def byte_alphabet(data, flags):
    """Dense, order-preserving alphabet of the bytes that survive folding / stripping: (lut uint8[256] with 0xff =
    deleted, alphabet = array of the surviving code points in ascending order)."""
    mapped = _byte_symbols(data, flags)
    alphabet = np.array(sorted(set(mapped.values())), dtype=np.uint32)
    ids = {int(c): i for i, c in enumerate(alphabet.tolist())}
    lut = np.full(256, 0xff, dtype=np.uint8)
    for c, c2 in mapped.items():
        lut[c] = ids[c2]
    return lut, alphabet


def fitted_byte_lut(data, flags, alphabet):
    """lut uint8[256] of new bytes through a FITTED alphabet (K1 transform): the symbol id of the folded byte, 0xff =
    deleted, SG_LUT_UNKNOWN = a character the fitted alphabet does not hold."""
    lut = np.full(256, 0xff, dtype=np.uint8)
    for c, c2 in _byte_symbols(data, flags).items():
        i = int(np.searchsorted(alphabet, c2))
        lut[c] = i if i < len(alphabet) and int(alphabet[i]) == c2 else SG_LUT_UNKNOWN
    return lut


def fitted_symbol_ids(code_points, alphabet):
    """uint32 symbol ids of new code points through a FITTED alphabet (K1 transform); SG_SYMBOL_UNKNOWN where the
    alphabet does not hold the character (no nearest id: it would alias a real n-gram)."""
    code_points = np.asarray(code_points, dtype=np.uint32)
    if not len(alphabet):
        return np.full(len(code_points), SG_SYMBOL_UNKNOWN, dtype=np.uint32)
    ids = np.searchsorted(alphabet, code_points)
    found = alphabet[np.minimum(ids, len(alphabet) - 1)] == code_points
    return np.where(found, ids, SG_SYMBOL_UNKNOWN).astype(np.uint32)


def symbol_bits(n_symbols):
    return max(1, int(np.ceil(np.log2(max(int(n_symbols), 2)))))


def decode_vocab_keys64(keys, ngram, bits, alphabet):
    """64-bit keys over a dense alphabet -> the n-gram strings."""
    keys = np.asarray(keys, dtype=np.uint64)
    mask = np.uint64((1 << bits) - 1)
    cols = [alphabet[((keys >> np.uint64(bits * (ngram - 1 - q))) & mask).astype(np.int64)] for q in range(ngram)]
    mat = np.stack(cols, axis=1).astype(np.uint32)
    return [row.tobytes().decode('utf-32-le', 'surrogatepass') for row in mat]
