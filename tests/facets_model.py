"""Executable restatement of the facets state of one batch (vlscan_facets): what a pipeFacetsProcessorShard holds after it saw the selected
rows of a batch with concurrency 1 (lib/logstorage/pipe_facets.go:162-307, hits_map.go:85-115).  Pure Python, for the CPU suite and as the
reference of the GPU differential, where `oracle_cells` reads the cells from the oracle's stored blocks.

A cell is what one block holds for one field:
  ("const", text)                the block's const value
  ("dict", entries, ids)         dictionary entries and the entry id of every row
  ("uint", numbers)              uint8..uint64 values of every row
  ("int", numbers)               int64 values of every row
  ("text", texts)                strings / float64 / ipv4 / iso8601 values as their texts (vlscan_gather_values)
  ("time", timestamps)           `_time` in nanoseconds
A field a block does not have has no cell.
"""
import datetime

U64, NEG, STR = 0, 1, 2
MAX_U64 = (1 << 64) - 1
DEFAULT_MAX_VALUES, DEFAULT_MAX_VALUE_LEN = 1000, 128


def try_parse_uint64(s):
    """tryParseUint64 (values_encoder.go:553-585) -> int or None"""
    if len(s) == 0 or len(s) > 26 or (len(s) > 1 and s[:1] == b"0"):
        return None
    n = 0
    for ch in s:
        if ch == 0x5F:
            continue
        if not 0x30 <= ch <= 0x39 or n > MAX_U64 // 10:
            return None
        n = n * 10 + ch - 0x30
        if n > MAX_U64:
            return None
    return n


def try_parse_int64(s):
    """tryParseInt64 (values_encoder.go:622-645) -> int or None"""
    neg = s[:1] == b"-"
    n = try_parse_uint64(s[1:] if neg else s)
    if n is None:
        return None
    if n >= 1 << 63:
        return -(1 << 63) if neg and n == 1 << 63 else None
    return -n if neg else n


def generic_key(text):
    """hitsMapAdaptive.updateStateGeneric: the (class, key) a text is counted under"""
    n = try_parse_uint64(text)
    if n is not None:
        return (U64, n)
    if text[:1] == b"-":
        v = try_parse_int64(text)
        if v is not None:
            return (NEG, v)
    return (STR, text)


def key_text(key):
    cls, k = key
    return k if cls == STR else str(k).encode()


def uint64_string_len(n):
    """uint64StringLen (pipe_facets.go:250-282): 20 for every n >= 10^10"""
    return len(str(n)) if n < 10 ** 10 else 20


def int64_string_len(n):
    if n >= 0:
        return uint64_string_len(n)
    return 21 if n == -(1 << 63) else 1 + uint64_string_len(-n)


def rfc3339_nano(ts):
    """marshalTimestampRFC3339NanoString in UTC"""
    secs, frac = divmod(ts, 10 ** 9)
    s = (datetime.datetime(1970, 1, 1) + datetime.timedelta(seconds=secs)).strftime("%Y-%m-%dT%H:%M:%S")
    return (s + ("." + ("%09d" % frac).rstrip("0") if frac else "") + "Z").encode()


class Shard:
    """pipeFacetsProcessorShard with concurrency 1, fed block by block"""

    def __init__(self, max_values_per_field=0, max_value_len=0):
        self.max_values = max_values_per_field or DEFAULT_MAX_VALUES
        self.max_len = max_value_len or DEFAULT_MAX_VALUE_LEN
        self.fields = {}
        self.rows = 0

    def block(self, cells, sel):
        """cells: {field: cell} of one block; sel: its selected rows (writeBlock skips a block without any)"""
        if not sel:
            return
        for name, cell in cells.items():
            self._column(name, cell, sel)
        self.rows += len(sel)

    def _column(self, name, cell, sel):   # updateFacetsForColumn
        f = self.fields.setdefault(name, {"ignore": False, "m": {}})
        if f["ignore"]:
            return
        if len(f["m"]) > self.max_values:
            self._ignore(f)
            return
        kind = cell[0]
        if kind == "const":
            self._generic(f, cell[1], len(sel))
        elif kind == "dict":
            hits = {}
            for r in sel:
                hits[cell[2][r]] = hits.get(cell[2][r], 0) + 1
            for i, v in enumerate(cell[1]):
                if hits.get(i):
                    self._generic(f, v, hits[i])
        elif kind == "uint":
            for r in sel:
                n = cell[1][r]
                if self.max_len <= 20 and uint64_string_len(n) > self.max_len:
                    self._ignore(f)
                    return
                self._add(f, (U64, n), 1)
        elif kind == "int":
            for r in sel:
                n = cell[1][r]
                if self.max_len <= 21 and int64_string_len(n) > self.max_len:
                    self._ignore(f)
                    return
                self._add(f, (U64, n) if n >= 0 else (NEG, n), 1)
        elif kind == "time":
            for r in sel:
                self._generic(f, rfc3339_nano(cell[1][r]), 1)
        else:
            for r in sel:
                self._generic(f, cell[1][r], 1)

    def _ignore(self, f):
        f["m"].clear()
        f["ignore"] = True

    def _generic(self, f, text, hits):   # updateStateGeneric
        if f["ignore"] or len(text) == 0:
            return
        if len(text) > self.max_len:
            self._ignore(f)
            return
        self._add(f, generic_key(text), hits)

    @staticmethod
    def _add(f, key, hits):
        f["m"][key] = f["m"].get(key, 0) + hits

    def state(self, fields):
        """{field: None when dropped, else [(class, text, hits)] by hits descending, then text, then class} for the requested fields"""
        out = {}
        for name in fields:
            f = self.fields.get(name)
            if f is None:
                out[name] = []
            elif f["ignore"] or len(f["m"]) > self.max_values:
                out[name] = None
            else:
                ents = [(k[0], key_text(k), h) for k, h in f["m"].items()]
                out[name] = sorted(ents, key=lambda e: (-e[2], e[1], e[0]))
        return out


def oracle_cells(blk, fields, vloracle):
    """the cells of the requested fields of a vloracle.Block, decoded from its stored bytes ("" and "_msg" both name the message field)"""
    consts = dict(blk.consts)
    cols = {c.name: c for c in blk.columns}
    out = {}
    for name in fields:
        if name == "_time":
            data, mt, mn, _mx = blk.timestamps_block()
            out[name] = ("time", [int(x) for x in vloracle.unmarshal_timestamps(data, mt, mn, blk.rows)])
            continue
        stored = [n for n in ((b"_msg", b"") if name in ("", "_msg") else (name.encode(),)) if n in consts or n in cols]
        if not stored:
            continue
        if stored[0] in consts:
            out[name] = ("const", consts[stored[0]])
        else:
            c = cols[stored[0]]
            items = None
            for cap in (1 << 20, 64 << 20):
                try:
                    items = vloracle.unmarshal_strings_block(c.values_block, blk.rows, cap)
                    break
                except Exception:
                    if cap == 64 << 20:
                        raise
            if c.value_type == 2:
                out[name] = ("dict", list(c.dict), [it[0] for it in items])
            elif c.value_type in (3, 4, 5, 6):
                out[name] = ("uint", [int(vloracle.encoded_to_string(c.value_type, it)) for it in items])
            elif c.value_type == 10:
                out[name] = ("int", [int(vloracle.encoded_to_string(c.value_type, it)) for it in items])
            elif c.value_type == 1:
                out[name] = ("text", items)
            else:
                out[name] = ("text", [vloracle.encoded_to_string(c.value_type, it) for it in items])
    return out
