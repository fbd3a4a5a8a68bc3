"""CPU tier: the C-ABI library loads and exports every symbol include/gpumqtt.h declares."""
import ctypes as C
import re
from pathlib import Path

import pytest
import torch

from rmqtt_b200 import _native as N

ROOT = Path(__file__).resolve().parent.parent


def _declared():
    src = (ROOT / "include" / "gpumqtt.h").read_text()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(gmr?_[a-z0-9_]+)\s*\(", src)))


def test_every_declared_symbol_is_exported_and_bound():
    names = _declared()
    assert len(names) >= 18
    lib = C.CDLL(str(N.LIB_PATH))
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/gpumqtt.h but not exported"
        assert n in N.SIGNATURES, f"{n} has no ctypes signature in rmqtt_b200/_native.py"
    assert set(N.SIGNATURES) <= set(names)


def test_version_and_shard_fn():
    lib = N.lib()
    assert b"sm_90a" in lib.gm_version()
    s = lib.gm_shard_of(b"reg-01/x", 8, 8)
    assert 0 <= s < 8
    assert lib.gm_shard_of(b"reg-01", 6, 8) == s            # only level 0 counts
    assert lib.gm_shard_of(b"+/x", 3, 8) == 0xFFFFFFFF       # root wildcards are replicated
    assert lib.gm_shard_of(b"#", 1, 8) == 0xFFFFFFFF


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-device error path")
def test_no_cpu_fallback_without_a_device():
    lib = N.lib()
    h = C.c_void_p()
    assert lib.gm_create(None, C.byref(h)) == N.GM_ERR_NO_DEVICE
    assert b"no CPU fallback" in lib.gm_last_error(None)


def test_error_codes_of_the_boundary_host_only():
    """Status codes instead of exceptions / aborts across the boundary (SURVEY §8b): bad arguments, invalid and too
    deep filters, matching on an engine without a device, unknown knobs — and a readable gm_last_error each time."""
    import numpy as np
    from rmqtt_b200.engine import Engine, GpuMqttError, pack
    lib = N.lib()
    eng = Engine(host_only=True, max_levels=4)
    h = eng._h
    ch = C.c_int32(0)
    assert lib.gm_sub_add(None, b"a", 1, 1, C.byref(ch)) == N.GM_ERR_INVALID_ARG
    assert lib.gm_sub_add(h, None, 3, 1, C.byref(ch)) == N.GM_ERR_INVALID_ARG
    assert lib.gm_sub_add(h, b"a/#/b", 5, 1, C.byref(ch)) == N.GM_ERR_INVALID_TOPIC and lib.gm_last_error(h)
    assert lib.gm_sub_add(h, b"a/b/c/d/e", 9, 1, C.byref(ch)) == N.GM_ERR_TOO_DEEP
    assert lib.gm_sub_add(h, b"a/b/c/d", 7, 1, C.byref(ch)) == N.GM_OK and ch.value == 1
    assert lib.gm_sub_add(h, b"a/b/c/d", 7, 1, C.byref(ch)) == N.GM_OK and ch.value == 0       # already present
    assert lib.gm_sub_remove(h, b"a/b/c/d", 7, 2, C.byref(ch)) == N.GM_OK and ch.value == 0    # other value
    assert lib.gm_sub_remove(h, b"x+", 2, 1, C.byref(ch)) == N.GM_ERR_INVALID_TOPIC
    had, old = C.c_int32(0), C.c_uint32(0)
    assert lib.gm_retain_set(h, b"a/+x", 4, 1, C.byref(had), C.byref(old)) == N.GM_ERR_INVALID_TOPIC
    assert lib.gm_retain_set(h, b"t/1", 3, 5, C.byref(had), C.byref(old)) == N.GM_OK and had.value == 0
    assert lib.gm_retain_set(h, b"t/1", 3, 6, C.byref(had), C.byref(old)) == N.GM_OK and (had.value, old.value) == (1, 5)
    assert lib.gm_retain_remove(h, b"t/2", 3, C.byref(had), C.byref(old)) == N.GM_OK and had.value == 0
    blob, offs = pack(["a/b"])
    spans, ids, status, needed = np.zeros((1, 2), np.uint32), np.zeros(8, np.uint32), np.zeros(1, np.int32), C.c_uint64(0)
    args = (blob.ctypes.data, offs.ctypes.data, 1, spans.ctypes.data, ids.ctypes.data, 8, C.byref(needed), status.ctypes.data)
    assert lib.gm_match_batch(h, *args) == N.GM_ERR_NO_DEVICE and b"no CPU fallback" in lib.gm_last_error(h)
    assert lib.gm_retain_match_batch(h, *args) == N.GM_ERR_NO_DEVICE
    assert lib.gm_match_batch(None, *args) == N.GM_ERR_INVALID_ARG
    assert lib.gm_debug_knob(h, b"no_such_knob", 1) == N.GM_ERR_INVALID_ARG and lib.gm_debug_knob(h, b"tile_chunk", 16) == N.GM_OK
    assert lib.gm_shard_of_batch(blob.ctypes.data, offs.ctypes.data, 1, 0, ids.ctypes.data) == N.GM_ERR_INVALID_ARG
    assert lib.gm_flush(h) == N.GM_OK and lib.gm_compact(h) == N.GM_OK
    with pytest.raises(GpuMqttError):
        eng.add("$SYS/a/$b", 1)                 # Metadata level below the root (topic.rs:357-359)


def test_publish_topic_decoder_matches_the_mqtt_fixed_header_layout():
    """gm_publish_topic: fixed header, remaining-length varint, u16-BE-prefixed topic (rmqtt-codec/src/v3/decode.rs:103-104,
    rmqtt-codec/src/v5/packet/publish.rs:27-28, utils.rs:142-155).  Pure host function: no GPU needed."""
    import ctypes as C
    from rmqtt_b200 import _native as N
    lib = N.lib()

    def varint(x):
        out = bytearray()
        while True:
            b = x & 0x7F
            x >>= 7
            out.append(b | (0x80 if x else 0))
            if not x:
                return bytes(out)

    def publish(topic: bytes, payload: bytes, qos=0, v5=False):
        var = len(topic).to_bytes(2, "big") + topic + (b"\x00\x07" if qos else b"") + (b"\x00" if v5 else b"") + payload
        return bytes([0x30 | (qos << 1)]) + varint(len(var)) + var

    for topic, payload, qos, v5 in ((b"a/b", b"x", 0, False), (b"reg-01/site-0001/dev-0000001/sen-1", b"p" * 300, 1, True), (b"", b"", 0, False), (b"t", b"z" * 20000, 2, False)):
        pkt = publish(topic, payload, qos, v5)
        tp, tl = C.c_char_p(), C.c_uint32(0)
        buf = (C.c_uint8 * len(pkt)).from_buffer_copy(pkt)
        assert lib.gm_publish_topic(buf, len(pkt), C.byref(tp), C.byref(tl)) == 0
        assert C.string_at(C.cast(tp, C.c_void_p).value, tl.value) == topic
    for bad in (b"\x10\x02\x00\x00", b"\x30", b"\x30\x05\x00\x09abc", b"\x30\xff\xff\xff\xff\x01"):
        buf = (C.c_uint8 * len(bad)).from_buffer_copy(bad)
        tp, tl = C.c_char_p(), C.c_uint32(0)
        assert lib.gm_publish_topic(buf, len(bad), C.byref(tp), C.byref(tl)) == N.GM_ERR_INVALID_ARG


def _split_params(s: str):
    s = s.strip()
    if s in ("", "void"):
        return []
    out, depth, cur = [], 0, ""
    for ch in s:
        if ch in "([":
            depth += 1
        elif ch in ")]":
            depth -= 1
        if ch == "," and depth == 0:
            out.append(cur.strip())
            cur = ""
        else:
            cur += ch
    if cur.strip():
        out.append(cur.strip())
    return out


def test_sys_crate_declares_every_function_of_the_header():
    """The Rust `-sys` crate under integration/ cannot be compiled here (no cargo): at least keep it mechanically in step with
    the header — every function present with the same number of parameters, every struct with the same number of fields."""
    hdr = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "gpumqtt.h").read_text(), flags=re.S)
    rs = re.sub(r"//[^\n]*", "", (ROOT / "integration" / "gpumqtt-sys" / "src" / "lib.rs").read_text())
    c_fns = {m.group(1): _split_params(m.group(2)) for m in re.finditer(r"\b(gmr?_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", hdr, flags=re.S)}
    r_fns = {m.group(1): _split_params(m.group(2)) for m in re.finditer(r"\bfn\s+(gmr?_[a-z0-9_]+)\s*\((.*?)\)\s*(?:->\s*[^;]+)?;", rs, flags=re.S)}
    assert set(c_fns) == set(_declared())
    assert sorted(set(c_fns) - set(r_fns)) == [], "declared in include/gpumqtt.h but missing from the sys crate"
    assert sorted(set(r_fns) - set(c_fns)) == [], "the sys crate declares functions the header does not have"
    for name, params in c_fns.items():
        assert len(params) == len(r_fns[name]), f"{name}: {len(params)} parameters in the header, {len(r_fns[name])} in the sys crate"
    # structs: `typedef struct X { ... } X;` with fields vs `pub struct X { pub a: T, ... }`
    c_structs = {}
    for m in re.finditer(r"typedef\s+struct\s+(gm_[a-z_]+)\s*\{(.*?)\}\s*\1\s*;", hdr, flags=re.S):
        n = 0
        for decl in m.group(2).split(";"):
            decl = decl.strip()
            if decl:
                n += len(_split_params(decl))                   # `uint64_t a, b` declares two fields
        c_structs[m.group(1)] = n
    r_structs = {m.group(1): len(re.findall(r"\bpub\s+(?:r#)?[a-z_0-9]+\s*:", m.group(2)))
                 for m in re.finditer(r"pub\s+struct\s+(gm_[a-z_]+)\s*\{(.*?)\n\}", rs, flags=re.S)}
    for name, n in c_structs.items():
        assert name in r_structs, f"struct {name} missing from the sys crate"
        assert r_structs[name] == n, f"struct {name}: {n} fields in the header, {r_structs[name]} in the sys crate"
