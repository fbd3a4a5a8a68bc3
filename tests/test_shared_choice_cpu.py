"""CPU tier of the shared-subscription choice (relations.cuh k_relations<true>, include/gpumqtt.h gm_relations_choose_device):
the key of the draw against two independent restatements, and the kernel, run on the CPU emulation (tests/native/emu/emu_choose.cpp), against a direct Python
model, topic by topic — also under AddressSanitizer + UBSan."""
import ctypes as C
import random
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import _shared_oracle as SO
import test_emu_kernels as T

ROOT = Path(__file__).resolve().parent.parent

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")

# an independent C++ restatement of the key (include/gpumqtt.h)
_KEY_CPP = r"""
#include <cstdint>
static uint64_t mix(uint64_t x) { x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull; x ^= x >> 27; x *= 0x94d049bb133111ebull; x ^= x >> 31; return x; }
extern "C" uint64_t ref_share_key(uint64_t seed, uint32_t row, uint32_t group, uint32_t occ, uint32_t ck) {
    return mix(mix(seed ^ (uint64_t(row) << 32 | group)) ^ (uint64_t(occ) << 32 | ck));
}
"""


class GmRel(C.Structure):                                   # include/gpumqtt.h gm_rel (24 bytes)
    _fields_ = [("node_id", C.c_uint64), ("client_key", C.c_uint32), ("id_idx", C.c_uint32), ("sub_id", C.c_uint32), ("flags", C.c_uint32)]


class GmSubRelation(C.Structure):
    _fields_ = [("node_id", C.c_uint64), ("handle", C.c_uint32), ("group", C.c_uint32), ("sub_ids_off", C.c_uint32), ("sub_ids_cnt", C.c_uint32)]


def _build(tmp, san: bool):
    """tests/native/emu/emu_choose.cpp with the real relations.cuh on the CPU emulation, built like test_emu_kernels._build."""
    out = tmp / ("libemu_choose_asan.so" if san else "libemu_choose.so")
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-DGM_CPU_EMU", f"-I{T.EMU}", f"-I{T.CSRC}", "-shared", "-fPIC", "-pthread", "-fno-omit-frame-pointer",
           *(["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined"] if san else []),
           "-Wl,--no-undefined", "-o", str(out), str(T.EMU / "emu_choose.cpp")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0 and "sanitize" in r.stderr and "cannot find" in r.stderr:
        pytest.skip("sanitizer runtime not installed")
    assert r.returncode == 0, r.stderr[-3000:]
    return out


def _emu_lib(tmp, san=False):
    lib = C.CDLL(str(_build(tmp, san=san)))
    lib.emu_relations_choose.restype = C.c_int32
    lib.emu_share_key.restype = C.c_uint64
    lib.emu_share_key.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]
    return lib


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return _emu_lib(tmp_path_factory.mktemp("emu_share"))


def test_share_key_restatements_agree(tmp_path, emu):
    """gm_share_key (the product library), the kernel's own function (emulator build), a C++ and a Python restatement agree."""
    from rmqtt_b200 import _native as N
    so = tmp_path / "libkeyref.so"
    (tmp_path / "k.cpp").write_text(_KEY_CPP)
    subprocess.check_call(["g++", "-O1", "-shared", "-fPIC", "-o", str(so), str(tmp_path / "k.cpp")])
    ref = C.CDLL(str(so))
    ref.ref_share_key.restype = C.c_uint64
    ref.ref_share_key.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]
    prod = N.lib().gm_share_key
    rng = random.Random(7)
    e64, e32 = [0, 2**32 - 1, 2**64 - 1], [0, 2**32 - 1]
    cases = [(s, r, g, o, k) for s in e64 for r in e32 for g in e32 for o in e32 for k in e32]
    while len(cases) < 10_000:
        cases.append((rng.choice(e64 + [rng.getrandbits(64)] * 3), *(rng.choice(e32 + [rng.getrandbits(32)] * 3) for _ in range(4))))
    for c in cases:
        want = SO.share_key(*c)
        assert prod(*c) == want and emu.emu_share_key(*c) == want and ref.ref_share_key(*c) == want, c
    assert SO.share_key(0, 0, 0, 0, 0) == SO.mix(SO.mix(0))


# ---- the kernel against a Python model -----------------------------------------------------------------------------------------
class Case:
    """Synthetic relation table, group table, online bitmap and match lists covering every rule of the choice."""

    def __init__(self, seed=11):
        rng = random.Random(seed)
        self.rng = rng
        self.rels = []                                      # dicts: node_id, client_key, id_idx, sub_id, flags
        self.groups = [(0, 0)]                              # group id -> (off, cnt); [0] unused
        self.members = []
        self.n_clients = 400

        def rel(live=True, v5=False, no_local=False, group=0, ck=None, id_idx=None, sub_id=None):
            ck = rng.randrange(self.n_clients) if ck is None else ck
            self.rels.append(dict(node_id=1 + ck % 3, client_key=ck, id_idx=ck if id_idx is None else id_idx,
                                  sub_id=rng.choice([0, 0, 3, 7, 9, 11]) if sub_id is None else sub_id,
                                  flags=(1 if live else 0) | (2 if v5 else 0) | (4 if no_local else 0) | (group << 8)))
            return len(self.rels) - 1

        self.direct = [rel(live=rng.random() < 0.9, v5=rng.random() < 0.6, no_local=rng.random() < 0.3) for _ in range(600)]
        # groups: sizes 1, 31, 32, 33, 1000, a few small ones; distinct client keys within a group
        self.group_sizes = [1, 31, 32, 33, 1000, 2, 5, 7, 3]
        for size in self.group_sizes:
            g = len(self.groups)
            cks = rng.sample(range(self.n_clients if size < 100 else self.n_clients * 4), size)     # unique within the group
            hs = [rel(live=rng.random() < 0.95, v5=rng.random() < 0.5, no_local=rng.random() < 0.3, group=g, ck=ck, id_idx=ck) for ck in cks]
            if size >= 31:
                hs[rng.randrange(1, size)] = len(self.rels) + 10**6   # an out-of-range handle in the block
            self.groups.append((len(self.members), size))
            self.members += hs
            # a live representative (the block's first entry) keeps the group reachable
            self.rels[self.members[self.groups[g][0]]]["flags"] |= 1
        # a group whose only member is a v5 no_local subscriber (the publisher of row 0 / 1)
        g = len(self.groups)
        self.solo = rel(v5=True, no_local=True, group=g, ck=5, id_idx=4242)
        self.groups.append((len(self.members), 1))
        self.members.append(self.solo)
        # an empty block, and a relation naming a group id past the table
        self.groups.append((len(self.members), 0))
        self.empty_g = len(self.groups) - 1
        self.bad_group = rel(group=len(self.groups) + 3)
        self.empty_member = rel(group=self.empty_g)
        self.n_groups = len(self.groups)
        # v5 relations of clients that are also v5 members of groups: merges
        self.merge = [rel(v5=True, ck=self.rels[h]["client_key"]) for h in self.members[:40] if h < len(self.rels)]
        self.reps = [self.members[off] for off, cnt in self.groups[1:] if cnt]
        # online bitmap: every third client key offline; group 2 (31 members) entirely offline
        nbits = self.n_clients * 4 + 64
        self.online_bits = nbits - 40                        # keys past it count as offline
        bits = np.zeros((nbits + 31) // 32, dtype=np.uint32)
        for k in range(nbits):
            if k % 3:
                bits[k >> 5] |= np.uint32(1 << (k & 31))
        off, cnt = self.groups[2]
        for h in self.members[off:off + cnt]:
            if h < len(self.rels):
                k = self.rels[h]["client_key"]
                bits[k >> 5] &= np.uint32(~(1 << (k & 31)) & 0xFFFFFFFF)
        self.online = bits

    def lists(self):
        rng, lists = self.rng, []
        nonrep = [h for h in self.members if h < len(self.rels) and h not in self.reps]
        for t in range(90):
            lst = [rng.choice(self.direct) for _ in range(rng.choice([0, 3, 20, 60]))]
            lst += rng.sample(self.reps, rng.randint(1, len(self.reps)))
            lst += rng.sample(nonrep, 30)                    # members that are not representatives: dropped
            lst += [rng.randint(0, len(self.rels) + 50) for _ in range(5)]   # dead and out-of-range handles
            lst += [self.bad_group, self.empty_member]
            if t % 3 == 0:
                lst += rng.sample(self.reps, 3)              # representatives appearing twice
            if t % 4 == 0:
                lst += self.merge
            if t < 2:
                lst = [self.solo] + lst[:10]
            if t == 5:                                       # more than 256 v5 relations, chosen ones among them
                lst += [h for h in self.direct if self.rels[h]["flags"] & 3 == 3] * 2 + self.merge
            rng.shuffle(lst)
            lists.append(lst)
        self.pubs = [4242 if t < 2 else self.rng.choice([0xFFFFFFFF, self.rng.randrange(self.n_clients)]) for t in range(len(lists))]
        return lists


def model(case, lists, seed, online):
    """Per row: sorted list of (node_id, handle, group field, sorted sub ids), and the expected status."""
    rels, n_rels = case.rels, len(case.rels)

    def is_online(ck):
        return online is None or (ck < case.online_bits and (int(online[ck >> 5]) >> (ck & 31)) & 1)

    out = []
    for t, lst in enumerate(lists):
        pub = case.pubs[t]
        direct, v5, seen = [], [], {}
        for h in lst:
            if h >= n_rels or not rels[h]["flags"] & 1:
                continue
            r = rels[h]
            g = r["flags"] >> 8
            if g:
                occ = seen.get(h, 0)
                seen[h] = occ + 1
                if g >= case.n_groups or case.groups[g][1] == 0 or case.members[case.groups[g][0]] != h:
                    continue
                off, cnt = case.groups[g]
                cands = []
                for m in case.members[off:off + cnt]:
                    if m >= n_rels or not rels[m]["flags"] & 1:
                        continue
                    rm = rels[m]
                    if rm["flags"] & 6 == 6 and pub != SO.NONE and rm["id_idx"] == pub:
                        continue
                    cands.append((rm["client_key"], is_online(rm["client_key"]), m))
                ch = SO.choose(cands, seed, t, g, occ)
                if ch is None:
                    continue
                m, on = ch
                gw = g | (0 if on else 0x80000000)
                if rels[m]["flags"] & 2:
                    v5.append((m, gw))
                else:
                    direct.append((rels[m]["node_id"], m, gw, ()))
                continue
            if r["flags"] & 6 == 6 and pub != SO.NONE and r["id_idx"] == pub:
                continue
            if r["flags"] & 2:
                v5.append((h, 0))
            else:
                direct.append((r["node_id"], h, 0, ()))
        if len(v5) > 256:
            out.append((sorted(direct + [(rels[h]["node_id"], h, gw, ()) for h, gw in v5]), 1))
            continue
        by_client = {}
        for h, gw in v5:
            by_client.setdefault(rels[h]["client_key"], []).append((h, gw))
        for hs in by_client.values():
            h, gw = min(hs)
            direct.append((rels[h]["node_id"], h, gw, tuple(sorted(rels[x]["sub_id"] for x, _ in hs if rels[x]["sub_id"]))))
        out.append((sorted(direct), 0))
    return out


def run_choice(lib, case, lists, seed, online, cap_rels=None):
    n = len(lists)
    table = (GmRel * len(case.rels))()
    for h, r in enumerate(case.rels):
        table[h].node_id, table[h].client_key, table[h].id_idx, table[h].sub_id, table[h].flags = r["node_id"], r["client_key"], r["id_idx"], r["sub_id"], r["flags"]
    groups = np.asarray(case.groups, dtype=np.uint32).reshape(-1, 2)
    members = np.asarray(case.members + [0], dtype=np.uint32)
    spans = np.zeros((n, 2), dtype=np.uint32)
    o = 0
    for i, l in enumerate(lists):
        spans[i] = (o, len(l))
        o += len(l)
    ids = np.asarray([h for l in lists for h in l] + [0], dtype=np.uint32)
    pubs = np.asarray(case.pubs, dtype=np.uint32)
    cap_r = len(ids) + 8 if cap_rels is None else cap_rels
    cap_s = len(ids) + 8
    out_spans = np.zeros((n, 2), dtype=np.uint32)
    out_rels = (GmSubRelation * max(cap_r, 1))()
    out_subs = np.zeros(cap_s, dtype=np.uint32)
    needed = np.zeros(3, dtype=np.uint64)
    status = np.zeros(n, dtype=np.int32)
    vp = lambda a: C.c_void_p(a.ctypes.data)   # noqa: E731
    rc = lib.emu_relations_choose(vp(spans), vp(ids), C.c_uint64(n), vp(pubs), table, C.c_uint64(len(case.rels)),
                                  vp(groups), C.c_uint32(case.n_groups), vp(members), None if online is None else vp(online),
                                  C.c_uint32(case.online_bits), C.c_uint64(seed), vp(out_spans), out_rels, C.c_uint64(cap_r),
                                  vp(out_subs), C.c_uint64(cap_s), vp(needed), vp(status))
    assert rc == 0
    got = []
    for t in range(n):
        off, cnt = int(out_spans[t, 0]), int(out_spans[t, 1])
        rows = []
        for k in range(cnt):
            sr = out_rels[off + k]
            rows.append((sr.node_id, sr.handle, sr.group, tuple(sorted(int(x) for x in out_subs[sr.sub_ids_off:sr.sub_ids_off + sr.sub_ids_cnt]))))
        got.append((sorted(rows), int(status[t])))
    return got, needed


def check_choice_kernel(lib):
    case = Case()
    lists = case.lists()
    for seed, online in ((1, case.online), (2**64 - 1, case.online), (12345, None)):
        got, needed = run_choice(lib, case, lists, seed, online)
        want = model(case, lists, seed, online)
        for t in range(len(lists)):
            assert got[t] == want[t], (seed, t)
        assert int(needed[0]) == sum(len(w[0]) for w in want)
        assert int(needed[1]) == sum(len(r[3]) for w in want if w[1] == 0 for r in w[0])
        # the cases the corpus must contain
        assert sum(w[1] for w in want) >= 1                                     # > 256 v5 relations incl. chosen ones
        assert want[0][0] == [r for r in want[0][0] if r[1] != case.solo]      # the no_local-only group chose nothing
        chosen = [r for w in want for r in w[0] if r[2]]
        assert any(r[2] & 0x80000000 for r in chosen) == (online is not None)
        assert any(r[3] and (r[2] & 0xFFFFFF) for r in chosen)                 # a chosen v5 member carrying sub ids
    return case


def test_choice_kernel_against_a_python_model(emu):
    """k_relations<true> on the emulator equals the model topic by topic: groups of 1 to 1000 members, representatives twice,
    dead / out-of-range handles and group ids, no_local (a group whose only member is the publisher), an offline group and a
    NULL bitmap, chosen v5 members merging with the same client's v5 relations, and the > 256 hand-over with status 1."""
    case = check_choice_kernel(emu)
    # every group size was chosen from at least once
    got, _ = run_choice(emu, case, case.lists(), 3, case.online)
    chosen_groups = {r[2] & 0xFFFFFF for rows, _ in got for r in rows if r[2]}
    assert set(range(1, len(case.group_sizes) + 1)) <= chosen_groups


def test_choice_kernel_capacity_protocol(emu):
    case = Case(seed=3)
    lists = case.lists()
    _, needed = run_choice(emu, case, lists, 9, case.online)
    need = int(needed[0])
    full, n2 = run_choice(emu, case, lists, 9, case.online, cap_rels=need)
    assert int(n2[0]) == need and full == [(sorted(w[0]), w[1]) for w in model(case, lists, 9, case.online)]
    _, n3 = run_choice(emu, case, lists, 9, case.online, cap_rels=need - 1)
    assert int(n3[0]) == need                     # the count of a short output is still exact: the caller grows and retries


def test_choice_kernel_under_asan_ubsan(tmp_path):
    so = _build(tmp_path, san=True)
    script = tmp_path / "run.py"
    script.write_text(f"""
import sys, ctypes as C
sys.path.insert(0, {str(ROOT)!r}); sys.path.insert(0, {str(ROOT / 'tests')!r})
import test_shared_choice_cpu as S
lib = C.CDLL({str(so)!r})
lib.emu_relations_choose.restype = C.c_int32
S.check_choice_kernel(lib)
print("asan run ok")
""")
    libasan = subprocess.run(["g++", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    env = {"PATH": "/usr/bin:/bin", "LD_PRELOAD": libasan, "ASAN_OPTIONS": "detect_leaks=0:detect_stack_use_after_return=0", "PYTHONPATH": str(ROOT)}
    import os
    for k in ("HOME", "LD_LIBRARY_PATH", "VIRTUAL_ENV"):
        if k in os.environ:
            env[k] = os.environ[k]
    run = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=1500, env=env)
    assert run.returncode == 0 and "asan run ok" in run.stdout, (run.stdout[-1500:], run.stderr[-4000:])
