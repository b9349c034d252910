"""OBJ import on the device (csrc/nvc_obj.cuh / nvc_obj_load): loadObj over fast_obj, bit for bit.
The checkers are the reference's own loadObj output: obj_vertices.npz for kitten.obj and pirate.obj, and oracle/_ref/load_obj
(the reference's scene.cpp and fast_obj, built by oracle/refobj) for generated files.  End to end, kitten.obj through
nvc_obj_load -> nvc_cook_mesh_vertices -> nvc_cook_mesh_lods -> nvc_cook_meshlets -> nvc_scene_cache_write must give the
reference's kitten.z.cache byte for byte.  The CPU tier runs the product's kernels under the SIMT emulation (tests/emu_lib.py)
through the C ABI; the -m gpu tier runs them on the device."""
import ctypes
import lzma
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import emu_lib
import test_cook_vertices as cv
from niagara_b200.obj import ObjInfo, file_table, info_dict

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden")
LOAD_OBJ = os.path.join(ROOT, "oracle", "_ref", "load_obj")
needs_load_obj = pytest.mark.skipif(not os.path.exists(LOAD_OBJ), reason="needs the reference's loadObj (oracle/_ref/load_obj)")
OK, INVALID, UNSUPPORTED, CORRUPT = 0, -1, -6, -7
CANARY = 0xA5A5


KITTEN_OBJ = os.path.join(ROOT, "oracle", "_ref", "kitten.obj")
needs_kitten = pytest.mark.skipif(not os.path.exists(KITTEN_OBJ), reason="needs the reference's data/kitten.obj (oracle/_ref/kitten.obj)")


def golden(name):
    """pirate.obj is kept xz-compressed in tests/golden; kitten.obj (1.9 MB) is copied from the reference by oracle/refdata"""
    if name == "kitten.obj":
        with open(KITTEN_OBJ, "rb") as f:
            return f.read()
    with open(os.path.join(GOLDEN, name + ".xz"), "rb") as f:
        return lzma.decompress(f.read())


def fixture_records(name):
    with np.load(os.path.join(GOLDEN, "obj_vertices.npz")) as z:
        return np.ascontiguousarray(z[name + "_records"][z[name + "_corners"]])


def ref_load(blob):
    """loadObj's Vertex[] of one file, as (n, 8) uint16"""
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.obj"), os.path.join(d, "out.bin")
        with open(src, "wb") as f:
            f.write(blob)
        subprocess.run([LOAD_OBJ, src, dst], check=True)
        return np.fromfile(dst, np.uint16).reshape(-1, 8)


# ---- the product, emulated (host pointers) or on the device ---------------------------------------------------------------

class Emu:
    def __init__(self):
        self.lib = emu_lib.load()
        self.ctx = ctypes.c_void_p()
        assert self.lib.nvc_create(0, None, ctypes.byref(self.ctx)) == 0

    def close(self):
        self.lib.nvc_destroy(self.ctx)

    def load(self, blobs, capacity=None, query=False):
        """(status, Vertex[] (n, 8) uint16, infos); a refused call must leave `vertices` untouched"""
        table, keep = file_table(blobs)
        infos = (ObjInfo * max(len(blobs), 1))()
        st = self.lib.nvc_obj_load(self.ctx, None, table, len(blobs), None, 0, infos)
        if st != OK or query:
            return st, None, [info_dict(infos[k]) for k in range(len(blobs))]
        total = sum(int(infos[k].corner_count) for k in range(len(blobs)))
        cap = total if capacity is None else capacity
        out = np.full((cap + 1, 8), CANARY, np.uint16)
        st = self.lib.nvc_obj_load(self.ctx, None, table, len(blobs), out.ctypes.data, cap, infos)
        if st != OK:
            assert (out == CANARY).all(), "a refused call wrote its output"
            return st, None, [info_dict(infos[k]) for k in range(len(blobs))]
        assert (out[total:] == CANARY).all(), "write past the corners"
        return st, out[:total], [info_dict(infos[k]) for k in range(len(blobs))]


class Gpu:
    def __init__(self):
        import torch

        from niagara_b200.lib import load_library

        self.torch = torch
        self.lib = load_library()
        self.ctx = ctypes.c_void_p()
        assert self.lib.nvc_create(0, None, ctypes.byref(self.ctx)) == 0

    def close(self):
        self.lib.nvc_destroy(self.ctx)

    def load(self, blobs, stream=None):
        torch = self.torch
        table, keep = file_table(blobs)
        infos = (ObjInfo * max(len(blobs), 1))()
        s = stream.cuda_stream if stream is not None else None
        st = self.lib.nvc_obj_load(self.ctx, s, table, len(blobs), None, 0, infos)
        if st != OK:
            return st, None, [info_dict(infos[k]) for k in range(len(blobs))]
        total = sum(int(infos[k].corner_count) for k in range(len(blobs)))
        out = torch.full(((total + 1) * 8,), CANARY - 0x10000, dtype=torch.int16, device="cuda")
        st = self.lib.nvc_obj_load(self.ctx, s, table, len(blobs), out.data_ptr(), total, infos)
        torch.cuda.synchronize()
        got = out.cpu().numpy().view(np.uint16).reshape(-1, 8)
        assert (got[total:] == CANARY).all(), "write past the corners"
        return st, got[:total], [info_dict(infos[k]) for k in range(len(blobs))]


# ---- generated files ---------------------------------------------------------------------------------------------------------

def number(rng, special=False):
    """a token parse_float reads: plain, signed, exponents, odd forms"""
    r = rng.random()
    if special:
        return str(rng.choice(["1" * int(rng.integers(300, 330)), "9" * 400 + ".5", "0." + "1" * 400, "1" + "0" * 320 + "e25",
                               "1" * 320 + "." + "1" * 320, "-" + "7" * 330 + "e-3", "1e308e", "2" * 310 + "E19", "-" + "3" * 330 + "e20"]))
    if r < 0.35:
        return "%.6f" % rng.normal(0, 10)
    if r < 0.5:
        return "%de%s%d" % (rng.integers(-99, 99), rng.choice(["", "+", "-"]), rng.integers(0, 25))
    if r < 0.6:
        return "%.3fE%s%d" % (rng.normal(0, 3), rng.choice(["", "+", "-"]), rng.integers(0, 40))
    if r < 0.75:
        return str(rng.choice(["1.2.3", "-0", "+0.0", "-0.0", ".5", "5.", "1e", "1e-", "-", "+", "1e+", "7e4", "1e-7", "3e-8", "6.1e-5",
                               "65504", "65520", "70000", "-1e5", "1e38", "4e38", "1e-40", "1.4e-45", "abc", "0x10", "2e4294967297",
                               "1.5e4294967295", "123456789012345678901234567890", "00001.0000100"]))
    return "%.9g" % rng.uniform(-2, 2)


def index(rng, v, count, relative, big=False):
    """a reference to element v (1-based) of `count`: absolute, relative, or wrapped past 2^32"""
    if big:
        return str(v + (int(rng.integers(1, 200)) << 32)) if rng.random() < 0.5 else "-" + str(((int(rng.integers(1, 200)) << 32) - (count - v + 1)) % (1 << 40))
    return str(v - count - 1) if relative else str(v)


def gen_obj(rng, nl="\n", faces=True, big_indices=False, special=False):
    """a file the reference accepts: every face window in range, 3 to 12 vertices"""
    lines = []
    np_ = nt = nn = 0
    junk = ["# comment %d" % rng.integers(1e6), "o obj", "g group a", "s 1", "s off", "usemtl mat", "mtllib none.mtl", "vp 1 2 3", "x junk",
            "", "   ", "\t# tabbed", "v", "vn", "f", "f\t# no face here"]
    for _ in range(int(rng.integers(1, 60))):
        r = rng.random()
        lead = str(rng.choice(["", " ", "\t", " \t\r "]))
        sep = str(rng.choice([" ", "\t", "  ", " \r "]))
        if r < 0.25:
            k = int(rng.choice([3, 3, 3, 2, 1, 0, 4, 6]))
            lines.append(lead + "v" + sep + sep.join(number(rng, special) for _ in range(k)))
            np_ += 1
        elif r < 0.35:
            k = int(rng.choice([2, 2, 1, 3]))
            lines.append(lead + "vt" + str(rng.choice(["", " ", "\t"])) + sep.join(number(rng, special) for _ in range(k)))
            nt += 1
        elif r < 0.45:
            lines.append(lead + "vn" + str(rng.choice(["", " "])) + sep.join(number(rng, special) for _ in range(int(rng.choice([3, 3, 2])))))
            nn += 1
        elif r < 0.8 and faces and np_:
            n = int(rng.integers(3, 13)) if rng.random() < 0.5 else int(rng.choice([3, 4]))
            form = int(rng.integers(0, 4))
            toks = []
            for _ in range(n):
                rel = rng.random() < 0.3
                big = big_indices and rng.random() < 0.3
                v = index(rng, int(rng.integers(1, np_ + 1)), np_, rel, big)
                t = index(rng, int(rng.integers(0, nt + 1)) or 1, nt, rel) if nt else ""
                nv = index(rng, int(rng.integers(0, nn + 1)) or 1, nn, rel) if nn else ""
                if form == 0 or (not nt and not nn):
                    toks.append(v)
                elif form == 1 and nt:
                    toks.append(v + "/" + t)
                elif form == 2 and nn:
                    toks.append(v + "//" + nv)
                else:
                    toks.append(v + "/" + (t if nt else "") + "/" + (nv if nn else ""))
            if rng.random() < 0.1:
                # an orphan line: records pushed, then a 0 or junk ends it without a face
                toks.insert(int(rng.integers(1, len(toks))), str(rng.choice(["0", "x", "#c", "+1", "0/1"])))
            lines.append(lead + "f" + sep + sep.join(toks) + str(rng.choice(["", " ", "\r", "\t"])))
        elif r < 0.85 and faces and np_ > 2:
            # a forward reference: a later position, to be defined before the file ends
            lines.append("f %d %d %d" % (1, 2, np_ + 1))
            lines.append("v 1 2 3")
            np_ += 1
        else:
            lines.append(str(rng.choice(junk)))
    text = nl.join(lines)
    if rng.random() < 0.7:
        text += nl
    return text.encode()


def seeded_files(count, seed0=0):
    out = []
    for seed in range(seed0, seed0 + count):
        rng = np.random.default_rng(seed)
        k = seed % 6
        out.append(gen_obj(rng, nl="\r\n" if k == 1 else "\n", faces=k != 2, big_indices=k == 3))
    return out


def sized_file(size, seed, cut_line=None):
    """a valid file of exactly `size` bytes: faces over 3 positions, padded with comments; a line of `cut_line` bytes
    (no '\\n') in the middle when given"""
    rng = np.random.default_rng(seed)
    head = b"v 0 0 0\nv 1 0 0\nv 0 1 0\nvn 0 0 1\n"
    body = bytearray(head)
    mid = size // 2
    while len(body) < size - 40:
        if cut_line and len(body) >= mid:
            body += b"#" + b"x" * (cut_line - 1) + b"\n"
            cut_line = None
            continue
        if rng.random() < 0.5:
            body += b"f 1//1 2//1 3//1\n"
        else:
            body += b"# " + b"c" * int(rng.integers(0, 30000 if rng.random() < 0.1 else 60)) + b"\n"
    body = body[: size - 40] if len(body) > size - 40 else body
    body += b"v 3 3 3\n" + b"f 1 2 -1\n"
    body += b"#" * (size - len(body) - 1) + b"\n"
    assert len(body) == size
    return bytes(body)


BOUNDARY_FILES = {
    "65535": sized_file(65535, 1),
    "65536": sized_file(65536, 2),
    "65537": sized_file(65537, 3),
    "straddle": b"v 1 2 3\nv 4 5 6\nv 7 8 9\n" + b"#" * (65536 - 24 - 5) + b"\nf 1 2 3 1 2 3 1 2 3\n" + b"f 3 2 1\n" * 10,
    "long_line": sized_file(200000, 4, cut_line=140000),
    "long_line_last": b"v 1 2 3\nv 3 2 1\nv 0 0 1\nf 1 2 3\n" + b"#" * 140000,
    "no_final_newline": b"v 1 2 3\nv 3 2 1\nv 0 0 1\nf 1 2 3",
    "exact_block_open": b"v 1 2 3\nv 3 2 1\nv 0 0 1\n" + b"#" * (65536 - 24 - 10) + b"\nf 1 2 3 1",
    "nul": b"v 1 \x00 2\nv 3\x002 1\nv 0 0 1\n\x00f 1 2 3\nf 1 2 3\x00 1\nf 1 2 3 \x00\nf\x00 1 2 3\n",
    "no_faces": b"v 1 2 3\nvn 0 1 0\nvt 0.5 0.5\n# nothing else\n",
    "empty": b"",
    "newlines_only": b"\n\n\n",
    "orphans": b"v 1 2 3\nv 3 2 1\nv 0 0 1\nv 5 5 5\nf 1 2 x\nf 1 2 3\nf 1 2 3 +4\nf 4 3 2 1\nf 1 2 0\nf 2 3 4\n",
    "big_indices": b"v 1 2 3\nv 3 2 1\nv 0 0 1\nf 4294967297 8589934594 3\nf -4294967295 -12884901889 1\nf 12884901891 2 1\n",
    "relative_dummy": b"v 1 2 3\nv 3 2 1\nf -2 -1 1\nvn 0 0 1\nf 1//-2 2//-1 1//0\n",
}
assert len(BOUNDARY_FILES["exact_block_open"]) == 65536 and len(BOUNDARY_FILES["straddle"]) > 65536


def check_against_ref(load, blob, what):
    want = ref_load(blob)
    st, got, infos = load([blob])
    assert st == OK, (what, st)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert len(bad) == 0, (what, len(bad), bad[:4], got[bad[:4]], want[bad[:4]])
    assert infos[0]["corner_count"] == len(want)
    return got


# ---- CPU tier: emulated kernels ----------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def emu():
    e = Emu()
    yield e
    e.close()


@pytest.fixture(scope="module")
def emu_fixtures(emu):
    """one emulated call per fixture, made when a test first asks for it"""
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = emu.load([golden(name + ".obj")])
        return cache[name]

    return get


FIXTURES = [pytest.param("kitten", marks=needs_kitten), "pirate"]


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_emulated(emu_fixtures, name):
    st, got, infos = emu_fixtures(name)
    want = fixture_records(name)
    assert st == OK and got.shape == want.shape and np.array_equal(got, want), name
    i = infos[0]
    assert i["bytes_parsed"] == len(golden(name + ".obj")) and i["corner_offset"] == 0 and i["corner_count"] == len(want)
    if name == "kitten":
        assert (i["position_count"], i["texcoord_count"], i["normal_count"], i["face_count"]) == (14472, 0, 14851, 28944)
        assert i["index_count"] == 86832 and len(want) == 86832


def test_several_files_one_call_emulated(emu, emu_fixtures):
    blobs = [golden("pirate.obj"), BOUNDARY_FILES["orphans"], b"", golden("pirate.obj")]
    singles = [emu_fixtures("pirate")] + [emu.load([b]) for b in blobs[1:3]] + [emu_fixtures("pirate")]
    st, got, infos = emu.load(blobs)
    assert st == OK
    assert np.array_equal(got, np.concatenate([x[1] if x[1] is not None else np.zeros((0, 8), np.uint16) for x in singles]))
    offset = 0
    for a, x in zip(infos, singles):
        b = x[2][0]
        assert a["corner_offset"] == offset
        assert {k: y for k, y in a.items() if k != "corner_offset"} == {k: y for k, y in b.items() if k != "corner_offset"}
        offset += a["corner_count"]


@needs_kitten
def test_end_to_end_emulated(emu_fixtures, monkeypatch):
    """kitten.obj -> nvc_obj_load -> identity indices -> vertices -> LODs -> meshlets -> cache: kitten.z.cache"""
    v = emu_fixtures("kitten")[1]
    monkeypatch.setattr(cv, "obj_input", lambda name: (v, np.arange(len(v), dtype=np.uint32)))
    e = cv.Emu()
    try:
        got = cv.end_to_end_emulated(e, "kitten", False)
    finally:
        e.close()
    want = np.fromfile(os.path.join(GOLDEN, "kitten.z.cache"), np.uint8)
    assert len(got) == len(want) and np.array_equal(got, want)


@needs_load_obj
@pytest.mark.parametrize("seed0", range(0, 48, 8))
def test_seeded_emulated(emu, seed0):
    for k, blob in enumerate(seeded_files(8, seed0)):
        a = check_against_ref(emu.load, blob, seed0 + k)
        b = emu.load([blob])[1]
        assert np.array_equal(a, b), "two runs differ"


@needs_load_obj
@pytest.mark.parametrize("name", sorted(BOUNDARY_FILES))
def test_boundary_files_emulated(emu, name):
    blob = BOUNDARY_FILES[name]
    check_against_ref(emu.load, blob, name)
    st, _, infos = emu.load([blob], query=True)
    i = infos[0]
    if name in ("long_line", "long_line_last"):
        assert i["bytes_parsed"] < len(blob) and blob[i["bytes_parsed"] - 1: i["bytes_parsed"]] == b"\n"
    else:
        assert i["bytes_parsed"] == len(blob)


def test_boundary_file_counts_emulated(emu):
    _, _, infos = emu.load([BOUNDARY_FILES["orphans"]], query=True)
    # f 1 2 x: 2 orphans; f 1 2 3; f 1 2 3 +4: 3 orphans; f 4 3 2 1; f 1 2 0: 2 orphans; f 2 3 4
    assert infos[0]["face_count"] == 3 and infos[0]["index_count"] == 2 + 3 + 3 + 4 + 2 + 3
    _, _, infos = emu.load([b""], query=True)
    assert infos[0] == dict(bytes_parsed=0, position_count=0, texcoord_count=0, normal_count=0, face_count=0, index_count=0, corner_offset=0, corner_count=0)


REFUSED = {
    "face0": (b"v 1 2 3\nf \n", CORRUPT),
    "face1": (b"v 1 2 3\nf 1\n", CORRUPT),
    "face2": (b"v 1 2 3\nv 1 2 3\nf 1 2\n", CORRUPT),
    "position_past_end": (b"v 1 2 3\nv 1 2 3\nf 1 2 3\n", CORRUPT),
    "texcoord_past_end": (b"v 1 2 3\nv 1 2 3\nv 1 2 3\nvt 0 0\nf 1/2 2/1 3/1\n", CORRUPT),
    "normal_past_end": (b"v 1 2 3\nv 1 2 3\nv 1 2 3\nf 1//1 2//1 3//1\n", CORRUPT),
    "relative_before_start": (b"v 1 2 3\nv 1 2 3\nv 1 2 3\nf -1 -2 -5\n", CORRUPT),  # -4 would be the dummy
    "wrapped_past_end": (b"v 1 2 3\nv 1 2 3\nv 1 2 3\nf 1 2 4294967300\n", CORRUPT),
    "shifted_window": (b"v 1 2 3\nv 1 2 3\nv 1 2 3\nf 1 2 9 0\nf 1 2 3\n", CORRUPT),  # the face's window reads the orphans
}


@pytest.mark.parametrize("name", sorted(REFUSED))
def test_refusals_emulated(emu, name):
    blob, status = REFUSED[name]
    st, _, _ = emu.load([blob])
    assert st == status, (name, st)
    # with a valid file before it, the whole call is refused and nothing is written
    out = np.full((64, 8), CANARY, np.uint16)
    table, keep = file_table([b"v 1 2 3\nf 1 1 1\n", blob])
    infos = (ObjInfo * 2)()
    assert emu.lib.nvc_obj_load(emu.ctx, None, table, 2, out.ctypes.data, 63, infos) == status
    assert (out == CANARY).all()


def test_unread_orphans_are_not_checked_emulated(emu):
    # records past the last face window, and records of orphan lines no window covers, are never read
    st, got, _ = emu.load([b"v 1 2 3\nv 1 2 3\nv 1 2 3\nf 1 2 3\nf 7 8 9 x\n"])
    assert st == OK and len(got) == 3


def test_argument_refusals_emulated(emu):
    lib, ctx = emu.lib, emu.ctx
    blob = b"v 1 2 3\nf 1 1 1 1\n"
    table, keep = file_table([blob])
    infos = (ObjInfo * 1)()
    out = np.full((16, 8), CANARY, np.uint16)
    assert lib.nvc_obj_load(None, None, table, 1, out.ctypes.data, 6, infos) == INVALID
    assert lib.nvc_obj_load(ctx, None, None, 1, out.ctypes.data, 6, infos) == INVALID
    assert lib.nvc_obj_load(ctx, None, table, 1, out.ctypes.data, 6, None) == INVALID
    assert lib.nvc_obj_load(ctx, None, table, 1, out.ctypes.data + 8, 6, infos) == INVALID
    bad = (type(table[0]) * 1)()
    bad[0].data, bad[0].size = None, 5
    assert lib.nvc_obj_load(ctx, None, bad, 1, out.ctypes.data, 6, infos) == INVALID
    assert (out == CANARY).all()
    # over capacity: infos filled, nothing written
    assert lib.nvc_obj_load(ctx, None, table, 1, out.ctypes.data, 5, infos) == INVALID
    assert (out == CANARY).all() and infos[0].corner_count == 6 and infos[0].index_count == 4
    assert lib.nvc_obj_load(ctx, None, table, 0, out.ctypes.data, 0, infos) == OK
    assert lib.nvc_obj_load(ctx, None, table, 1, out.ctypes.data, 6, infos) == OK
    assert (out[6:] == CANARY).all() and not (out[:6] == CANARY).all()


HOSTILE = [
    b"f 1 2 3",
    b"v 1 2 3\nv 1 2 3\nv 1 2 3\nf 1 2 3 4",
    b"v 1 2 3\nv 1 2 3\nv 1 2 3\nf 1/1/1 2/",
    b"v 1 2 3\nv 1 2 3\nv 1 2 3\nf 1 2 3\nv 1.5e",
    b"v 1 2 3\nv 1 2 3\nv 1 2 3\nf 1 2 3\nvt 1.",
    b"v 1 2 3\nv 1 2 3\nv 1 2 3\nf 1 2 3\nvn -",
    b"v 1 2 3\nv 1 2 3\nv 1 2 3\nf 1 2 3\n" + b"7" * 5000,
    b"v",
    b"\t\r ",
    b"v 1 2 3\nv 1 2 3\nv 1 2 3\nf -1 -2 -3" + b"1" * 40,
]


def test_guarded_allocations_emulated():
    """hostile files, each cut at its last byte, on guarded allocations: no kernel reads past the call's bytes"""
    lib = emu_lib.load()
    ctx = ctypes.c_void_p()
    assert lib.nvc_create(0, None, ctypes.byref(ctx)) == 0
    lib.emu_guard_allocations(1)
    try:
        for blob in HOSTILE + [BOUNDARY_FILES["long_line_last"], BOUNDARY_FILES["exact_block_open"], REFUSED["shifted_window"][0]]:
            for k in range(1, len(blob) + 1) if len(blob) < 64 else (len(blob),):
                table, keep = file_table([blob[:k]])
                infos = (ObjInfo * 1)()
                st = lib.nvc_obj_load(ctx, None, table, 1, None, 0, infos)
                assert st in (OK, CORRUPT), (blob[:k], st)
                if st == OK and infos[0].corner_count:
                    out = np.zeros((int(infos[0].corner_count), 8), np.uint16)
                    assert lib.nvc_obj_load(ctx, None, table, 1, out.ctypes.data, len(out), infos) == OK
    finally:
        lib.emu_guard_allocations(0)
        lib.nvc_destroy(ctx)
        assert lib.emu_guarded_live() == 0


# ---- GPU tier ----------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def gpu():
    g = Gpu()
    yield g
    g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_gpu(gpu, name):
    st, got, infos = gpu.load([golden(name + ".obj")])
    assert st == OK and np.array_equal(got, fixture_records(name))


@pytest.mark.gpu
@needs_kitten
def test_end_to_end_gpu(gpu, monkeypatch):
    st, v, _ = gpu.load([golden("kitten.obj")])
    assert st == OK
    monkeypatch.setattr(cv, "obj_input", lambda name: (v, np.arange(len(v), dtype=np.uint32)))
    g = cv.Gpu()
    try:
        cv.test_end_to_end_gpu(g, "kitten.z.cache", "kitten", False)
    finally:
        g.close()


@pytest.mark.gpu
@needs_load_obj
def test_seeded_gpu(gpu):
    blobs = seeded_files(2000, 1000)
    for k, blob in enumerate(blobs):
        a = check_against_ref(gpu.load, blob, 1000 + k)
        if k % 10 == 0:
            assert np.array_equal(a, gpu.load([blob])[1]), "two runs differ"
    # all of them in one call: the concatenation, at the offsets the infos give
    st, got, infos = gpu.load(blobs[:200])
    assert st == OK
    for k in range(200):
        i = infos[k]
        assert np.array_equal(got[i["corner_offset"]: i["corner_offset"] + i["corner_count"]], ref_load(blobs[k]))


@pytest.mark.gpu
@needs_load_obj
@pytest.mark.parametrize("name", sorted(BOUNDARY_FILES))
def test_boundary_files_gpu(gpu, name):
    check_against_ref(gpu.load, BOUNDARY_FILES[name], name)


@pytest.mark.gpu
@needs_load_obj
def test_overflow_and_nan_gpu(gpu):
    """values that overflow to inf or give NaN: the NaN must be x86's, 0xffc00000, and quantise to 0xfe00"""
    nan_seen = 0
    for seed in range(200):
        rng = np.random.default_rng(50000 + seed)
        blob = gen_obj(rng, special=True)
        got = check_against_ref(gpu.load, blob, "special %d" % seed)
        nan_seen += int((got[:, :3] == 0xFE00).sum())
    assert nan_seen > 0


@pytest.mark.gpu
@needs_load_obj
def test_large_file_gpu(gpu):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import obj_load_bench

    blob = obj_load_bench.generate(40 << 20, seed=7)
    check_against_ref(gpu.load, blob, "40 MB generated file")


@pytest.mark.gpu
def test_busy_nonblocking_stream_gpu(gpu):
    import torch

    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        a = torch.randn(4096, 4096, device="cuda")
        for _ in range(8):
            a = a @ a.T / 4096
    st, got, _ = gpu.load([golden("pirate.obj"), golden("pirate.obj")], stream=s)
    torch.cuda.synchronize()
    assert st == OK and np.array_equal(got, np.concatenate([fixture_records("pirate"), fixture_records("pirate")]))
