"""Host side of building datasets from meshes (sonet_mesh_sample_f32, sonet_b200.meshes), no GPU: the
OBJ / OFF parsers on hand-written files, the C entry's argument validation, its export, declaration
and binding, the scratch-size arithmetic, the order of draw_host's draws, and save_npz files read
back by the reference's own ModelNet_Shrec_Loader."""
import ctypes
import os
import re
import types

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "sonet_mesh_sample_f32"
SIZE = "sonet_mesh_sample_scratch_bytes"
P_ = 256     # a non-null, 256-byte aligned placeholder pointer: validation fails before any read


def _write(tmp_path, name, text, crlf=False):
    p = tmp_path / name
    p.write_bytes(text.replace("\n", "\r\n" if crlf else "\n").encode())
    return str(p)


# ---- OBJ ------------------------------------------------------------------------------------------
OBJ = """# a square and a triangle, every token form
v 0 0 0
v 1 0 0
v 1 1 0   # trailing comment
v 0 1 0
vn 0 0 1
vt 0 0
f 1 2 3 4
f 1/1 2/1 3/1
f 1/1/1 3/1/1 4/1/1
f 1//1 2//1 4//1
v 0 0 2
f -1 -4 -3
o ignored
g ignored
s off
"""


@pytest.mark.parametrize("crlf", [False, True])
def test_read_obj_token_forms_fans_and_relative_indices(tmp_path, crlf):
    from sonet_b200 import meshes
    v, f = meshes.read_obj(_write(tmp_path, "a.obj", OBJ, crlf))
    assert v.dtype == np.float64 and f.dtype == np.int32
    assert np.array_equal(v, [[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [0, 0, 2]])
    # the quad as a fan (0,1,2), (0,2,3); then the three triangles; -1 is vertex 4, -4 is vertex 1
    assert np.array_equal(f, [[0, 1, 2], [0, 2, 3], [0, 1, 2], [0, 2, 3], [0, 1, 3], [4, 1, 2]])


def test_read_obj_pentagon_fan(tmp_path):
    from sonet_b200 import meshes
    txt = "".join("v %d %d 0\n" % (i, i * i) for i in range(5)) + "f 1 2 3 4 5\n"
    _, f = meshes.read_obj(_write(tmp_path, "p.obj", txt))
    assert np.array_equal(f, [[0, 1, 2], [0, 2, 3], [0, 3, 4]])


@pytest.mark.parametrize("face,msg", [("f 1 2 9", "outside"), ("f 1 2 -9", "outside"),
                                      ("f 0 1 2", "index 0"), ("f 1 2", "fewer than 3")])
def test_read_obj_bad_indices_raise(tmp_path, face, msg):
    from sonet_b200 import meshes
    with pytest.raises(ValueError, match=msg):
        meshes.read_obj(_write(tmp_path, "b.obj", "v 0 0 0\nv 1 0 0\nv 0 1 0\n" + face + "\n"))


# ---- OFF ------------------------------------------------------------------------------------------
OFF_BODY = """0 0 0
1 0 0
1 1 0
0 1 0
3 0 1 2
4 0 1 2 3
3 1 2 3 255 0 0
"""
WANT_OFF_F = [[0, 1, 2], [0, 1, 2], [0, 2, 3], [1, 2, 3]]


@pytest.mark.parametrize("header", ["OFF\n4 3 0\n", "OFF 4 3 0\n", "OFF4 3 0\n",
                                    "# comment\nOFF\n# counts next\n4 3 0\n"])
@pytest.mark.parametrize("crlf", [False, True])
def test_read_off_headers_comments_and_fans(tmp_path, header, crlf):
    from sonet_b200 import meshes
    v, f = meshes.read_off(_write(tmp_path, "a.off", header + OFF_BODY, crlf))
    assert np.array_equal(v, [[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]])
    assert np.array_equal(f, WANT_OFF_F) and f.dtype == np.int32


def test_read_off_modelnet_merged_header_large_counts(tmp_path):
    """ModelNet writes `OFF<nv> <nf> 0` on one line; counts of several digits."""
    from sonet_b200 import meshes
    nv = 1234
    rs = np.random.RandomState(0)
    v = rs.uniform(-1, 1, size=(nv, 3))
    f = rs.randint(0, nv, size=(56, 3))
    txt = "OFF%d %d 0\n" % (nv, len(f)) + "".join("%.17g %.17g %.17g\n" % tuple(r) for r in v) \
        + "".join("3 %d %d %d\n" % tuple(r) for r in f)
    gv, gf = meshes.read_off(_write(tmp_path, "m.off", txt))
    assert np.array_equal(gv, v) and np.array_equal(gf, f)


@pytest.mark.parametrize("text,msg", [
    ("OFF\n3 1 0\n0 0 0\n1 0 0\n0 1 0\n3 0 1 3\n", "outside"),
    ("OFF\n3 1 0\n0 0 0\n1 0 0\n0 1 0\n3 0 -1 2\n", "outside"),
    ("OFF\n3 2 0\n0 0 0\n1 0 0\n0 1 0\n3 0 1 2\n", "declared"),
    ("PLY\n", "not an OFF"),
    ("OFF\n3 1 0\n0 0 0\n1 0 0\n0 1 0\n2 0 1\n", "at least 3"),
])
def test_read_off_errors(tmp_path, text, msg):
    from sonet_b200 import meshes
    with pytest.raises(ValueError, match=msg):
        meshes.read_off(_write(tmp_path, "e.off", text))


# ---- the C entry ----------------------------------------------------------------------------------
def _call(lib, verts=P_, v_off=P_, total_V=10, faces=P_, f_off=P_, total_F=20, ids=P_, B=2, N=16,
          draws=None, seed=0, scratch=P_, scratch_bytes=1 << 40, out=P_, face=None, area=None):
    return lib.sonet_mesh_sample_f32(verts, v_off, total_V, faces, f_off, total_F, ids, B, N, draws,
                                     seed, scratch, scratch_bytes, out, face, area, None)


@pytest.mark.parametrize("kw,msg", [
    (dict(B=-1), "B=-1"), (dict(N=0), "N=0"), (dict(N=-3), "N=-3"),
    (dict(N=(1 << 24) + 1), "N=16777217"),
    (dict(total_F=-1), "total_F=-1"), (dict(total_F=(1 << 40) + 1), "total_F="),
    (dict(total_V=-1), "total_V=-1"), (dict(total_V=(1 << 40) + 1), "total_V="),
    (dict(v_off=None), "must not be null"), (dict(f_off=None), "must not be null"),
    (dict(ids=None), "must not be null"), (dict(scratch=None), "must not be null"),
    (dict(out=None), "must not be null"),
    (dict(verts=None), "verts must not be null"), (dict(faces=None), "faces must not be null"),
    (dict(scratch_bytes=0), "scratch of 0 bytes"),
    (dict(scratch=P_ + 8), "256-byte aligned"),
])
def test_bad_arguments_fail_before_any_cuda_call(lib_built, kw, msg):
    from sonet_b200 import _C
    lib = _C.lib()
    assert _call(lib, **kw) == -1
    assert msg in _C.last_error(), _C.last_error()


def test_edges_are_accepted_arguments(lib_built):
    """N at its limit, empty vertex / face arrays with null pointers, and B = 0 (which returns
    before any launch) pass validation."""
    from sonet_b200 import _C
    lib = _C.lib()
    assert _call(lib, B=0, N=1 << 24) == 0
    assert _call(lib, B=0, N=1) == 0
    assert _call(lib, B=0, verts=None, total_V=0, faces=None, total_F=0) == 0
    assert _call(lib, B=0, total_F=1 << 40, total_V=1 << 40, scratch_bytes=1 << 62) == 0


def _align(x):
    return (x + 255) // 256 * 256


@pytest.mark.parametrize("B,F", [(0, 0), (1, 1), (3, 2047), (3, 2048), (7, 2049), (1000, 10 ** 7)])
def test_scratch_size_arithmetic(lib_built, B, F):
    """The f64 CDF, then per tile (at most F/TILE + B of them) a f64 prefix and two int32 flags,
    then per mesh its first tile (i64, B+1), total (f64) and last face (i32); 256-byte aligned."""
    from sonet_b200 import _C
    tile = _C.CONSTANTS["SONET_MESH_TILE"]
    T = F // tile + B
    o = _align(8 * F)
    for nbytes in (8 * T, 4 * T, 4 * T, 8 * (B + 1), 8 * B, 4 * B):
        o = _align(o + nbytes)
    assert _C.lib().sonet_mesh_sample_scratch_bytes(B, F) == o
    assert _C.lib().sonet_mesh_sample_scratch_bytes(-1, F) == -1
    assert _C.lib().sonet_mesh_sample_scratch_bytes(B, -1) == -1


def test_symbol_exported_declared_and_bound(lib_built):
    from sonet_b200 import _C, ops
    h = ctypes.CDLL(lib_built)
    text = open(os.path.join(ROOT, "include", "sonet_b200.h")).read()
    for name in (NAME, SIZE):
        assert hasattr(h, name)
        assert re.search(r"\b%s\s*\(" % name, text)
        assert name in _C.EXPORTED_SYMBOLS
    assert len(_C._SIGNATURES[NAME]) == 17 and _C._RESTYPE[SIZE] is ctypes.c_longlong
    assert _C._SIGNATURES[NAME][2] is ctypes.c_longlong and _C._SIGNATURES[NAME][5] is ctypes.c_longlong
    assert ops.MESH_MAX_N == 1 << 24
    assert (_C.CONSTANTS["SONET_MESH_RUN"], _C.CONSTANTS["SONET_MESH_TILE"]) == (8, 2048)


# ---- host helpers ---------------------------------------------------------------------------------
def test_draw_host_order():
    """Per mesh, sampler.m's order: N face uniforms, then N u, then N v."""
    from sonet_b200 import meshes
    B, N = 3, 5
    d = meshes.draw_host(np.random.RandomState(7), B, N)
    assert d.shape == (B * N, 3) and d.dtype == np.float64
    rs = np.random.RandomState(7)
    for b in range(B):
        for k in range(3):
            assert np.array_equal(d[b * N:(b + 1) * N, k], rs.random_sample(N)), (b, k)


def test_meshes_validation():
    from sonet_b200 import meshes
    tri = (np.eye(3), np.array([[0, 1, 2]]))
    with pytest.raises(ValueError, match="expected \\[V,3\\]"):
        meshes.Meshes([(np.zeros((3, 2)), np.array([[0, 1, 2]]))], device="cpu")
    with pytest.raises(ValueError, match="mesh ids"):
        meshes.Meshes([tri, tri], mesh_ids=[5], device="cpu")
    m = meshes.Meshes([tri, (np.zeros((4, 3)), np.zeros((0, 3), np.int64))], mesh_ids=[9, 4],
                      device="cpu")
    assert m.v_off.tolist() == [0, 3, 7] and m.f_off.tolist() == [0, 1, 1]
    assert m.mesh_ids.tolist() == [9, 4] and len(m) == 2
    assert m.verts.dtype.is_floating_point and str(m.faces.dtype) == "torch.int32"


def test_save_npz_round_trip_through_the_reference_loader(tmp_path):
    """Files written by save_npz, read by the reference's own ModelNet_Shrec_Loader (shrec, test
    mode, input_pc_num = all points: the loader's choice is then a permutation we replay)."""
    from oracle import ref_shims
    if not os.path.isdir(os.path.join(ref_shims.REF, "data")):
        pytest.skip("the reference checkout is not on this machine")
    from sonet_b200 import meshes
    ref_shims.install(use_ref_plugin=False)
    import torch
    from data.modelnet_shrec_loader import ModelNet_Shrec_Loader
    rs = np.random.RandomState(3)
    B, N, M = 3, 50, 16
    pts = rs.uniform(-1, 1, size=(B, N, 6)).astype(np.float32)
    nodes = torch.from_numpy(rs.uniform(-1, 1, size=(B, M, 3)).astype(np.float32))
    names = ["%06d" % (55 * (i + 1) + i) for i in range(B)]
    root = tmp_path / "shrec"
    paths = meshes.save_npz(str(root / "4x4" / "test"), names, pts, nodes)
    assert [os.path.basename(p) for p in paths] == ["model_%s.npz" % n for n in names]
    (root / "category.txt").write_text("".join("cat%02d\n" % c for c in range(55)))
    (root / "test.txt").write_text("".join(n + "\n" for n in names))
    opt = types.SimpleNamespace(dataset="shrec", input_pc_num=N, node_num=M, som_k=1, classes=55,
                                batch_size=B, rot_horizontal=False, rot_perturbation=False,
                                translation_perturbation=False)
    loader = ModelNet_Shrec_Loader(str(root), "test", opt)
    assert len(loader) == B
    for b in range(B):
        np.random.seed(100 + b)
        item = loader[b]
        perm = np.random.RandomState(100 + b).choice(N, N, replace=False)
        pc, sn, label, som = item[0].numpy(), item[1].numpy(), item[2], item[3].numpy()
        assert np.array_equal(pc, pts[b][perm, 0:3].T)
        assert np.array_equal(sn, pts[b][perm, 3:6].T)
        assert np.array_equal(som, nodes[b].numpy().T)
        assert int(label) == int(names[b]) % 55
