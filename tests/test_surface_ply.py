"""scene_io.save_surface_ply on a small hand-made surface, parsed back with numpy: header, counts, coordinates,
per-vertex colours (the polygon's colour, clamped and truncated from x 255) and face lists."""
import numpy as np
import pytest

from radfoam_b200 import scene_io


def parse(path):
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    header = data[:end].decode("ascii").splitlines()
    nv = int(next(h for h in header if h.startswith("element vertex")).split()[-1])
    nf = int(next(h for h in header if h.startswith("element face")).split()[-1])
    vdt = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    verts = np.frombuffer(data, vdt, nv, end)
    at = end + nv * vdt.itemsize
    faces = []
    for _ in range(nf):
        c = data[at]
        faces.append(np.frombuffer(data, "<i4", c, at + 1).tolist())
        at += 1 + 4 * c
    assert at == len(data)
    return header, verts, faces


def test_round_trip(tmp_path):
    surface = {
        "vertices": np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0],
                              [0, 0, 1], [2, 0, 1], [0, 2, 1.5]], np.float32),
        "offsets": np.array([0, 4, 7], np.int64),
        "cells": np.array([[3, 8], [3, 9]], np.uint32),
        "rgb": np.array([[0.5, 1.7, -0.2], [np.nan, 0.999, 0.0]], np.float16),
    }
    path = tmp_path / "s.ply"
    scene_io.save_surface_ply(str(path), surface)
    header, verts, faces = parse(str(path))
    assert header[:2] == ["ply", "format binary_little_endian 1.0"]
    assert "element vertex 7" in header and "element face 2" in header
    assert "property list uchar int vertex_indices" in header and header[-1] == "end_header"
    assert np.array_equal(np.stack([verts["x"], verts["y"], verts["z"]], 1), surface["vertices"])
    want = np.array([[127, 255, 0]] * 4 + [[255, 254, 0]] * 3, np.uint8)  # 0.5*255 = 127.5 -> 127; NaN -> 255
    got = np.stack([verts["red"], verts["green"], verts["blue"]], 1)
    assert np.array_equal(got, want), got
    assert faces == [[0, 1, 2, 3], [4, 5, 6]]


def test_empty_and_malformed(tmp_path):
    empty = {"vertices": np.zeros((0, 3), np.float32), "offsets": np.zeros(1, np.int64),
             "cells": np.zeros((0, 2), np.uint32), "rgb": np.zeros((0, 3), np.float32)}
    scene_io.save_surface_ply(str(tmp_path / "e.ply"), empty)
    header, verts, faces = parse(str(tmp_path / "e.ply"))
    assert verts.size == 0 and faces == []
    bad = dict(empty, vertices=np.zeros((2, 3), np.float32), offsets=np.array([0, 2]), rgb=np.zeros((1, 3)))
    with pytest.raises(ValueError):
        scene_io.save_surface_ply(str(tmp_path / "b.ply"), bad)
