"""The shared synthetic scenes reproduce, bit for bit, the arrays the tests and tools built inline before they moved into
photo_slam_b200.synthetic: the stored outputs of tests/golden/test_quality_gpu.npz depend on them. The digests below were computed by
running that earlier inline code (test_quality_gpu.py's scene, views and trainee, and test_mcmc_gpu.py's 25 k-row trainee)."""
import hashlib

import numpy as np
import torch

import photo_slam_b200.synthetic as syn

QUALITY_SCENE = {
    "xyz": "09401a90143cab40e5439927a3d92e8f99baad70", "features_dc": "97d0cb3269a2e2bb96130da4611c5a63a596ee3e",
    "features_rest": "dce86f3676bb7083e8a1ae2b558884e4c83cb6a6", "scaling": "2d5b27d58e866661aaf611ff31fa08e6414de4d1",
    "rotation": "6fd9c7b118f7038279af61a7e7c20f285f92a1cd", "opacity": "5e967d2a0a6eeb152aa63b874e4349fd53896d15"}
# one digest per key over the six views in order
QUALITY_CAMERAS = {
    "viewmatrix": "3174e7a4a82e138df21f6ce9b72376357ca768b9", "projmatrix": "5890ee05344fef5fd5bd514ec3127051ffbc9171",
    "campos": "fa9f5b1f41cdc1e013c8aaae192a1125d7afacce", "tanfovx": "e8fdb2c54a5f039be77c5ac2b0bcf0fe2ec20343",
    "tanfovy": "742ca4a5a2b4b0cc00e18ad82dd557c6002b6f07", "W": "72d1ec86901133c4ce49bf33b048b5bb1b8551ed",
    "H": "a2647542268a72a90083c46d39ca33c0f26ecdcf", "Rt": "51c53548d2bcdbd4d0c64d542c8520f22e12574a"}
QUALITY_TRAINEE = {
    "xyz": "ff278bcd3c2af9cfce1a3b0932a4f0c2d9cea4b3", "features_dc": "8d24b3dc48a96f879f4b0fc5864537f55ccdf369",
    "features_rest": "cdfc64881750d9b32591c36d92e715c932372edc", "scaling": "f44345c6380943573c90ad954831507b2ab46938",
    "rotation": "d6a3b93862bac0539bd7e7ffb76990c5fa7e1748", "opacity": "a3243c42dcbd57b648479de3471cb81c9ee569af"}
# test_mcmc_gpu.py's trainee: make_scene(25 000, make_camera(320, 240, 260, 260), seed=21, scale_px=3.0) thinned
SMALL_TRAINEE = {
    "xyz": "a5eb133f82679804900721984eb6199ef4909725", "features_dc": "12a769a775a9c0a4e0e07afb6e6932d2089260e5",
    "features_rest": "191add54559e0fa087fdb252a90668913b4c16c2", "scaling": "e65ffebd753affcb6251b65f64f7304b75680352",
    "rotation": "3e3be08b98474bf16e7287a207b11fe4f4179448", "opacity": "a1d93f2035deba328088496b55fe3ca8bf6bd40b"}


def _digest(*arrays):
    h = hashlib.sha1()
    for a in arrays:
        a = np.asarray(a)
        h.update(f"{a.dtype.str}{a.shape}".encode())
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def test_quality_scene_and_trainee_are_bit_identical():
    scene, cams = syn.quality_scene()
    assert {k: _digest(v) for k, v in scene.items()} == QUALITY_SCENE
    assert len(cams) == 6
    assert {k: _digest(*[c[k] for c in cams]) for k in cams[0]} == QUALITY_CAMERAS
    assert {k: _digest(v) for k, v in syn.thinned_trainee(scene).items()} == QUALITY_TRAINEE


def test_thinned_trainee_of_another_scene_is_bit_identical():
    scene = syn.make_scene(25_000, syn.make_camera(320, 240, 260.0, 260.0), seed=21, scale_px=3.0)
    before = {k: v.copy() for k, v in scene.items()}
    assert {k: _digest(v) for k, v in syn.thinned_trainee(scene).items()} == SMALL_TRAINEE
    assert all(np.array_equal(scene[k], before[k]) for k in scene), "the source scene is left as it was"


def test_device_camera_equals_the_inline_dict():
    cam = syn.make_camera(320, 240, 250.0, 260.0, *syn.random_pose(np.random.default_rng(7)))
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to("cpu")
    old = dict(viewmatrix=T(cam["viewmatrix"]), projmatrix=T(cam["projmatrix"]), campos=T(cam["campos"]), tanfovx=float(cam["tanfovx"]),
               tanfovy=float(cam["tanfovy"]), W=320, H=240)
    new = syn.device_camera(cam, "cpu")
    assert new.keys() == old.keys()
    for k, v in old.items():
        if isinstance(v, torch.Tensor):
            assert new[k].dtype == v.dtype and new[k].device == v.device and torch.equal(new[k], v), k
        else:
            assert type(new[k]) is type(v) and new[k] == v, k
