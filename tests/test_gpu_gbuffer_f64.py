"""The vis-buffer decode on the device (oxc_decode_gbuffer and oxc_decode_visbuffer) on non-uniformly scaled, sheared, mirrored and
tilted instances, from the device's own vis buffer: bit for bit against the CPU oracle, and against the binary64 restatement of
tests/test_oracle_gbuffer_f64.py under that module's rules."""
import numpy as np
import pytest

from tests.test_gpu_gbuffer import PLANES, decode_gpu, gpu_frame
from tests.test_gpu_parity import _assert_planes_equal, make_ctx
from tests.test_oracle_gbuffer_f64 import compare, deformed_scene, material_table, planes_scene, restate

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def capi():
    from oxylus_b200 import capi

    capi.load()
    return capi


@pytest.fixture(scope="module")
def gb():
    import pyoracle_gbuffer

    pyoracle_gbuffer.build()
    return pyoracle_gbuffer


def check_device(capi, orc, gb, sc, seed):
    ctx = make_ctx(capi, sc)
    table = material_table(seed)
    dev_images, ptrs = table["host"].device_images(ctx)
    ctx.set_materials(table["materials"], dev_images, table["samplers"])
    w, h = sc.width, sc.height
    cam = sc.camera(0.0)
    hs, ref, vis_dev, total = gpu_frame(capi, orc, sc, ctx, cam)
    v32, _ = orc.resolve(ref["vis64"])
    mi = ref["meshlet_instances"]
    sentinel = np.float32(-7.25)
    want, bad = gb.decode_gbuffer(hs, mi, total, cam, v32, table["host"], init=sentinel)
    assert bad == 0
    got = decode_gpu(ctx, cam, w, h, vis64_dev=vis_dev, init=sentinel)
    for k in PLANES:
        _assert_planes_equal(got[k], want[k], k)
    names = ("lambda_", "ddx", "ddy", "uv_normal", "uv_grad")
    dev = {n: ctx.alloc(w * h * 16) for n in names}
    ctx.decode_visbuffer(cam, w, h, dev, vis64_dev=vis_dev)
    geom = {n: ctx.download(p, np.float32, w * h * 4).reshape(h, w, 4) for n, p in dev.items()}
    want_geom = orc.decode_visbuffer(hs, mi, total, cam, v32)
    decoded = want_geom["lambda_"][:, :, 3] != 0
    for n in names:
        _assert_planes_equal(geom[n][decoded], want_geom[n][decoded], n)
    r = restate(sc, mi, total, cam, v32, table["materials"], table["images"], table["samplers"])
    measured = compare(r, got, geom)
    for p in list(dev.values()) + ptrs + [vis_dev]:
        ctx.free(p)
    ctx.close()
    return measured, r


@pytest.mark.parametrize("seed", [1, 2])
def test_tilted_planes_on_the_device(capi, orc, gb, seed):
    m, r = check_device(capi, orc, gb, planes_scene(seed, 320, 192), seed)
    assert m["decoded"] > 1500 and (r["det"] < 0).sum() > 100


@pytest.mark.parametrize("seed", [1, 2])
def test_deformed_instances_on_the_device(capi, orc, gb, seed):
    m, r = check_device(capi, orc, gb, deformed_scene(seed, 640, 360, n_meshlets=100_000), seed)
    assert m["decoded"] > 40_000 and (r["det"] < 0).sum() > 5000


def test_benchmark_scene_with_deformed_transforms_1080p(capi, orc, gb):
    """the scene bench.py measures (1 M meshlet instances, make_scene's default seed) at 1920 x 1080, with its transforms replaced by
    non-uniform, sheared and mirrored ones scaled up three times"""
    m, r = check_device(capi, orc, gb, deformed_scene(7, 1920, 1080, n_meshlets=1_000_000, scale=3.0, bench=True), 7)
    assert m["decoded"] > 500_000 and (r["det"] < 0).sum() > 50_000
