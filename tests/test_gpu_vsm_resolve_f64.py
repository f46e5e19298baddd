"""The renderer's VSM chain on the device, at 1920 x 1080 with unit-length suns, against the binary64 cast and restatement of
tests/test_oracle_vsm_resolve_f64.py and against the oracle: oxr_render -> oxr_vsm_update_pages -> oxr_vsm_draw_shadows ->
oxr_vsm_resolve_shadows over an oxb_* scene of a ground, floating squares and a tilted plane, each with its own instance transform.

Suns at 30 and 80 degrees of elevation take perpendicular_basis's +y axis; the one at 88.5 degrees (|L.y| >= 0.999) takes +x.  Per
sun, three frames with the camera turning in place (the page offsets stay, sun_moved in the first frame only), so the later frames
resolve through pages drawn this frame and resident clean pages drawn before.  Every frame:
- every Backed page of the renderer's atlas equals the inverse-mapped cast on a 1-in-SUB x 1-in-SUB lattice of its texels (under the
  tolerance and silhouette band of the CPU module);
- the device's shadow equals the oracle resolve bit for bit on the renderer's page table, atlas and depth and the oracle decode's
  normals;
- the device's shadow equals the restatement under the CPU module's rules on PIXELS random non-sky pixels (the restatement's cost
  keeps it to a subset)."""
import numpy as np
import pytest

from oxylus_b200 import abi, synth
from tests.test_gpu_vsm_pages import vsm_context
from tests.test_gpu_vsm_resolve import _two_sided_grid, inverse_pv
from tests.test_oracle_vsm_resolve_f64 import (AMBIGUOUS_ANALYTIC, B, cast_atlas_pages, check_atlas, compare, oracle_noise, restate,
                                               unit_sun)

pytestmark = pytest.mark.gpu

W, H = 1920, 1080
SUB = 4
PIXELS = 40000
SUNS = {"sun30": unit_sun(30.0), "sun80": unit_sun(80.0), "zenith": unit_sun(88.5, 10.0)}


@pytest.fixture(scope="module")
def capi():
    from oxylus_b200 import capi

    capi.load()
    return capi


@pytest.fixture(scope="module")
def vr():
    import pyoracle_vsm_resolve

    pyoracle_vsm_resolve.build()
    return pyoracle_vsm_resolve


def _xf(scale, translate):
    m = np.diag([scale[0], scale[1], scale[2], 1.0]).astype(np.float64)
    m[:3, 3] = translate
    return m


# (grid cells, height, row-major instance transform): a ground and three casters, one of them tilted
INSTANCES = [(4, 0.0, _xf((96.0, 1.0, 96.0), (0.0, 0.0, -64.0))),
             (2, 0.0, _xf((4.0, 1.0, 4.0), (0.0, 5.0, -28.0))),
             (2, 0.0, _xf((2.0, 1.0, 2.0), (8.0, 2.5, -18.0))),
             (2, 0.0, _xf((4.0, 1.0, 3.0), (18.0, 3.5, -43.0)) @ np.array([[1, 0, 0, 0], [0, 0.8, -0.6, 0], [0, 0.6, 0.8, 0], [0, 0, 0, 1.0]]))]


def build_scene(capi):
    built, xf, tris = [], np.zeros((len(INSTANCES), 16), np.float32), []
    for k, (n, y, m) in enumerate(INSTANCES):
        p, i, nrm = _two_sided_grid(n, y)
        built.append(capi.BuiltMesh(p, [(i, 0.0)], normals=nrm))
        m32 = m.astype(np.float32)
        xf[k] = m32.T.reshape(16)
        # world triangles: the dequantised binary16 positions times the instance transform, binary64; one winding of each pair
        q = p.astype(np.float16).astype(np.float64)
        wp = (np.concatenate([q, np.ones((len(q), 1))], 1) @ m32.astype(np.float64).T)[:, :3]
        tris.append(wp[i.reshape(-1, 3)[: len(i) // 6]])
    sc = capi.assemble_scene(built, list(range(len(built))), xf, W, H)
    return sc, np.concatenate(tris)


def camera(sc, yaw_deg, eye):
    yaw = np.radians(yaw_deg)
    target = np.asarray(eye) + np.array([np.sin(yaw), -0.45, -np.cos(yaw)])
    cam = np.zeros(1, dtype=abi.CULL_CAMERA_DT)
    cam["projection_view"][0] = synth.mat_mul_cm(synth.perspective_reverse_z(60.0, W / H, 0.1, 1000.0), synth.look_at(eye, target, (0.0, 1.0, 0.0)))
    cam["position"][0] = eye
    cam["acceptable_lod_error"], cam["near_clip"], cam["mesh_instance_count"] = 2.0, 0.1, sc.mesh_instance_count
    cam["resolution"][0] = (W, H)
    return cam


@pytest.mark.parametrize("sun", list(SUNS))
def test_unit_sun_frames(capi, orc, vr, sun):
    L = SUNS[sun]
    sc, tris = build_scene(capi)
    hs = orc.HostScene(sc)
    eye = np.float64([0.0, 14.0, 6.0])
    vsm = vsm_context(width=W, height=H)
    vsm["directional_light_dir"][0] = L
    cm = synth.make_vsm_clipmaps(L, eye)
    coarse = np.zeros(1, dtype=abi.CULL_CAMERA_DT)  # clipmap 9's view (Shadowmaps.cpp:433-463)
    coarse["projection_view"][0] = cm["projection_view_mat"][9]
    coarse["position"][0] = L
    coarse["acceptable_lod_error"], coarse["near_clip"], coarse["mesh_instance_count"] = 2.0, 0.0, sc.mesh_instance_count
    coarse["resolution"][0] = (8192, 8192)
    r = capi.Renderer(0, sc)
    mask = np.zeros(r.ctx.out.visibility_mask_words, dtype=np.uint32)
    rng = np.random.default_rng(7)
    seen_clean = 0
    drawn_before = set()
    try:
        for f, yaw in enumerate((-12.0, 0.0, 12.0)):
            cam = camera(sc, yaw, eye)
            out = r.render(cam, want_indices=False)
            ref = orc.frame(hs, cam, W, H, mask, None)
            v32, depth = orc.resolve(ref["vis64"])
            np.testing.assert_array_equal(out["depth"].view(np.uint32), depth.view(np.uint32))
            inv_pv, res = inverse_pv(cam), cam["resolution"][0]
            pg = r.vsm_update_pages(vsm, cm, inv_pv, res, sun_moved=(f == 0), hpb_levels=7)
            r.vsm_draw_shadows(coarse)
            pt = r.ctx.download(pg.page_tables, np.uint32, 10 * 64 * 64).reshape(10, 64, 64)
            atlas = r.ctx.download(pg.physical_atlas, np.float32, 8192 * 8192).reshape(8192, 8192)
            got = r.vsm_resolve_shadows(cam)
            # the atlas: every Backed page, drawn this frame or resident from an earlier one
            backed = np.argwhere((pt & B) != 0)
            addrs = set(int(a) for a in (pt[tuple(backed.T)] >> 16))
            seen_clean += len(addrs & drawn_before)
            drawn_before |= addrs
            check_atlas(atlas, cast_atlas_pages(tris, vsm, cm, pt, 8192, sub=SUB), 8192, 128, f"{sun} frame {f} atlas")
            # the oracle, bit for bit
            normals = orc.decode_visbuffer(hs, ref["meshlet_instances"], int(ref["visibility"]["total"][0]), cam, v32)["uv_normal"]
            want, pcf = vr.vsm_resolve_shadows(vsm, inv_pv, res, cm, depth, normals, pt, atlas)
            np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32), err_msg=f"{sun} frame {f}")
            # the restatement on a subset of the pixels holding depth
            live = np.nonzero(depth.reshape(-1) != 0)[0]
            pix = np.sort(rng.choice(live, size=min(PIXELS, len(live)), replace=False))
            res_r = restate(vsm, inv_pv, res, cm, depth, normals, pt, atlas, pixels=pix, ref_noise=oracle_noise(vr, H, W, pix))
            compare(got.reshape(-1)[pix], res_r, np.ones(len(pix), bool), f"{sun} frame {f} restatement", AMBIGUOUS_ANALYTIC)
            print(f"{sun} frame {f}: backed pages {len(addrs)}, shadowed {int((got == 0).sum())}, penumbra {int(((got > 0) & (got < 1)).sum())}, "
                  f"pcf pixels {int(pcf.sum())}")
            assert (got == 0).sum() > 1000 and pcf.sum() > 100
    finally:
        r.close()
    assert seen_clean > 0, "no page stayed resident from one frame to the next"
