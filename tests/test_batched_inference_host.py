"""Host side of batched inference (no GPU): the ragged descriptor table the Python side packs, argument validation of
the batched C entry points (refused on the host before any launch, reported through pk_last_error), the prompt
grouping of the SegGPT ensemble, and the machine code of the new kernels (no local-memory spills)."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from painter_b200 import _lib, build
from painter_b200 import seggpt_engine as se
from painter_b200.models_painter import Painter

NZ = ctypes.c_void_p(256)   # a non-null pointer: these calls are refused before anything dereferences it


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.lib()


def _refused(lib, rc, text):
    assert rc != 0
    assert text in lib.pk_last_error().decode()


def test_ragged_table_rows_and_offsets():
    sizes = [(427, 640), (9, 13), (50, 60)]
    tab, offs, total, max_pix = se.ragged_table(se.FIN_NEAREST_U8, [2, 0, 1], sizes, [0, 1, 1])
    assert tab.dtype == np.int32 and tab.shape == (3, se.RAG_FIELDS) and tab.flags.c_contiguous
    assert offs == [0, 427 * 640 * 3, 427 * 640 * 3 + 9 * 13 * 3]
    assert total == offs[-1] + 50 * 60 * 3 and max_pix == 427 * 640
    assert tab[:, :4].tolist() == [[2, 427, 640, 0], [0, 9, 13, 1], [1, 50, 60, 1]]
    assert [int(lo) & 0xFFFFFFFF | int(hi) << 32 for lo, hi in tab[:, 4:]] == offs
    # one element per pixel for the depth output, no cl_form given = 0
    tab, offs, total, _ = se.ragged_table(se.FIN_DEPTH, [0, 0], [(3, 5), (7, 2)])
    assert offs == [0, 15] and total == 29 and tab[:, 3].tolist() == [0, 0]


def test_ragged_table_offsets_beyond_32_bits():
    n = 40
    tab, offs, total, _ = se.ragged_table(se.FIN_BICUBIC_F64, [0] * n, [(8000, 8000)] * n)
    assert total > 2 ** 32 and offs[-1] > 2 ** 32
    lo, hi = tab[-1, 4], tab[-1, 5]
    assert (int(lo) & 0xFFFFFFFF) | (int(hi) << 32) == offs[-1] and hi > 0


@pytest.mark.parametrize("srcs,sizes", [([], []), ([0], [(0, 5)]), ([-1], [(4, 4)]), ([0, 1], [(4, 4)]),
                                        ([0], [(50000, 50000)])])
def test_ragged_table_rejects_bad_entries(srcs, sizes):
    with pytest.raises(ValueError, match="ragged_table"):
        se.ragged_table(se.FIN_BILINEAR_U8, srcs, sizes)


def test_finish_ragged_argument_validation(lib):
    L = lib
    _refused(L, L.pk_finish_ragged(se.FIN_BILINEAR_U8, None, 4, 4, NZ, 1, 16, None, NZ, None), "bad arguments")
    _refused(L, L.pk_finish_ragged(se.FIN_BILINEAR_U8, NZ, 4, 4, None, 1, 16, None, NZ, None), "bad arguments")
    _refused(L, L.pk_finish_ragged(se.FIN_BILINEAR_U8, NZ, 4, 4, NZ, 0, 16, None, NZ, None), "bad arguments")
    _refused(L, L.pk_finish_ragged(se.FIN_BILINEAR_U8, NZ, 4, 4, NZ, 65536, 16, None, NZ, None), "bad arguments")
    _refused(L, L.pk_finish_ragged(se.FIN_BILINEAR_U8, NZ, 0, 4, NZ, 1, 16, None, NZ, None), "bad arguments")
    _refused(L, L.pk_finish_ragged(se.FIN_BILINEAR_U8, NZ, 4, 4, NZ, 1, 0, None, NZ, None), "bad arguments")
    _refused(L, L.pk_finish_ragged(5, NZ, 4, 4, NZ, 1, 16, None, NZ, None), "unknown op 5")
    _refused(L, L.pk_finish_ragged(-1, NZ, 4, 4, NZ, 1, 16, None, NZ, None), "unknown op -1")
    # source images go with the blend and only with it
    _refused(L, L.pk_finish_ragged(se.FIN_NEAREST_BLEND, NZ, 4, 4, NZ, 1, 16, None, NZ, None), "blend")
    _refused(L, L.pk_finish_ragged(se.FIN_DEPTH, NZ, 4, 4, NZ, 1, 16, NZ, NZ, None), "blend")


def test_denorm_bottom_batched_argument_validation(lib):
    L = lib
    ok = dict(B=2, src_stride=1, h=56, w=28, p=16, finish=0)

    def call(bin_ptr=None, **kw):
        a = {**ok, **kw}
        return L.pk_denorm_bottom_batched(NZ, NZ, bin_ptr, a["B"], a["src_stride"], a["h"], a["w"], a["p"],
                                          a["finish"], None)

    _refused(L, L.pk_denorm_bottom_batched(None, NZ, None, 2, 1, 56, 28, 16, 0, None), "bad arguments")
    _refused(L, call(B=0), "bad arguments")
    _refused(L, call(src_stride=0), "bad arguments")
    _refused(L, call(h=55), "bad arguments")
    _refused(L, call(finish=3), "bad arguments")
    _refused(L, call(bin_ptr=NZ, finish=1), "binarised mask")
    _refused(L, call(bin_ptr=NZ, finish=2), "binarised mask")


def test_single_image_finishing_entry_points_are_not_exported(lib):
    """Every finishing step goes through pk_denorm_bottom_batched and pk_finish_ragged, for one image as for many."""
    for name in ("seg_postprocess", "denorm_bottom", "nearest_blend", "bilinear_u8", "bicubic_f64", "depth_finish",
                 "nearest_u8"):
        assert not hasattr(lib, "pk_" + name), name


@pytest.mark.parametrize("dtype", [np.float16, np.int32])
def test_painter_mirrors_refuse_canvases_that_are_not_float32_or_float64(dtype):
    """Refused before any device work, as run_batch refuses them, instead of being read as float32."""
    from painter_b200 import painter_inference as pi
    x = np.zeros((896, 448, 3), dtype)
    for mirror in ("run_one_image", "run_one_image_nearest", "run_one_image_depth", "run_one_image_restore"):
        with pytest.raises(ValueError, match="canvases"):
            getattr(pi, mirror)(x, x, (10, 10), None, "unused.png", "cuda")


def test_stitch_normalize_checks_every_member(lib):
    """Any number of members is accepted (launched in chunks of 16); each member is still checked."""
    L = lib
    n = 20
    arr, ia = ctypes.c_void_p * n, ctypes.c_int * n
    tops = [256] * n
    tops[17] = None
    _refused(L, L.pk_stitch_normalize(arr(*tops), ia(*[0] * n), arr(*[256] * n), ia(*[0] * n), NZ, n, 448, None),
             "bad member 17")
    dts = [0] * n
    dts[18] = 3
    _refused(L, L.pk_stitch_normalize(arr(*[256] * n), ia(*[0] * n), arr(*[256] * n), ia(*dts), NZ, n, 448, None),
             "bad member 18")


def test_prompt_groups_of_the_ensemble():
    ens = Painter._ensemble
    # default: the whole batch is one prompt ensemble (the reference's merge_between_batch semantics)
    assert [ens(None, i, 4, 0, None) for i in (0, 2, 3, 23)] == [(2, 4), (2, 4), (1, 4), (1, 4)]
    # Q = 2 queries x P = 2 prompts: [2][Q][P] before the early merge, [Q][P] after it
    assert [ens(None, i, 4, 0, 2) for i in (0, 2, 3, 23)] == [(4, 2), (4, 2), (2, 2), (2, 2)]
    assert ens(None, 5, 12, 0, 3) == (4, 3)
    assert ens(None, 1, 4, -1, 2) == (0, 0) and ens(None, 1, 4, 2, 2) == (0, 0)
    with pytest.raises(ValueError, match="does not divide"):
        ens(None, 0, 4, 0, 3)


def _sass(lib):
    tool = None
    for c in (os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"),
              shutil.which("cuobjdump")):
        if c and os.path.exists(c):
            tool = c
            break
    if tool is None:
        pytest.skip("cuobjdump (CUDA toolkit) not found")
    sass = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    out = {}
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split("\n", 1)[0].strip()
        out[name] = [m.group(1).strip() for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", body)]
    return out


def test_batched_finishing_kernels_do_not_spill(lib):
    k = _sass(lib)
    ragged = {n: i for n, i in k.items() if n.startswith("_ZN2pk20ragged_finish_kernelI")}
    post = {n: i for n, i in k.items() if n.startswith("_ZN2pk22seg_postprocess_kernelI")}
    assert len(ragged) == 5 and len(post) == 3, (sorted(ragged), sorted(post))
    for name, ins in {**ragged, **post}.items():
        assert not [i for i in ins if re.match(r"(STL|LDL)\b", i)], name
