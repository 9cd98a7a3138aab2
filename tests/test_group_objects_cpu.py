"""gs_group_frame_objects validates its arguments without a GPU: a NULL group and a bad object count come back as
GS_ERR_INVALID_ARGUMENT (never a throw or an abort)."""
import ctypes as C


def test_group_frame_objects_rejects_null_group_and_bad_count(g):
    from unitygaussiansplatting_b200 import _native as N
    lib = N.native()
    fps = (N.GsFrameParams * 1)()
    do_sort = (C.c_int32 * 1)(1)
    assets = (C.c_void_p * 1)()
    assert lib.gs_group_frame_objects(None, 1, assets, fps, do_sort, None, None, None) == -1
    assert lib.gs_group_frame_objects(None, 0, None, None, None, None, None, None) == -1
    assert b"null group" in lib.gs_last_error(None)


def test_python_group_object_knobs_match_the_renderer(g):
    """A group's further objects carry the knobs of GaussianSplatRenderer that a frame reads."""
    from unitygaussiansplatting_b200 import multigpu

    class _Stub:
        pass
    o = _Stub()
    multigpu._init_knobs(o)
    for name in ("localToWorldMatrix", "m_RenderOrder", "m_SplatScale", "m_OpacityScale", "m_SHOrder", "m_SHOnly", "m_SortNthFrame",
                 "m_FrameCounter", "m_Cutouts", "m_DeletedBits", "m_SelectedBits", "sceneDepth"):
        assert hasattr(o, name), name
