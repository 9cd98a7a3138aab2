"""The render-thread events of the camera run and the GPU group (GS_UNITY_EVENT_FRAME_CAMERAS, _GROUP_FRAME_OBJECTS, _GROUP_SYNC)
without a device: the payloads' C layout against the ctypes structs the managed-side checks mirror, the exported symbols, the
error paths that need no CUDA call, and the C++ mirror's payload fillers."""
import ctypes as C
import re
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
PAYLOADS = ["GsUnityFrameCamerasEvent", "GsUnityGroupFrameObjectsEvent", "GsUnityGroupSyncEvent"]


def _layout_program(N):
    """A C program that prints `name sizeof` and `name.field offsetof` for every field of the new payloads, as the header
    lays them out."""
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "include/gsplat_b200.h"', "int main(void) {"]
    for name in PAYLOADS:
        lines.append('  printf("%s %%zu\\n", sizeof(%s));' % (name, name))
        for field, _ in getattr(N, name)._fields_:
            lines.append('  printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (name, field, name, field))
    lines += ["  return 0;", "}"]
    return "\n".join(lines) + "\n"


def test_payload_layouts_match_the_header(tmp_path):
    """A managed struct that disagrees with the header is silent memory corruption on the render thread: every field's offset
    and every size, from the C compiler, must be the ctypes binding's."""
    from unitygaussiansplatting_b200 import _native as N
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text(_layout_program(N))
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I" + str(ROOT), str(src), "-o", str(exe)],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    got = dict(line.split() for line in subprocess.run([str(exe)], stdout=subprocess.PIPE, text=True, check=True).stdout.splitlines())
    for name in PAYLOADS:
        cls = getattr(N, name)
        assert int(got[name]) == C.sizeof(cls), name
        for field, _ in cls._fields_:
            assert int(got["%s.%s" % (name, field)]) == getattr(cls, field).offset, "%s.%s" % (name, field)
    # the header's own statement of the sizes, which the managed side's StructLayout must reach
    assert [C.sizeof(getattr(N, n)) for n in PAYLOADS] == [112, 104, 16]
    # and no field of the header is missing from the binding (a field hidden in padding would keep the size)
    text = (ROOT / "include" / "gsplat_b200.h").read_text()
    for name in PAYLOADS:
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), text, re.S).group(1)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        declared = re.findall(r"(\w+)(?:\[\d+\])?\s*[,;]", body)
        assert declared == [f for f, _ in getattr(N, name)._fields_], name


def test_event_ids_and_limits_match_the_header():
    from unitygaussiansplatting_b200 import _native as N
    text = (ROOT / "include" / "gsplat_b200.h").read_text()
    for name in ("FRAME", "SYNC", "FRAME_OBJECTS", "FRAME_CAMERAS", "GROUP_FRAME_OBJECTS", "GROUP_SYNC"):
        m = re.search(r"GS_UNITY_EVENT_%s = (\d+)" % name, text)
        assert m and int(m.group(1)) == getattr(N, "GS_UNITY_EVENT_" + name), name
    assert (N.GS_UNITY_EVENT_FRAME_CAMERAS, N.GS_UNITY_EVENT_GROUP_FRAME_OBJECTS, N.GS_UNITY_EVENT_GROUP_SYNC) == (4, 5, 6)
    m = re.search(r"#define GS_UNITY_EVENT_MAX_CAMERAS (\d+)u", text)
    assert m and int(m.group(1)) == N.GS_UNITY_EVENT_MAX_CAMERAS


def test_new_symbols_are_exported_and_sizes_reported():
    from unitygaussiansplatting_b200 import _native as N
    lib = N.native()
    assert lib.gs_unity_frame_cameras_event_size() == C.sizeof(N.GsUnityFrameCamerasEvent)
    assert lib.gs_unity_group_frame_objects_event_size() == C.sizeof(N.GsUnityGroupFrameObjectsEvent)
    assert lib.gs_unity_group_sync_event_size() == C.sizeof(N.GsUnityGroupSyncEvent)


def test_error_paths_without_a_device():
    """A NULL context or group is the direct call's refusal, with its code and text; nothing is thrown and no CUDA call made."""
    from unitygaussiansplatting_b200 import _native as N
    lib = N.native()
    fn = lib.gs_unity_get_render_event_func()
    cases = [
        (N.GS_UNITY_EVENT_FRAME_CAMERAS, N.GsUnityFrameCamerasEvent(camera_count=1),
         lambda: lib.gs_frame_cameras(None, 1, None, None, None, None, None, None, None)),
        (N.GS_UNITY_EVENT_GROUP_FRAME_OBJECTS, N.GsUnityGroupFrameObjectsEvent(object_count=1),
         lambda: lib.gs_group_frame_objects(None, 1, None, None, None, None, None, None)),
        (N.GS_UNITY_EVENT_GROUP_SYNC, N.GsUnityGroupSyncEvent(), lambda: lib.gs_group_sync(None)),
    ]
    for event_id, ev, direct in cases:
        want = direct()
        want_text = lib.gs_last_error(None)
        lib.gs_group_balance_rows(None, 0, 1, None)   # another error in between: the event must set the text again
        ev.status = N.GS_ERR_NOT_READY
        assert ev.status == N.GS_ERR_NOT_READY
        assert N.unity_event(event_id, ev) == want == -1
        assert lib.gs_last_error(None) == want_text
        fn(event_id, None)                            # a NULL payload is ignored
    # more cameras than one event takes: refused by the callback itself, before gs_frame_cameras
    ev = N.GsUnityFrameCamerasEvent(camera_count=N.GS_UNITY_EVENT_MAX_CAMERAS + 1, status=N.GS_ERR_NOT_READY)
    assert N.unity_event(N.GS_UNITY_EVENT_FRAME_CAMERAS, ev) == -1
    assert b"GS_UNITY_EVENT_MAX_CAMERAS" in lib.gs_last_error(None)


SRC = r'''
#include "unitygaussiansplatting_b200/host/GaussianSplatRenderer.hpp"
int main() {
  using namespace GaussianSplatting;
  GaussianSplatRenderer a, b;
  b.OnEnable(GsAssetDesc{}, a.context());
  std::vector<CameraState> cams(2);
  std::vector<GsImage *> rts = {nullptr, nullptr}, targets = {nullptr, nullptr};
  UnityFrameCamerasEvent ev;
  bool filled = GaussianSplatRenderer::FillFrameCamerasEvent(cams, {&a, &b}, rts, targets, &ev);
  if (filled) gs_unity_get_render_event_func()(GS_UNITY_EVENT_FRAME_CAMERAS, &ev.event);
  GaussianSplatRendererGroup grp;
  UnityGroupFrameObjectsEvent gev;
  GsImage *none[1] = {nullptr};
  if (grp.FillFrameObjectsEvent(cams[0], {&grp}, none, none, &gev))
    gs_unity_get_render_event_func()(GS_UNITY_EVENT_GROUP_FRAME_OBJECTS, &gev.event);
  GsUnityGroupSyncEvent sync = grp.SyncEvent();
  gs_unity_get_render_event_func()(GS_UNITY_EVENT_GROUP_SYNC, &sync);
  return filled ? 1 : 0;
}
'''


def test_mirror_payload_fillers_compile(tmp_path):
    src = tmp_path / "unity_events.cpp"
    src.write_text(SRC)
    r = subprocess.run(["/usr/bin/g++", "-std=c++17", "-Wall", "-Werror", "-fsyntax-only", "-I" + str(ROOT), str(src)],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
