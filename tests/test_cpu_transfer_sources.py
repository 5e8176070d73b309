"""Source checks of the library's host<->device copies and device entry (no GPU needed).

Every host<->device copy goes through the counted staging helpers of csrc/ekf.cu (ovp_transfer_bytes counts them all), the pinned staging
of the MSCKF and SLAM updates included.  ovp_create must name the context's device before ovp::enter makes a device current, or every
process would first create a context on device 0."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ov_plane_b200", "csrc")
KINDS = re.compile(r"\bcudaMemcpy(HostToDevice|DeviceToHost)\b")
# a top-level function definition: return type and name at column 0, then the parameter list
FUNC = re.compile(r"^(?:static\s+)?(?:inline\s+)?[A-Za-z_][\w:<>\s\*&]*?\b([A-Za-z_]\w*)\s*\(")
ALLOWED = {("ekf.cu", "stage_copy_in"), ("ekf.cu", "stage_copy_out"), ("ekf.cu", "stage_copy2d_in"), ("ekf.cu", "stage_copy2d_out")}


def _sources():
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".inc", ".h", ".cuh")) and f != "debug_hooks.cu":
            with open(os.path.join(CSRC, f)) as fh:
                yield f, fh.read().splitlines()


def copies():
    """(file, enclosing function, line number) of every host<->device copy kind named in the product sources"""
    out = []
    for f, lines in _sources():
        func = None
        for i, line in enumerate(lines, 1):
            m = FUNC.match(line)
            if m and not line.startswith(("return", "#")):
                func = m.group(1)
            if KINDS.search(line):
                out.append((f, func, i))
    return out


def test_copies_go_through_the_staging_helpers():
    found = copies()
    assert any(f == "ekf.cu" and fn == "stage_copy_in" for f, fn, _ in found)  # the scan sees the helpers themselves
    stray = [c for c in found if (c[0], c[1]) not in ALLOWED]
    assert not stray, "host<->device copies outside the counted staging helpers: %s" % stray


def test_helpers_are_defined_once():
    defs = [(f, i) for f, lines in _sources() for i, line in enumerate(lines, 1)
            if re.match(r"^int (ensure_stage|stage_copy_in|stage_copy_out|stage_copy2d_in|stage_copy2d_out)\(Ctx.*\{$", line)]
    assert len(defs) == 5 and {f for f, _ in defs} == {"ekf.cu"}, defs


def test_create_names_the_device_before_enter():
    with open(os.path.join(CSRC, "capi.cu")) as fh:
        src = fh.read()
    body = src[src.index("int ovp_create("):]
    body = body[:body.index("\n}\n")]
    assign = re.search(r"\b(?:h->c|c)\.?(?:->)?device\s*=\s*device\s*;", body)
    enter = body.find("enter(")
    cuda = re.search(r"\bcuda(?!GetDeviceCount)\w+\(", body)
    assert assign and enter >= 0, "ovp_create must set the context's device and enter it"
    assert assign.start() < enter, "ovp_create calls enter before it names the context's device"
    assert assign.start() < cuda.start(), "ovp_create makes a CUDA call before it names the context's device"
