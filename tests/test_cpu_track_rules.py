"""Source checks of the feature-track rules (no GPU needed).

Which feature tracks an entry point accepts is one decision, taken by check_offsets / check_tracks in csrc/features_host.inc: each refusal
message of a malformed track is written in one function, and no other function checks the clone handles of a measurement array.  The
anchor-handle checks (anchors.cu) and a shard's clone list (shard_cols) are single handles, not tracks."""
import re

from test_cpu_transfer_sources import FUNC, _sources

MESSAGES = ("must start at 0", "non-decreasing", "is not a clone in the state", "twice (mono camera assumed)", "is listed twice")
CLONE_CHECKS_ALLOWED = {("features_host.inc", "check_tracks"), ("anchors.cu", "ovp_feature_jacobian_full_rep"),
                        ("anchors.cu", "ovp_slam_set_representation"), ("anchors.cu", "ovp_slam_perform_anchor_change"), ("capi2.cu", "shard_cols")}
SINGLE_HANDLES = CLONE_CHECKS_ALLOWED - {("features_host.inc", "check_tracks")}  # an anchor, a shard's clone list; the landmark list of
# ovp_msckf_update_landmarks is checked for duplicates on its own


def _functions():
    """(file, enclosing function, line) of every line of the product sources (debug_hooks.cu is not one)"""
    for f, lines in _sources():
        func = None
        for line in lines:
            m = FUNC.match(line)
            if m and not line.startswith(("return", "#")):
                func = m.group(1)
            yield f, func, line


def test_each_refusal_message_is_written_once():
    for msg in MESSAGES:
        where = {(f, fn) for f, fn, line in _functions() if msg in line and "landmark %lld" not in line} - SINGLE_HANDLES
        assert len(where) == 1, (msg, sorted(where))


def test_clone_handles_are_checked_by_the_validator():
    calls = {(f, fn) for f, fn, line in _functions() if re.search(r"\bis_clone\(", line) and "static inline bool is_clone" not in line}
    assert ("features_host.inc", "check_tracks") in calls
    assert calls <= CLONE_CHECKS_ALLOWED, sorted(calls - CLONE_CHECKS_ALLOWED)
