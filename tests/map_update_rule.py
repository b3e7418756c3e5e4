"""The frame path's map-update rule (include/kicp.h kicp_ctx_set_map_update) restated in Python, and a table of cases at its exact
boundaries, shared by the CPU, emulator and GPU tests."""
import math

ALWAYS, NEVER, GATED = 0, 1, 2
APPLIED, NO_CORRESPONDENCES, REJECTED, SKIPPED, NONE = 0, 1, 2, 3, 4
KICP_OK, KICP_WARN_NO_CORRESPONDENCES = 0, 16


def rule(mode, min_inliers, min_fitness, max_inlier_rmse, reg_status, map_was_empty, n_inliers, fitness, inlier_rmse):
    """the outcome of a frame, in the header's order"""
    if mode == NEVER:
        return SKIPPED
    if reg_status != KICP_OK:
        return NO_CORRESPONDENCES
    if mode == ALWAYS or map_was_empty:
        return APPLIED
    ok = n_inliers >= min_inliers and fitness >= min_fitness and inlier_rmse <= max_inlier_rmse
    return APPLIED if ok else REJECTED


def rule_stats(policy, reg_status, map_was_empty, st):
    """rule() of a (mode, min_inliers, min_fitness, max_inlier_rmse) policy and a report with n_inliers, fitness and inlier_rmse"""
    return rule(*policy, reg_status, map_was_empty, st.n_inliers, st.fitness, st.inlier_rmse)


def table():
    """[(policy, reg_status, map_was_empty, (n_points, n_inliers, fitness, inlier_rmse))]: every threshold met exactly and missed by
    one ulp or one inlier, n_points == 0, the empty-map clause, a non-OK status, NaN statistics, and every mode"""
    gate = (GATED, 100, 0.5, 0.25)
    base = (200, 100, 0.5, 0.25)  # every threshold met with equality
    rows = []
    for mode in (ALWAYS, NEVER, GATED):
        for status in (KICP_OK, KICP_WARN_NO_CORRESPONDENCES):
            for empty in (False, True):
                for st in (base, (200, 99, 0.5, 0.25), (0, 0, 0.0, 0.0)):
                    rows.append(((mode,) + gate[1:], status, empty, st))
    for st in [base, (200, 99, 0.5, 0.25), (200, 101, 0.5, 0.25), (200, 100, math.nextafter(0.5, 0.0), 0.25),
               (200, 100, math.nextafter(0.5, 1.0), 0.25), (200, 100, 0.5, math.nextafter(0.25, 1.0)),
               (200, 100, 0.5, math.nextafter(0.25, 0.0)), (0, 0, 0.0, 0.0), (200, 100, math.nan, 0.25), (200, 100, 0.5, math.nan)]:
        rows.append((gate, KICP_OK, False, st))
    for pol in [(GATED, 0, 0.0, math.inf), (GATED, 0, 1.0, math.inf), (GATED, 1, 0.0, math.inf), (GATED, 0, 0.0, 5e-324)]:
        for st in [(0, 0, 0.0, 0.0), (10, 10, 1.0, 0.0), (10, 3, 0.3, 0.7), (10, 0, 0.0, 0.0)]:
            for empty in (False, True):
                rows.append((pol, KICP_OK, empty, st))
    return rows
