"""Restatement of the two `frontier_exploration` functions VLFM calls.

TEST INFRASTRUCTURE.  PARITY UNPINNED: the package
(git+https://github.com/naokiyokoyama/frontier_exploration.git, no commit pinned,
$VLFM_REFERENCE/pyproject.toml:25) is NOT present in $VLFM_REFERENCE and cannot be
fetched; no reference test pins its results.  The functions are filled in by
oracle/explore_oracle.py (see there for the rule-by-rule restatement).
"""
from __future__ import annotations


def reveal_fog_of_war(top_down_map, current_fog_of_war_mask, current_point, current_angle, fov=90, max_line_len=100, **_):
    from .explore_oracle import reveal_fog_of_war as f

    return f(top_down_map, current_fog_of_war_mask, current_point, current_angle, fov, max_line_len)


def detect_frontier_waypoints(full_map, explored_mask, area_thresh=-1, xy=None):
    from .explore_oracle import detect_frontier_waypoints as f

    return f(full_map, explored_mask, area_thresh, xy)
