"""The PointNav navigator (vlfm/policy/utils/pointnav_policy.py) on the library's kernels."""
