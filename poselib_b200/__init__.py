"""poselib_b200 — H100-native LO-RANSAC / minimal-solver engine behind PoseLib's call surface."""
__version__ = "0.1.0"
