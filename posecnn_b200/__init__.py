"""posecnn_b200 — H100-native (sm_90a) implementation of the PoseCNN hot path.

Sub-packages mirror the reference's op modules one to one (lib/<layer>/<layer>_op.py of
yuxng/PoseCNN): put this directory on sys.path and `import hough_voting_gpu_layer.
hough_voting_gpu_op as hough_voting_gpu_op` exactly as lib/networks/network.py:6-26 does.
"""
__version__ = "0.1.0"
