"""`from inception import InceptionV3` (fid_score.py:52): the FID Inception-v3 wrapper, on diff_pruning_b200.fid (device feature pass).
The weights are read from a local file (diff_pruning_b200.fid.find_weights); nothing is downloaded."""
from diff_pruning_b200.fid import WEIGHTS_FILE, InceptionV3, find_weights  # noqa: F401

FID_WEIGHTS_URL = "https://github.com/mseitzer/pytorch-fid/releases/download/fid_weights/" + WEIGHTS_FILE   # the name only: never fetched
