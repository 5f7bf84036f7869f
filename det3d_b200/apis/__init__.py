from .dist import all_gather_detections, init_from_env, interleave_rank_major, shard_indices
from .pipeline import InferencePipeline, PendingResult, SweepStream
