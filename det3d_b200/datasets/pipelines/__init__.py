from .compose import Compose
from .formating import Reformat
from .loading import LoadPointCloudAnnotations, LoadPointCloudFromFile, ingest_sweeps, ingest_sweeps_batched, read_file
from .preprocess import AssignTarget, Preprocess, Voxelization
