from . import data_util, dataset, sdf_util  # noqa: F401
