import sys
import os; sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_shim
sys.path.append(ref_shim.REFERENCE_ROOT)               # the reference checkout, or its verbatim copy under oracle/_ref
sys.meta_path.insert(0, ref_shim._MockFinder())        # GUI / mesh libraries are absent in this container
import isdf
from isdf import visualisation
from isdf.modules import trainer, fc_map
from isdf.eval import metrics
from isdf.geometry import transform
print('trainer from', trainer.__file__)
print('visualisation from', visualisation.__file__)
print('metrics.start_timing from', metrics.start_timing.__module__, '| accuracy_comp (fallback):', metrics.accuracy_comp.__module__)
print('transform.ray_dirs_C', transform.ray_dirs_C.__module__, '| to_trimesh (fallback):', transform.to_trimesh.__module__)
import isdf.eval.plot_utils as pu
print('isdf.eval.plot_utils from', pu.__file__)
import isdf.datasets.sdf_util as su
print('isdf.datasets.sdf_util from', su.__file__)
