"""TEST INFRASTRUCTURE: builds oracle/liboracle.so (+ oracle/_ref when /root/reference exists)."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "liboracle.so")
REF_LIB = os.path.join(HERE, "_ref", "libiou3d_ref.so")
REF_VOXEL_SRC = "/root/reference/det3d/ops/point_cloud/point_cloud_ops.py"
REF_VOXEL_NAME = "ref_voxel_aot"


def _stale(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def build(force=False):
    srcs = [os.path.join(HERE, f) for f in ("voxel_oracle.c", "iou3d_oracle.c", "Makefile")]
    if force or _stale(LIB, srcs):
        subprocess.run(["make", "-C", HERE, "liboracle.so"] + (["-B"] if force else []), check=True,
                       stdout=subprocess.DEVNULL)
    ref_src = "/root/reference/det3d/ops/iou3d/src/iou3d_kernel.cu"
    # rebuilt when the recipe (architecture flags) changed, not only when missing: an image for another GPU does not load
    if os.path.exists(ref_src) and (force or _stale(REF_LIB, [ref_src, os.path.join(HERE, "Makefile")])):
        subprocess.run(["make", "-C", HERE, "ref"], check=True, stdout=subprocess.DEVNULL)
    build_ref_voxel(force)
    return LIB


def ref_voxel_path():
    """Path of the AOT-compiled reference voxelizer kernel in oracle/_ref (None if it was never built)."""
    d = os.path.join(HERE, "_ref")
    if os.path.isdir(d):
        for f in sorted(os.listdir(d)):
            if f.startswith(REF_VOXEL_NAME) and f.endswith(".so"):
                return os.path.join(d, f)
    return None


def build_ref_voxel(force=False):
    """oracle/_ref/ref_voxel_aot*.so: the REFERENCE's own numba kernel `_points_to_voxel_reverse_kernel`
    (det3d/ops/point_cloud/point_cloud_ops.py:7-55), loaded from the source where it lies and compiled ahead of time
    with numba.pycc -- a build output like libiou3d_ref.so (travels to the GPU box, never committed, no source copied).
    Only possible in the container that has /root/reference; elsewhere the prebuilt file is used."""
    if not os.path.exists(REF_VOXEL_SRC) or (ref_voxel_path() is not None and not force):
        return ref_voxel_path()
    try:
        import importlib.util
        import warnings
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            from numba.pycc import CC
            spec = importlib.util.spec_from_file_location("_ref_point_cloud_ops", REF_VOXEL_SRC)
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)
            cc = CC(REF_VOXEL_NAME)
            cc.output_dir = os.path.join(HERE, "_ref")
            cc.verbose = False
            # (points, voxel_size, coors_range, num_points_per_voxel, coor_to_voxelidx, voxels, coors, max_points, max_voxels)
            cc.export("points_to_voxel_reverse_kernel",
                      "i8(f4[:,:], f4[:], f4[:], i4[:], i4[:,:,:], f4[:,:,:], i4[:,:], i8, i8)")(
                mod._points_to_voxel_reverse_kernel.py_func)
            cc.compile()
    except Exception as e:      # numba.pycc is deprecated: treat its absence as "reference kernel unbuildable here"
        print("oracle: reference voxelizer AOT build skipped (%s: %s)" % (type(e).__name__, e))
    return ref_voxel_path()


if __name__ == "__main__":
    print(build(force=True))
