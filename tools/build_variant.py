"""build_variant.py NAME [extra nvcc flags...] -> variants/liblins_gpu_NAME.so (every translation unit, same flags as the product)."""
import importlib, os, sys
root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, root)
capi = importlib.import_module("lins---lidar-inertial-slam_b200.capi")
capi.build(force=True, out=os.path.join(root, "variants", f"liblins_gpu_{sys.argv[1]}.so"), extra=sys.argv[2:])
