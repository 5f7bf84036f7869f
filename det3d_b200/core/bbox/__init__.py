from . import box_coders, box_np_ops, box_torch_ops
