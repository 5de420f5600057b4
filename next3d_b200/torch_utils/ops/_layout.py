"""The memory format at::Tensor::suggest_memory_format() picks, which PyTorch does not expose in Python.  The reference's plugins
allocate their outputs in it (upfirdn2d.cpp:42, filtered_lrelu.cpp:84), so the drop-in ops return the same layouts."""
import torch


def suggest_memory_format(x):
    """channels_last when a 4-D x's strides order its dims C, W, H, N from fastest to slowest (c10's is_channels_last_strides_2d,
    with its tie-breaks towards NCHW for size-1 dims), else contiguous_format.  Dense or not: a channel slice of a channels_last
    tensor suggests channels_last."""
    if x.ndim != 4 or x.layout != torch.strided:
        return torch.contiguous_format
    sizes, strides = x.shape, x.stride()
    if strides[1] == 0:
        return torch.contiguous_format
    least = 0
    for d in (1, 3, 2, 0):
        if sizes[d] == 0 or strides[d] < least or (d == 0 and least == strides[1]):
            return torch.contiguous_format
        least = strides[d] * max(sizes[d], 1)
    return torch.channels_last
