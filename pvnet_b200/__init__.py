from . import optim  # noqa: F401  (pvnet_b200.optim.Adam: the training loop's optimizer)
