"""Dataset readers of the evaluation drivers and the demos (API of the reference's deva/inference/data/) and
``DeviceLoader``, which reads their frames and masks on the device."""
# Modules this package does not provide (the test-dataset listings, ...) resolve to the reference checkout when one is
# on sys.path *after* this package: same-named package directories are chained, ours first (pkgutil.extend_path), so
# the checkout's `vos_test_datasets` etc. import and yield the readers defined here.
from pkgutil import extend_path

__path__ = extend_path(__path__, __name__)
