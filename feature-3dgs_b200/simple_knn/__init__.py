"""Drop-in for the reference's `simple_knn` extension (submodules/simple-knn): with feature-3dgs_b200 on PYTHONPATH, the
reference's unmodified `from simple_knn._C import distCUDA2` (scene/gaussian_model.py) resolves to this package's native
kernel (csrc/knn.cu) instead of a separately built module."""
