"""Drop-in name.  `src/scene/gaussian_model.py:21` of the reference does

    from simple_knn._C import distCUDA2

Putting this repository's root on `sys.path` makes that import resolve to the H100-native implementation in
`gaussianhaircut_b200.knn`.  Importing it neither loads the native library nor touches CUDA.
"""
