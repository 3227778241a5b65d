"""Drop-in replacement for the reference's kNN extension `simple_knn` (submodules/simple-knn, built as `simple_knn._C`):
`from simple_knn._C import distCUDA2, distIndex2, distIndexQ` resolves to the H100-native kernels of gs_b200 (gsb_knn)."""
