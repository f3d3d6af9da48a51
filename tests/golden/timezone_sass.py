"""SASS fixtures (data only): the SHA-256 of each timezone.cu kernel's `cuobjdump -sass` listing (instructions and their
encodings, the anonymous-namespace hash in the names removed), compiled for sm_90a with -O3 by CUDA 12.9 (V12.9.86) from
timezone.cu as it stood before its zone evaluation moved into tz_eval.cuh.  The kernels must still compile to these."""
NVCC_RELEASE = "release 12.9, V12.9.86"
KERNELS = {
    '_ZN3srj44_GLOBAL__N__11_timezone_cu_9a93aace13orc_tz_kernelEPKlPllbS2_PKiiiS2_S5_ii' : 'e9037c9b6057c52a79f4c454ac5dc2f5f09706533ce2ffc3b0218118dc8e6e6d',
    '_ZN3srj44_GLOBAL__N__11_timezone_cu_9a93aace15tz_multi_kernelEPKlPKiPKhS6_S4_S4_NS0_7TzTableElPlPjPy' : '204193c188411efa1ecb29c648bab60b6b58f98389c1b1742c12fdf39114afad',
    '_ZN3srj44_GLOBAL__N__11_timezone_cu_9a93aace17tz_convert_kernelILl1000000000ELb0EEEvPKlPllbS3_PKiiS6_' : 'd1cd5d9ebdd720ae2f402f6b637e475b88bf25657eb64a4ecf06e26e800676ec',
    '_ZN3srj44_GLOBAL__N__11_timezone_cu_9a93aace17tz_convert_kernelILl1000000000ELb1EEEvPKlPllbS3_PKiiS6_' : '24a819e8c191ee2fff5beccc2036707e032b97c32be8523226e9b39ea35d98ce',
    '_ZN3srj44_GLOBAL__N__11_timezone_cu_9a93aace17tz_convert_kernelILl1000000ELb0EEEvPKlPllbS3_PKiiS6_' : '8401357e1a1864591e29047a811c4d80dd4f8ceb76628e9fda77d6dc1ee2840c',
    '_ZN3srj44_GLOBAL__N__11_timezone_cu_9a93aace17tz_convert_kernelILl1000000ELb1EEEvPKlPllbS3_PKiiS6_' : '558a05e29a07e8c2354bf235f5a506cef6a16292f0eb5c236f712ba51da38db2',
    '_ZN3srj44_GLOBAL__N__11_timezone_cu_9a93aace17tz_convert_kernelILl1000ELb0EEEvPKlPllbS3_PKiiS6_' : 'babf2c2424541a003d1b5c474fcc066d6995b07d2c8ca11f07fb645246cc557d',
    '_ZN3srj44_GLOBAL__N__11_timezone_cu_9a93aace17tz_convert_kernelILl1000ELb1EEEvPKlPllbS3_PKiiS6_' : 'b40c69e617fa486aad9f1e7fad595bafb0c01885bc5e6a341e10fa7b90710ad8',
    '_ZN3srj44_GLOBAL__N__11_timezone_cu_9a93aace17tz_convert_kernelILl1ELb0EEEvPKlPllbS3_PKiiS6_' : '607721e7d4646bd290038186e12565e167355c750346b4b6970264fdeb42d90e',
    '_ZN3srj44_GLOBAL__N__11_timezone_cu_9a93aace17tz_convert_kernelILl1ELb1EEEvPKlPllbS3_PKiiS6_' : 'af346489bafc1a16b8e294b56bbc537abb9c22093070b231b69caee8ad3bf2e7',
}
