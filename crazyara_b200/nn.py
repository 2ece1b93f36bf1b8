"""Host-side mirror of the reference's NeuralNetAPI (engine/src/nn/neuralnetapi.h:148-311) over the C-ABI.

Same names and argument meaning as the reference class: predict(inputPlanes, valueOutput, probOutputs,
auxiliaryOutputs) on caller-owned host buffers; shape getters.  No fallback: construction raises AraError when the
CUDA library or an sm_90 device is missing.
"""
import ctypes

import numpy as np

from ._lib import AraError, check, lib


_PINNED = {}  # pinned_array: address -> owner whose finaliser frees the block


def _fptr(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


class NeuralNetAPI:
    def __init__(self, ctx="gpu", deviceID=0, batchSize=8, modelDirectory="", enableTensorrt=True, precision="float16"):
        """precision: the reference's UCI option `Precision` (uci/optionsuci.cpp:144): "float16" (default) or "float32"."""
        if ctx != "gpu":
            raise AraError("crazyara_b200 has no CPU context (ctx must be 'gpu')")
        L = lib()
        L.ara_net_create.restype = ctypes.c_void_p
        L.ara_net_create.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.ara_net_destroy.argtypes = [ctypes.c_void_p]
        L.ara_net_shape.argtypes = [ctypes.c_void_p] + [ctypes.POINTER(ctypes.c_int)] * 6
        L.ara_net_predict.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_float), ctypes.c_int,
                                      ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float),
                                      ctypes.POINTER(ctypes.c_float)]
        L.ara_net_forward_device.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                             ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_void_p)]
        L.ara_net_predict_priors.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_float), ctypes.c_int, ctypes.c_void_p,
                                             ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_float),
                                             ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float)]
        L.ara_host_alloc.restype = ctypes.c_void_p
        L.ara_host_alloc.argtypes = [ctypes.c_ulonglong]
        L.ara_host_free.argtypes = [ctypes.c_void_p]
        L.ara_net_launch_count.restype = ctypes.c_longlong
        L.ara_net_launch_count.argtypes = [ctypes.c_void_p]
        if precision not in ("float16", "float32"):
            raise AraError(f"Precision must be float16 or float32, not {precision!r}")
        self.precision = precision
        self._h = L.ara_net_create(modelDirectory.encode(), deviceID, batchSize, 1 if precision == "float32" else 0)
        if not self._h:
            raise AraError(L.ara_last_error().decode())
        v = [ctypes.c_int() for _ in range(6)]
        check(L.ara_net_shape(self._h, *[ctypes.byref(x) for x in v]))
        self.nbInputChannels, self.nbPolicyValues, self.nbAuxiliaryOutputs = v[0].value, v[1].value, v[2].value
        self.isPolicyMap, self.version, self.batchSize = bool(v[3].value), v[4].value, v[5].value
        self.deviceID = deviceID

    # reference getters (nn/neuralnetapi.h:116-293)
    def get_batch_size(self):
        return self.batchSize

    def get_nb_input_values_total(self):
        return self.nbInputChannels * 64

    def get_nb_policy_values(self):
        return self.nbPolicyValues

    def get_nb_auxiliary_outputs(self):
        return self.nbAuxiliaryOutputs

    def is_policy_map(self):
        return self.isPolicyMap

    def get_version(self):
        return self.version

    def predict(self, inputPlanes, valueOutput, probOutputs, auxiliaryOutputs=None, n=None):
        """inputPlanes: float32 [n, C, 8, 8] host array; outputs are written in place (caller-owned buffers)."""
        n = self.batchSize if n is None else n
        for a in (inputPlanes, valueOutput, probOutputs):
            if a.dtype != np.float32 or not a.flags["C_CONTIGUOUS"]:
                raise AraError("predict buffers must be C-contiguous float32")
        aux = _fptr(auxiliaryOutputs) if auxiliaryOutputs is not None else None
        check(lib().ara_net_predict(self._h, _fptr(inputPlanes), n, _fptr(valueOutput), _fptr(probOutputs), aux))

    def predict_priors(self, inputPlanes, policyIdx, counts, valueOutput, priorsOutput, auxiliaryOutputs=None, n=None):
        """fill_nn_results for a host-side tree (searchthread.cpp:290-299, node.cpp:961-979): like predict, but only the
        policy entries policyIdx[b][:counts[b]] of every position come back (priorsOutput [n, stride] float32)."""
        n = self.batchSize if n is None else n
        for a in (inputPlanes, valueOutput, priorsOutput):
            if a.dtype != np.float32 or not a.flags["C_CONTIGUOUS"]:
                raise AraError("predict buffers must be C-contiguous float32")
        idx = np.ascontiguousarray(policyIdx, np.int32)
        cnt = np.ascontiguousarray(counts, np.int32)
        if idx.shape != priorsOutput.shape:
            raise AraError("policyIdx and priorsOutput must have the same [n, stride] shape")
        aux = _fptr(auxiliaryOutputs) if auxiliaryOutputs is not None else None
        check(lib().ara_net_predict_priors(self._h, _fptr(inputPlanes), n, idx.ctypes.data, cnt.ctypes.data, idx.shape[1],
                                           _fptr(valueOutput), _fptr(priorsOutput), aux))

    @staticmethod
    def pinned_array(shape, dtype=np.float32):
        """A numpy array over pinned host memory (ara_host_alloc = cudaMallocHost, as neuralnetapiuser.cpp:52-59 allocates
        the predict buffers); freed when the array is garbage-collected."""
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        p = lib().ara_host_alloc(n)
        if not p:
            raise AraError(lib().ara_last_error().decode())
        buf = (ctypes.c_char * n).from_address(p)
        arr = np.frombuffer(buf, dtype=dtype).reshape(shape)

        class _Owner:
            def __del__(self, p=p):
                lib().ara_host_free(p)
        _PINNED[arr.ctypes.data] = _Owner()
        return arr

    def forward_device(self, planes_dev_ptr, n):
        """planes already in HBM ([n, C, 8, 8] fp32 device pointer, or 0 to use the encoded NHWC input buffer).
        Returns (value_dev_ptr, prob_dev_ptr)."""
        v, p = ctypes.c_void_p(), ctypes.c_void_p()
        check(lib().ara_net_forward_device(self._h, ctypes.c_void_p(planes_dev_ptr), n, ctypes.byref(v), ctypes.byref(p)))
        return v.value, p.value

    def launch_count(self):
        return lib().ara_net_launch_count(self._h)

    def close(self):
        if getattr(self, "_h", None):
            lib().ara_net_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
