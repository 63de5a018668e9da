"""yadcc_b200 -- H100-native implementation of yadcc's scheduler hot path.

Only what the path needs lives here:

  csrc/            host C++ + sm_90a CUDA kernels behind include/ydsched.h
  _abi.py          ctypes declarations of that C ABI
  dispatcher.py    host-side mirror of the reference's `TaskDispatcher`
                   interface (yadcc/scheduler/task_dispatcher.h:120-181)
  service.py       restatement of `SchedulerServiceImpl`'s request expansion
                   (yadcc/scheduler/scheduler_service_impl.cc:67-318)
  streams.py       seeded synthetic event streams (SURVEY.md 8(d))

The product path is the CUDA library `yadcc_b200/libydsched.so`; importing this
package never touches `oracle/`.
"""
from ._abi import (  # noqa: F401
    GRANT_DTYPE,
    REQ_DTYPE,
    SERVANT_STATE_DTYPE,
    STATUS_ENVIRONMENT_NOT_FOUND,
    STATUS_GRANTED,
    STATUS_TIMEOUT,
    PRIORITY_DEDICATED,
    PRIORITY_UNKNOWN,
    PRIORITY_USER,
    NO_SERVANT,
    cuda_library_path,
    load_library,
)
from .dispatcher import (Servant, RunningTask, TaskAllocation, TaskDispatcher, TaskKeysError, TaskSources, WaitStatus,  # noqa: F401
                         binary_digests, pack_requests, unpack_grants)
