// Instantiation group 3 of the streaming tensor-product kernels (see the end of tp_stream.cu), compiled as its own
// translation unit so that the build compiles the groups in parallel.
#define AB2_TP_STREAM_GROUP 3
#include "tp_stream.cu"
