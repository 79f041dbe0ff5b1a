// Build configuration, the counterpart of the reference's generated gloo/config.h
// (gloo/config.h.in): version macros and 0/1 feature switches. Nothing is generated here:
// the switches follow the compile definitions the build passes (build.py / CMakeLists.txt).
#pragma once

#define GLB_VERSION_MAJOR 0
#define GLB_VERSION_MINOR 2
#define GLB_VERSION_PATCH 0
#define GLB_VERSION_STRING "0.2.0"
#define GLB_VERSION (GLB_VERSION_MAJOR * 10000 + GLB_VERSION_MINOR * 100 + GLB_VERSION_PATCH)

#ifndef GLB_USE_CUDA
#define GLB_USE_CUDA 0
#endif
#ifndef GLB_USE_MPI
#define GLB_USE_MPI 0
#endif
// NCCL, OpenSSL and libibverbs are looked up with dlopen at run time, never linked.
#define GLB_USE_NCCL_LOAD 1
#define GLB_USE_TCP_OPENSSL_LOAD 1
#define GLB_USE_REDIS 1  // own RESP client, no hiredis

#define GLB_HAVE_TRANSPORT_TCP 1
#define GLB_HAVE_TRANSPORT_TCP_TLS 1
#define GLB_HAVE_TRANSPORT_UV 1       // source-compatible alias of the epoll transport
#define GLB_HAVE_TRANSPORT_IBVERBS 0  // probe + diagnostics only (transport/ibverbs/device.h)
#define GLB_HAVE_TRANSPORT_NVLINK GLB_USE_CUDA  // cuda::PeerContext peer-memory data plane

// The only GPU architecture this library is written for.
#define GLB_CUDA_ARCH "sm_90a"
