// fast_pass.cuh -- specialised pass kernel for 4-channel images: device code in
// fast_kernel.cuh, host side (effective phases, tile choice, launch) in fast_host.cuh.
#pragma once

#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <mutex>
#include <utility>
#include <vector>

#include "fast_kernel.cuh"
#include "host_util.h"

namespace avb {

#include "fast_host.cuh"
