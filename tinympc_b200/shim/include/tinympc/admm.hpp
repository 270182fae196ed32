// forwarding header: the reference layout <tinympc/admm.hpp> -> the H100 shim
#pragma once
#include "../../tinympc_shim.hpp"
