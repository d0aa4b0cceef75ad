// awm_engine.hh -- owner of the GPU context (awm_ctx) used by the host-side drivers.
// Replaces the reference's per-thread FFTProcessor / ThreadPool fan-out: one context, one stream,
// key tables uploaded once per key.  If no CUDA device is usable every operation fails: there is
// deliberately no CPU fallback.
#pragma once
#include <string>
#include <vector>
#include "awm_random.hh"
#include "awm_tables.hh"
#include "../../include/awm_b200.h"

class Engine
{
public:
  static awm_ctx *ctx();                       // nullptr (after logging) if the context cannot be created
  static void     shutdown();
  static int      key_slot (const Key& key);   // uploads sync (BLOCK + CLIP) and mix tables on first use; -1 on error
  static bool     set_embed_tables (const Key& key, const std::vector<int>& bitvec);
  static bool     set_embed_roles (const Key& key);    // role table of the batched embed, uploaded once per key / layout
  static std::string last_error();
  static bool     is_device_pointer (const void *p);   // true if p is CUDA device (or managed) memory
};
