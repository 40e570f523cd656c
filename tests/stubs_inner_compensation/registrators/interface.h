// The stand-in headers of tests/stubs with the inner-compensation members of the reference's
// registrator::Interface (interface.h:89-91, :115; interface.cc:34-36) added, for
// tests/cpp/adapter_compensation_run.cc.  The stand-in Interface is renamed while it is included and the
// reference's name then goes to a class that derives from it and adds the members.
#pragma once
#define Interface InterfaceWithoutCompensation
#include "../../stubs/registrators/interface.h"
#undef Interface

namespace static_map {
namespace registrator {
class Interface : public InterfaceWithoutCompensation {
 public:
  void EnableInnerCompensation() { inner_compensation_ = true; }     // interface.cc:34
  void DisableInnerCompensation() { inner_compensation_ = false; }   // interface.cc:36
 protected:
  bool inner_compensation_ = false;
};
}  // namespace registrator
}  // namespace static_map
